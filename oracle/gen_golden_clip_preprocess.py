"""Generate tests/golden/clip_preprocess_u8.npz from the REFERENCE'S OWN CODE  --  run in the build container only.

    python oracle/gen_golden_clip_preprocess.py [/root/reference]

The non-HD input path of the reference decodes an image with PIL (``Image.open(...).convert('RGB')``), pads it to a square with
``expand2square`` when ``image_aspect_ratio == 'pad'`` (llava/mm_utils.py:14-25; the same block at llava/train/train.py:680-692)
and runs ``CLIPImageProcessor.preprocess`` on it.  Here:

  * the images are PIL images built from seeded uint8 arrays (``Image.fromarray``, clip_preprocess_oracle.test_image)
  * ``expand2square`` is llava/mm_utils.py:14-25 exec'd verbatim, with the background ``tuple(int(x*255) for x in image_mean)``
  * the processor is the slow (PIL) CLIP processor that transformers 4.31, the version the reference pins, calls
    ``CLIPImageProcessor``; transformers >= 5 names it ``CLIPImageProcessorPil`` (its default ``CLIPImageProcessor`` is a
    torchvision "fast" processor with other bits).  The openai/clip-vit-large-patch14-336 configuration is written out below, so
    nothing is downloaded.

Per case the fixture holds the metadata (h, w, mode, seed), the SHA-256 of the float32 output bytes ([3, 336, 336], C order), a
probe grid and per-channel sums.  It also holds the (channel, byte) -> float32 table as the processor produced it from a 336 x 336
image in which every byte value occurs in every channel: no resize and no crop happen there, so the output is the table.
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np
import PIL
import transformers
from PIL import Image
from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import clip_preprocess_oracle as cpo                       # noqa: E402
from oracle.gen_golden import OUT, source_range                         # noqa: E402

# openai/clip-vit-large-patch14-336 preprocessor_config.json
IMAGE_MEAN = [0.48145466, 0.4578275, 0.40821073]
IMAGE_STD = [0.26862954, 0.26130258, 0.27577711]
PROCESSOR = dict(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336}, do_resize=True, do_center_crop=True,
                 do_rescale=True, rescale_factor=0.00392156862745098, do_normalize=True, image_mean=IMAGE_MEAN, image_std=IMAGE_STD,
                 resample=3, do_convert_rgb=True)

# (h, w, mode, seed): both orientations, an odd L - w, 336 x 336, a short side of exactly 336 (square), an upscale, a 20:1 strip and
# one large image, in both modes
CASES = [(480, 640, "pad", 700), (640, 480, "pad", 701), (500, 333, "pad", 702), (336, 336, "pad", 703), (120, 90, "pad", 704),
         (30, 600, "pad", 705), (3000, 4000, "pad", 706),
         (480, 640, "square", 710), (640, 480, "square", 711), (500, 333, "square", 712), (336, 336, "square", 713),
         (336, 500, "square", 714), (700, 336, "square", 715), (120, 90, "square", 716), (30, 600, "square", 717),
         (3000, 4000, "square", 718)]
PROBE = (slice(None), slice(None, None, 37), slice(None, None, 41))


def ref_expand2square():
    src = source_range("llava/mm_utils.py", 14, 25)
    assert src.startswith("def expand2square(pil_img, background_color):"), src[:80]
    ns = {"Image": Image}
    exec(src, ns)
    return ns["expand2square"]


def digest(x) -> str:
    return hashlib.sha256(np.ascontiguousarray(x, dtype=np.float32).tobytes()).hexdigest()


def main():
    expand2square = ref_expand2square()
    background = tuple(int(x * 255) for x in IMAGE_MEAN)                  # train.py:690, mm_utils.py:36
    assert background == cpo.BACKGROUND
    proc = CLIPImageProcessorPil(**PROCESSOR)

    def run(pixels, mode):
        img = Image.fromarray(pixels)
        if mode == "pad":
            img = expand2square(img, background)
        out = proc.preprocess(img, return_tensors="np")["pixel_values"][0]
        assert out.dtype == np.float32 and out.shape == (3, 336, 336), (out.dtype, out.shape)
        return out

    out = {}
    for ci, (h, w, mode, seed) in enumerate(CASES):
        t = run(cpo.test_image(h, w, seed), mode)
        out[f"case{ci}_meta"] = np.asarray([h, w, cpo.MODES.index(mode), seed], dtype=np.int64)
        out[f"case{ci}_sha256"] = np.asarray(digest(t))
        out[f"case{ci}_probe"] = t[PROBE].astype(np.float32)
        out[f"case{ci}_sum"] = t.astype(np.float64).sum(axis=(1, 2))
        print("clip preprocess", h, w, mode, seed, digest(t)[:16])
    out["n_cases"] = np.asarray(len(CASES))
    ramp = cpo.test_image(336, 336, -1)
    t = run(ramp, "square")
    table = np.zeros((3, 256), dtype=np.float32)
    for c in range(3):
        for u in range(256):
            vals = t[c][ramp[:, :, c] == u]
            assert vals.size > 0 and np.all(vals.view(np.uint32) == vals[0].view(np.uint32))
            table[c, u] = vals[0]
    out["table"] = table
    out["versions"] = np.asarray(f"Pillow {PIL.__version__}, transformers {transformers.__version__} (CLIPImageProcessorPil)")
    np.savez_compressed(os.path.join(OUT, "clip_preprocess_u8.npz"), **out)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    main()
