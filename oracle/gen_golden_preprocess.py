"""Generate tests/golden/hd_preprocess_u8.npz from the REFERENCE ITSELF  --  run in the build container only.

    python oracle/gen_golden_preprocess.py [/root/reference]

Its own entry so that the fixtures of oracle/gen_golden.py are not rewritten.  The HD input path of the reference decodes an image
with PIL (``Image.open(...).convert('RGB')``), normalises it with ``preprocess`` and runs the tiling block on the result.  Here:

  * the images are PIL images built from seeded uint8 arrays (``Image.fromarray``, hd_preprocess_oracle.u8_test_image)
  * ``preprocess`` is ``llava/eval/model_vqa.py:62`` exec'd verbatim (Compose([ToTensor(), Normalize(CLIP mean, std)]))
  * the tiling block is ``llava/eval/model_vqa.py:88-123`` exec'd verbatim, as in gen_golden.gen_tile

The fixture holds per case the metadata, per-crop sums and absolute sums and a probe grid (like hd_tile.npz), and the 768-entry
normalisation table as the reference's ``preprocess`` produced it (a 1 x 256 image whose pixel u has byte u in every channel).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image
from torchvision.transforms import Compose, Normalize, ToTensor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import hd_preprocess_oracle as hpo                         # noqa: E402
from oracle.gen_golden import OUT, load_by_path, source_range           # noqa: E402

# the six sizes of gen_golden.gen_tile, on seeded bytes; then a ramp in which every byte value occurs in every channel
CASES = [(500, 700, 9, 500), (1088, 1088, 9, 501), (336, 336, 9, 502), (224, 1344, 9, 503), (901, 333, 16, 504), (640, 1500, 25, 505),
         (300, 457, 9, -1)]


def ref_preprocess():
    src = source_range("llava/eval/model_vqa.py", 62, 62)
    assert src.startswith("preprocess = Compose([ToTensor(), Normalize("), src
    ns = {"Compose": Compose, "ToTensor": ToTensor, "Normalize": Normalize}
    exec(src, ns)
    return ns["preprocess"]


def gen_preprocess(pd):
    preprocess = ref_preprocess()
    tile = source_range("llava/eval/model_vqa.py", 88, 123)
    assert tile.lstrip().startswith("image = preprocess(image)"), tile[:80]
    out = {}
    for ci, (h, w, patch_num, seed) in enumerate(CASES):
        pixels = hpo.u8_test_image(h, w, seed)
        ns = {"image": Image.fromarray(pixels), "preprocess": preprocess,
              "image_patch": pd.Image_Patch(image_size=336, patch_num=patch_num), "F": F, "torch": torch}
        exec(tile, ns)
        t = ns["image_tensor"].numpy()
        out[f"case{ci}_meta"] = np.asarray([h, w, patch_num, ns["h_block"], ns["w_block"], seed], dtype=np.int64)
        out[f"case{ci}_sum"] = t.astype(np.float64).sum(axis=(1, 2, 3))
        out[f"case{ci}_abs"] = np.abs(t.astype(np.float64)).sum(axis=(1, 2, 3))
        out[f"case{ci}_probe"] = t[:, :, ::37, ::41].astype(np.float32)
        print("preprocess+tile", h, w, patch_num, seed, t.shape)
    out["n_cases"] = np.asarray(len(CASES))
    ramp = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)        # [1, 256, 3]
    out["table"] = preprocess(Image.fromarray(ramp)).numpy()[:, 0, :].astype(np.float32)   # [3, 256]
    np.savez(os.path.join(OUT, "hd_preprocess_u8.npz"), **out)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    gen_preprocess(load_by_path("ref_patch_divide", "llava/patch_divide.py"))
