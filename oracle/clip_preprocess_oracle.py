"""CPU oracle for the non-HD CLIP input path (``clip_preprocess_batch``)  --  TEST INFRASTRUCTURE ONLY (see tokenpacker_oracle.py).

numpy restatement, needing neither PIL nor transformers, of what the released non-HD recipes do to a decoded RGB image:

  1. pad mode only: ``expand2square(image, tuple(int(x * 255) for x in image_processor.image_mean))``  (llava/mm_utils.py:14-25,
     llava/train/train.py:680-692), pasting the image into the middle of a square canvas of the CLIP mean colour (122, 116, 104)
  2. ``CLIPImageProcessor.preprocess`` of transformers 4.31 (the slow, PIL-based processor; ``CLIPImageProcessorPil`` in
     transformers >= 5) with the openai/clip-vit-large-patch14-336 configuration: shortest edge -> 336 with PIL's 8-bit BICUBIC
     resample, center crop 336 x 336, rescale by 1/255, normalise by the CLIP mean and std

PIL's 8-bit resample is fixed-point: coefficients in double precision, rounded to int32 with 22 fraction bits, a horizontal and
then a vertical pass with a clipped uint8 image in between.  ``coeffs`` restates ``precompute_coeffs`` + ``normalize_coeffs_8bpc``
of Pillow's Resample.c operation for operation (sequential sums, truncating int conversions), so the result is PIL's, bit for bit.
The final (channel, byte) -> float32 map is ``table()``, which has the bits of ``tokenpacker_b200.hd.norm_table()``.
"""
from __future__ import annotations

import numpy as np

from oracle.hd_preprocess_oracle import CLIP_MEAN, CLIP_STD

SIZE = 336                                      # shortest edge and crop of openai/clip-vit-large-patch14-336
PRECISION_BITS = 22                             # Resample.c: 32 - 8 - 2
BACKGROUND = (122, 116, 104)                    # tuple(int(x * 255) for x in OPENAI_CLIP_MEAN)
RESCALE = 0.00392156862745098                   # 1 / 255 as the processor config spells it
MODES = ("square", "pad")


def bicubic(x):
    """Resample.c bicubic_filter (a = -0.5), elementwise on float64, same operation order."""
    a = -0.5
    x = np.abs(np.asarray(x, dtype=np.float64))
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def coeffs(in_size: int, out_size: int):
    """precompute_coeffs + normalize_coeffs_8bpc for BICUBIC over the box [0, in_size).
    Returns (xmin [out] int64, count [out] int64, k [out, ksize] int64: the int32 weights, zero past count)."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    ss = 1.0 / filterscale
    x = np.arange(ksize, dtype=np.int64)[None, :]
    live = x < xmax[:, None]
    w = np.where(live, bicubic(((x + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * ss), 0.0)
    ww = np.zeros(out_size, dtype=np.float64)
    for j in range(ksize):                      # the sum is sequential in Resample.c; numpy's pairwise sum could differ in the last bit
        ww = ww + w[:, j]
    nz = ww != 0.0
    w = np.where(nz[:, None], w / np.where(nz, ww, 1.0)[:, None], w)
    one = float(1 << PRECISION_BITS)
    k = np.where(w < 0, (-0.5 + w * one).astype(np.int64), (0.5 + w * one).astype(np.int64))
    return xmin, xmax, np.where(live, k, 0)


def resample_axis(img, axis: int, out_size: int, first: int = 0, count: int | None = None):
    """One 8-bit pass of PIL's resample along ``axis`` (0 rows, 1 columns) of uint8 [h, w, 3], keeping outputs [first, first+count)."""
    in_size = img.shape[axis]
    count = out_size - first if count is None else count
    xmin, n, k = coeffs(in_size, out_size)
    xmin, n, k = xmin[first:first + count], n[first:first + count], k[first:first + count]
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((count,) + src.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for j in range(k.shape[1]):
        idx = np.minimum(xmin + j, in_size - 1)             # the weight is 0 past the count; any valid index will do
        acc += src[idx] * k[:, j][:, None, None]
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img, out_h: int, out_w: int):
    """``PIL.Image.resize((out_w, out_h), BICUBIC, reducing_gap=None)`` of uint8 [h, w, 3]: the horizontal pass, then the vertical
    one; a pass whose axis keeps its size is skipped, as in Resample.c."""
    img = np.asarray(img, dtype=np.uint8)
    if out_w != img.shape[1]:
        img = resample_axis(img, 1, out_w)
    if out_h != img.shape[0]:
        img = resample_axis(img, 0, out_h)
    return img


def geometry(h: int, w: int, mode: str):
    """Per-image plan: canvas size, paste offsets, resized size, crop offsets (what tp_clip_preprocess_plan computes)."""
    if mode not in MODES:
        raise ValueError(mode)
    ch, cw, py, px = h, w, 0, 0
    if mode == "pad" and h != w:
        side = max(h, w)
        ch = cw = side
        if w > h:
            py = (w - h) // 2
        else:
            px = (h - w) // 2
    short, long = (cw, ch) if cw <= ch else (ch, cw)
    if short == SIZE:
        rh, rw = ch, cw
    else:
        new_long = int(SIZE * long / short)
        rh, rw = (new_long, SIZE) if cw <= ch else (SIZE, new_long)
    return {"canvas_h": ch, "canvas_w": cw, "pad_y": py, "pad_x": px, "rh": rh, "rw": rw,
            "top": (rh - SIZE) // 2, "left": (rw - SIZE) // 2}


def canvas(pixels, mode: str):
    """expand2square's canvas (pad mode) or the image itself (square mode), uint8 [L, L, 3] / [h, w, 3]."""
    pixels = np.asarray(pixels, dtype=np.uint8)
    h, w = pixels.shape[:2]
    g = geometry(h, w, mode)
    if (g["canvas_h"], g["canvas_w"]) == (h, w):
        return pixels
    out = np.empty((g["canvas_h"], g["canvas_w"], 3), dtype=np.uint8)
    out[:] = BACKGROUND
    out[g["pad_y"]:g["pad_y"] + h, g["pad_x"]:g["pad_x"] + w] = pixels
    return out


def resize_crop_u8(pixels, mode: str):
    """Steps 1-4: the 336 x 336 uint8 crop, [336, 336, 3].  Only the kept columns and the rows the vertical pass reads are computed."""
    pixels = np.asarray(pixels, dtype=np.uint8)
    g = geometry(pixels.shape[0], pixels.shape[1], mode)
    img = canvas(pixels, mode)
    ch, cw = img.shape[:2]
    if g["rh"] != ch:
        ymin, yn, _ = coeffs(ch, g["rh"])
        r0 = int(ymin[g["top"]:g["top"] + SIZE].min())
        r1 = int((ymin + yn)[g["top"]:g["top"] + SIZE].max())
    else:
        r0, r1 = g["top"], g["top"] + SIZE
    rows = img[r0:r1]
    if g["rw"] != cw:
        rows = resample_axis(rows, 1, g["rw"], g["left"], SIZE)
    else:
        rows = rows[:, g["left"]:g["left"] + SIZE]
    if g["rh"] != ch:
        # the vertical pass on rows r0.. of the canvas: shift its bounds by r0, as Resample.c does after its row-limited horizontal pass
        ymin, yn, k = coeffs(ch, g["rh"])
        ymin, k = ymin[g["top"]:g["top"] + SIZE] - r0, k[g["top"]:g["top"] + SIZE]
        src = rows.astype(np.int64)
        acc = np.full((SIZE, SIZE, 3), 1 << (PRECISION_BITS - 1), dtype=np.int64)
        for j in range(k.shape[1]):
            acc += src[np.minimum(ymin + j, src.shape[0] - 1)] * k[:, j][:, None, None]
        return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.ascontiguousarray(rows)


def table():
    """float32 [3, 256]: float32(u * (1/255) in float64), then (x - mean) / std in float32 (the processor's rescale + normalize)."""
    resc = (np.arange(256, dtype=np.float64) * RESCALE).astype(np.float32)
    return ((resc[None, :] - CLIP_MEAN[:, None]) / CLIP_STD[:, None]).astype(np.float32)


def clip_preprocess(pixels, mode: str):
    """The whole pipeline for one decoded RGB image uint8 [h, w, 3] -> float32 [3, 336, 336]."""
    crop = resize_crop_u8(pixels, mode)
    t = table()
    return np.stack([t[c][crop[:, :, c]] for c in range(3)])


def test_image(h: int, w: int, seed: int):
    """Seeded uniform bytes uint8 [h, w, 3]; seed < 0: a ramp in which every byte value occurs in every channel once h * w >= 256."""
    if seed >= 0:
        return np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    i = np.arange(h * w, dtype=np.int64).reshape(h, w)
    return np.stack([(i + 85 * c) % 256 for c in range(3)], axis=-1).astype(np.uint8)
