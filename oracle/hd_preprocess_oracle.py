"""CPU oracle for decoded 8-bit images entering the TokenPacker-HD front end  --  TEST INFRASTRUCTURE ONLY (see tokenpacker_oracle.py).

numpy restatement of ``preprocess = Compose([ToTensor(), Normalize(CLIP mean, CLIP std)])`` (llava/train/train.py:645; the same
line at llava/eval/model_vqa.py:62), which every HD recipe applies to the decoded RGB image before the tiling block that
``hd_oracle.hd_tile`` restates.  Also the seeded pixels of the cases of ``tests/golden/hd_preprocess_u8.npz``, which
``oracle/gen_golden_preprocess.py`` generates from the reference itself.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32

# Normalize((0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711))   train.py:645, model_vqa.py:62
CLIP_MEAN = np.asarray([0.48145466, 0.4578275, 0.40821073], dtype=f32)
CLIP_STD = np.asarray([0.26862954, 0.26130258, 0.27577711], dtype=f32)


def preprocess_u8(pixels):
    """ToTensor + Normalize of a decoded RGB image, uint8 [h,w,3] (np.array of the PIL image) -> float32 [3,h,w]: u / 255, minus
    the channel mean, over the channel std, each step rounded to float32."""
    x = np.asarray(pixels, dtype=np.uint8).transpose(2, 0, 1).astype(f32) / f32(255)
    return ((x - CLIP_MEAN[:, None, None]) / CLIP_STD[:, None, None]).astype(f32)


def u8_test_image(h: int, w: int, seed: int):
    """The uint8 [h,w,3] pixels of a fixture case: seeded uniform bytes, or for seed < 0 a ramp in which every byte value occurs in
    every channel once h * w >= 256."""
    if seed >= 0:
        return np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    i = np.arange(h * w, dtype=np.int64).reshape(h, w)
    return np.stack([(i + 85 * c) % 256 for c in range(3)], axis=-1).astype(np.uint8)
