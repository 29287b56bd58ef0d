"""Gradients to the pixels under torch autograd, independent of the kernels: the yardstick of
include/tokenpacker_b200_clip_tower_crop_grad.h.

``crop_gradients`` is the whole tower (clip_tower_embed_oracle.embedding_stage, then clip_tower_train_oracle.layer) with the crops as a
leaf that requires grad, and a weighted-sum loss over hidden states.  ``tile`` restates the HD tiling block (train.py:695-731) with
torch ops (F.interpolate, zero padding, the split into crops, the thumbnail), so that autograd gives its adjoint in any dtype.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import clip_tower_embed_oracle as cte
from oracle import clip_tower_train_oracle as ctt
from oracle import hd_oracle

BLOCK = 336


def crop_gradients(w, images, d_outs, n_layers=23, dtype=torch.float64, device="cpu"):
    """Gradient of loss = sum_j <d_outs[j], hidden_states[j]> (d_outs: {j: tensor or None}, 0 <= j <= n_layers) w.r.t. the crops
    [N, 3, 336, 336], every op in ``dtype``."""
    e = {k: w[k].to(device=device, dtype=dtype) for k in cte.EMBED_KEYS}
    x0 = images.to(device=device, dtype=dtype).clone().requires_grad_(True)
    x = cte.embedding_stage(e, x0)
    hs = {0: x}
    for i in range(n_layers):
        x = ctt.layer(ctt.layer_params(w, i, dtype, device), x)
        hs[i + 1] = x
    loss = sum((hs[j] * d.to(device=device, dtype=dtype)).sum() for j, d in d_outs.items() if d is not None)
    loss.backward()
    return x0.grad


def crop_gradients_chunked(w, images, d_outs, chunk, n_layers=23, dtype=torch.float64, device="cpu"):
    """crop_gradients over ``chunk`` crops at a time (each crop's gradient depends on that crop alone)."""
    parts = []
    for c0 in range(0, images.shape[0], chunk):
        part = {j: None if d is None else d[c0:c0 + chunk] for j, d in d_outs.items()}
        parts.append(crop_gradients(w, images[c0:c0 + chunk], part, n_layers, dtype, device))
    return torch.cat(parts, dim=0)


def tile(image, patch_num: int = 9):
    """train.py:695-731 with torch ops.  image: [3, h, w] (any float dtype, may require grad).  Returns (crops [n, 3, 336, 336], hb, wb):
    the grid from hd_oracle.hd_grid, the bilinear resize (align_corners=False, scale from sizes) into the zero-padded canvas, its crops
    row-major, and, when there is more than one, the thumbnail resized from the padded canvas, last."""
    h, w = int(image.shape[-2]), int(image.shape[-1])
    hb, wb = hd_oracle.hd_grid(h, w, patch_num)
    h_, w_ = hd_oracle._fit(h, w, hb, wb)
    resized = F.interpolate(image[None], size=(h_, w_), mode="bilinear", align_corners=False)
    canvas = F.pad(resized, (0, BLOCK * wb - w_, 0, BLOCK * hb - h_))
    crops = [canvas[:, :, BLOCK * i:BLOCK * (i + 1), BLOCK * j:BLOCK * (j + 1)] for i in range(hb) for j in range(wb)]
    if len(crops) > 1:
        th, tw = hd_oracle._fit(h, w, 1, 1)
        thumb = F.interpolate(canvas, size=(th, tw), mode="bilinear", align_corners=False)
        crops.append(F.pad(thumb, (0, BLOCK - tw, 0, BLOCK - th)))
    return torch.cat(crops, dim=0), hb, wb


def tile_gradients(images, d_crops, patch_num: int = 9, dtype=torch.float64):
    """d images (one [3, h, w] per image, in ``dtype``) of loss = <d_crops, the crops of the batch> (crops image by image, as
    tp_hd_tile_batch orders them)."""
    leaves = [im.detach().to(dtype).cpu().requires_grad_(True) for im in images]
    crops = torch.cat([tile(x, patch_num)[0] for x in leaves], dim=0)
    (crops * d_crops.detach().to(dtype).cpu()).sum().backward()
    return [x.grad for x in leaves]
