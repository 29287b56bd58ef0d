"""The whole CLIP tower under torch autograd, embedding stage included, independent of transformers: the yardstick of the
whole-tower training path (include/tokenpacker_b200_clip_tower_embed.h).

``embedding_stage`` is the bottom of the tower written out with explicit tensor ops: the 14 x 14 / 14 patch convolution (no bias), the
class embedding in front, the position embedding added, pre_layrnorm.  ``parameter_gradients`` is the training step of the tests with
every parameter trainable: the embedding stage, then layers 0 .. n_layers - 1 (clip_tower_train_oracle.layer), a weighted-sum loss
over any hidden states (not only 12 / 16 / 22 / 23, so that a tower of a few layers can be checked too), autograd.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import clip_tower_oracle as cto
from oracle import clip_tower_train_oracle as ctt

EMBED_KEYS = ("embeddings.patch_embedding.weight", "embeddings.class_embedding", "embeddings.position_embedding.weight",
              "pre_layrnorm.weight", "pre_layrnorm.bias")                      # the order of _lib.CLIP_TOWER_FIELDS


def embedding_stage(e, images):
    """e: EMBED_KEYS -> tensor; images [N, 3, 336, 336] -> hidden_states[0] [N, 577, 1024]."""
    n = images.shape[0]
    patches = F.conv2d(images, e["embeddings.patch_embedding.weight"], stride=cto.PATCH).flatten(2).transpose(1, 2)
    cls = e["embeddings.class_embedding"].expand(n, 1, cto.HIDDEN)
    emb = torch.cat([cls, patches], dim=1) + e["embeddings.position_embedding.weight"]
    return ctt._layer_norm(emb, e["pre_layrnorm.weight"], e["pre_layrnorm.bias"])


def parameter_gradients(w, images, d_outs, n_layers=23, dtype=torch.float64, device="cpu"):
    """Gradients of loss = sum_j <d_outs[j], hidden_states[j]> (d_outs: {j: tensor or None}, 0 <= j <= n_layers) w.r.t. every
    parameter of the embedding stage and of layers 0 .. n_layers - 1.  Returns (EMBED_KEYS -> gradient, a list of n_layers dicts
    clip_tower_train_oracle.PARAM_KEYS -> gradient, {j: hidden_states[j]} for every j)."""
    e = {k: w[k].to(device=device, dtype=dtype).clone().requires_grad_(True) for k in EMBED_KEYS}
    params = [{k: v.clone().requires_grad_(True) for k, v in ctt.layer_params(w, i, dtype, device).items()} for i in range(n_layers)]
    x = embedding_stage(e, images.to(device=device, dtype=dtype))
    hs = {0: x}
    for i in range(n_layers):
        x = ctt.layer(params[i], x)
        hs[i + 1] = x
    loss = sum((hs[j] * d.to(device=device, dtype=dtype)).sum() for j, d in d_outs.items() if d is not None)
    loss.backward()
    return ({k: e[k].grad for k in EMBED_KEYS}, [{k: p[k].grad for k in ctt.PARAM_KEYS} for p in params],
            {j: h.detach() for j, h in hs.items()})


def parameter_gradients_chunked(w, images, d_outs, chunk, n_layers=23, dtype=torch.float64, device="cpu"):
    """parameter_gradients over ``chunk`` crops at a time, summed (the loss is a sum over crops): the same gradients with the
    attention probabilities of ``chunk`` crops alive at once.  Returns (embedding gradients, layer gradients)."""
    total = None
    for c0 in range(0, images.shape[0], chunk):
        part = {j: None if d is None else d[c0:c0 + chunk] for j, d in d_outs.items()}
        eg, lg, _ = parameter_gradients(w, images[c0:c0 + chunk], part, n_layers, dtype, device)
        if total is None:
            total = (eg, lg)
        else:
            total = ({k: total[0][k] + eg[k] for k in EMBED_KEYS},
                     [{k: a[k] + b[k] for k in ctt.PARAM_KEYS} for a, b in zip(total[1], lg)])
    return total
