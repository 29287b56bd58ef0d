"""transformers' CLIP-ViT-L/14-336 tower in a 16-bit dtype, for the fp16 tower the reference's evaluation and serving scripts run
(``vision_tower.to(dtype=torch.float16)``, llava/eval/model_vqa_loader.py:143; images cast to the tower's dtype, clip_encoder.py:59).

``forward_eager(w, images, n_layers, dtype)`` is ``clip_tower_oracle.forward_bf16_eager`` with the dtype as a parameter: tensors of
``dtype`` between ops, so every linear output, residual add and the embedding sum round to it; LayerNorm and softmax compute inside in
fp32 (as torch does for 16-bit inputs); attention through SDPA.  At bf16 it gives ``forward_bf16_eager``'s bits (tested);
``forward_f16_eager`` is it at fp16.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.clip_tower_oracle import HIDDEN, PATCH, _attention, layer_keys, quick_gelu


def forward_eager(w, images, n_layers: int, dtype):
    """hidden_states[0 .. n_layers] of transformers' tower with parameters and activations in ``dtype``"""
    W = {k: v.to(dtype) for k, v in w.items()}
    x = images.to(dtype)
    n = x.shape[0]
    patches = F.conv2d(x, W["embeddings.patch_embedding.weight"], stride=PATCH).flatten(2).transpose(1, 2)
    cls = W["embeddings.class_embedding"].expand(n, 1, HIDDEN)
    emb = torch.cat([cls, patches], dim=1) + W["embeddings.position_embedding.weight"]
    h = F.layer_norm(emb, (HIDDEN,), W["pre_layrnorm.weight"], W["pre_layrnorm.bias"], 1e-5)
    out = [h]
    for i in range(n_layers):
        k = {a: W[b] for a, b in layer_keys(i).items()}
        y = F.layer_norm(h, (HIDDEN,), k["layer_norm1.weight"], k["layer_norm1.bias"], 1e-5)
        a = _attention(y, k["self_attn.q_proj.weight"], k["self_attn.q_proj.bias"], k["self_attn.k_proj.weight"], k["self_attn.k_proj.bias"],
                       k["self_attn.v_proj.weight"], k["self_attn.v_proj.bias"], sdpa=True)
        h = h + F.linear(a, k["self_attn.out_proj.weight"], k["self_attn.out_proj.bias"])
        y = F.layer_norm(h, (HIDDEN,), k["layer_norm2.weight"], k["layer_norm2.bias"], 1e-5)
        h = h + F.linear(quick_gelu(F.linear(y, k["mlp.fc1.weight"], k["mlp.fc1.bias"])), k["mlp.fc2.weight"], k["mlp.fc2.bias"])
        out.append(h)
    return out


def forward_f16_eager(w, images, n_layers: int = 23):
    """transformers' fp16 tower: the images cast to fp16, then every op in fp16 as in ``forward_eager``"""
    return forward_eager(w, images, n_layers, torch.float16)
