"""The CLIP tower's last K encoder layers under torch autograd, independent of transformers: the yardstick of the training path
(include/tokenpacker_b200_clip_tower_train.h).

``layer`` is one encoder layer written out with explicit tensor ops (so that it runs in any dtype on any device, and so that it is a
second statement of clip_tower_oracle.forward's layer, against which tests/test_clip_tower_train_host.py checks it);
``hidden_states`` runs layers ``first .. 22`` from hidden_states[first] and returns hidden states 12 / 16 / 22 / 23 (None for those
below ``first``); ``parameter_gradients`` is the whole training step of the tests: the frozen bottom without a graph, the trainable top
with one, a weighted-sum loss over the four hidden states, autograd.
"""
from __future__ import annotations

import torch

from oracle import clip_tower_oracle as cto

PARAM_KEYS = ("layer_norm1.weight", "layer_norm1.bias", "self_attn.q_proj.weight", "self_attn.q_proj.bias", "self_attn.k_proj.weight",
              "self_attn.k_proj.bias", "self_attn.v_proj.weight", "self_attn.v_proj.bias", "self_attn.out_proj.weight",
              "self_attn.out_proj.bias", "layer_norm2.weight", "layer_norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight",
              "mlp.fc2.bias")


def _layer_norm(x, gamma, beta):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-5) * gamma + beta


def layer(p, x):
    """p: PARAM_KEYS -> tensor; x [N, 577, 1024] -> the layer's output."""
    n = x.shape[0]
    y = _layer_norm(x, p["layer_norm1.weight"], p["layer_norm1.bias"])
    heads = lambda t: t.view(n, cto.TOKENS, cto.HEADS, cto.HEAD_DIM).transpose(1, 2)
    q = heads(y @ p["self_attn.q_proj.weight"].T + p["self_attn.q_proj.bias"]) * cto.HEAD_DIM ** -0.5
    k = heads(y @ p["self_attn.k_proj.weight"].T + p["self_attn.k_proj.bias"])
    v = heads(y @ p["self_attn.v_proj.weight"].T + p["self_attn.v_proj.bias"])
    a = (torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v).transpose(1, 2).reshape(n, cto.TOKENS, cto.HIDDEN)
    x = x + a @ p["self_attn.out_proj.weight"].T + p["self_attn.out_proj.bias"]
    z = _layer_norm(x, p["layer_norm2.weight"], p["layer_norm2.bias"]) @ p["mlp.fc1.weight"].T + p["mlp.fc1.bias"]
    return x + (z * torch.sigmoid(1.702 * z)) @ p["mlp.fc2.weight"].T + p["mlp.fc2.bias"]


def layer_params(w, i, dtype, device=None):
    keys = cto.layer_keys(i)
    return {k: w[keys[k]].to(device=device, dtype=dtype) for k in PARAM_KEYS}


def hidden_states(params, x, first, n_layers=23):
    """params[i - first]: the parameters of layer i; x = hidden_states[first].  Returns {j: hidden_states[j]} for j in 12 / 16 / 22 / 23
    (those above ``first`` and at most n_layers)."""
    out = {}
    for i in range(first, n_layers):
        x = layer(params[i - first], x)
        if i + 1 in cto.OUT_LAYERS:
            out[i + 1] = x
    return out


def parameter_gradients(w, images, k, d_outs, n_layers=23, dtype=torch.float64, device="cpu"):
    """Gradients of loss = sum_j <d_outs[j], hidden_states[j]> (d_outs: {12 / 16 / 22 / 23: tensor or None}) w.r.t. the parameters of
    the last k of n_layers layers: a list of k dicts PARAM_KEYS -> gradient.  Also returns the hidden states."""
    first = n_layers - k
    with torch.no_grad():
        wd = {key: v.to(device=device, dtype=dtype) for key, v in w.items()}
        below = cto.forward(wd, images.to(device), first, dtype)
    params = [{key: v.clone().requires_grad_(True) for key, v in layer_params(w, i, dtype, device).items()} for i in range(first, n_layers)]
    hs = hidden_states(params, below[first], first, n_layers)
    loss = sum((hs[j] * d_outs[j].to(device=device, dtype=dtype)).sum() for j in hs if d_outs.get(j) is not None)
    loss.backward()
    full = {j: below[j] for j in cto.OUT_LAYERS if j <= first}
    full.update({j: h.detach() for j, h in hs.items()})
    return [{key: p[key].grad for key in PARAM_KEYS} for p in params], full


def parameter_gradients_chunked(w, images, k, d_outs, chunk, n_layers=23, dtype=torch.float64, device="cpu"):
    """parameter_gradients over ``chunk`` crops at a time, summed: the loss is a sum over crops, so this is the same gradient with
    the attention probabilities of ``chunk`` crops alive at once instead of all of them (fp64 P is 21 MB per crop and head)."""
    total = None
    for c0 in range(0, images.shape[0], chunk):
        part = {j: None if d is None else d[c0:c0 + chunk] for j, d in d_outs.items()}
        grads, _ = parameter_gradients(w, images[c0:c0 + chunk], k, part, n_layers, dtype, device)
        total = grads if total is None else [{key: a[key] + b[key] for key in PARAM_KEYS} for a, b in zip(total, grads)]
    return total
