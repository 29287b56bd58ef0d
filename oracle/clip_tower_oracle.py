"""The CLIP-ViT-L/14-336 vision tower restated with torch ops, independent of transformers.

transformers' CLIPVisionTransformer (unchanged since 4.31):
    emb = cat(class_embedding, conv14x14/14(pixels), no bias) + position_embedding          [N, 577, 1024]
    hidden_states[0] = pre_layrnorm(emb)
    layer i: x = x + out_proj(attn(layer_norm1(x)));  x = x + fc2(quick_gelu(fc1(layer_norm2(x))));  hidden_states[i + 1] = x
    attention: 16 heads of 64, scale 1/8, no mask;  quick_gelu(x) = x sigmoid(1.702 x);  LayerNorm eps 1e-5

``forward`` computes it in one dtype (fp32 / fp64) throughout.  ``forward_bf16_eager`` is the same network in bf16 with the
rounding points of transformers' bf16 tower (every linear output, every residual add, the embedding sum; SDPA attention): the
yardstick the GPU tests and the benchmark measure the sm_90a kernels against.  ``make_weights`` draws seeded parameters at the real
shapes, keyed by transformers' names (without the ``vision_model.`` prefix); ``outlier=True`` drives a few residual channels to
+-50..100 through large fc2 / out_proj biases, the way the released CLIP-L's residual stream has a few huge channels.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

HIDDEN, INTER, HEADS, HEAD_DIM, PATCH, IMAGE, TOKENS = 1024, 4096, 16, 64, 14, 336, 577
OUT_LAYERS = (12, 16, 22, 23)
OUTLIER_CHANNELS = (7, 300, 611, 1000)


def layer_keys(i):
    p = f"encoder.layers.{i}."
    return {k: p + k for k in ("layer_norm1.weight", "layer_norm1.bias", "self_attn.q_proj.weight", "self_attn.q_proj.bias",
                               "self_attn.k_proj.weight", "self_attn.k_proj.bias", "self_attn.v_proj.weight", "self_attn.v_proj.bias",
                               "self_attn.out_proj.weight", "self_attn.out_proj.bias", "layer_norm2.weight", "layer_norm2.bias",
                               "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias")}


def make_weights(n_layers: int = 23, seed: int = 0, outlier: bool = False, device="cpu"):
    """Seeded fp32 parameters: weights N(0, 0.02), biases N(0, 0.02), LayerNorm gamma 1 + N(0, 0.1), beta N(0, 0.05),
    embeddings N(0, 0.5) (the patch weight N(0, 0.02))."""
    g = torch.Generator(device=device).manual_seed(seed)

    def rn(*shape, std=0.02, mean=0.0):
        return torch.randn(*shape, generator=g, device=device) * std + mean

    w = {"embeddings.class_embedding": rn(HIDDEN, std=0.5), "embeddings.patch_embedding.weight": rn(HIDDEN, 3, PATCH, PATCH),
         "embeddings.position_embedding.weight": rn(TOKENS, HIDDEN, std=0.5),
         "pre_layrnorm.weight": rn(HIDDEN, std=0.1, mean=1.0), "pre_layrnorm.bias": rn(HIDDEN, std=0.05)}
    for i in range(n_layers):
        k = layer_keys(i)
        for name in ("layer_norm1", "layer_norm2"):
            w[k[name + ".weight"]] = rn(HIDDEN, std=0.1, mean=1.0)
            w[k[name + ".bias"]] = rn(HIDDEN, std=0.05)
        for name in ("q_proj", "k_proj", "v_proj", "out_proj"):
            w[k[f"self_attn.{name}.weight"]] = rn(HIDDEN, HIDDEN)
            w[k[f"self_attn.{name}.bias"]] = rn(HIDDEN)
        w[k["mlp.fc1.weight"]], w[k["mlp.fc1.bias"]] = rn(INTER, HIDDEN), rn(INTER)
        w[k["mlp.fc2.weight"]], w[k["mlp.fc2.bias"]] = rn(HIDDEN, INTER), rn(HIDDEN)
    if outlier:
        # layer 0's fc2 bias lifts four residual channels to +-50..90; every later out_proj nudges them by +-2 more
        big = torch.tensor([70.0, -60.0, 90.0, -50.0], device=device)
        ch = torch.tensor(OUTLIER_CHANNELS, device=device)
        w[layer_keys(0)["mlp.fc2.bias"]][ch] += big
        for i in range(1, n_layers):
            w[layer_keys(i)["self_attn.out_proj.bias"]][ch] += torch.sign(big) * 2.0
    return w


def make_images(n: int, seed: int = 1, device="cpu"):
    """CLIP-normalised-looking crops: N(0, 1) clipped to [-2, 2.2]."""
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(n, 3, IMAGE, IMAGE, generator=g, device=device).clamp(-2.0, 2.2)


def round_bf16(w):
    return {k: v.to(torch.bfloat16).float() for k, v in w.items()}


def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


def _attention(x, q_w, q_b, k_w, k_b, v_w, v_b, sdpa: bool):
    n = x.shape[0]
    q = F.linear(x, q_w, q_b)
    k = F.linear(x, k_w, k_b)
    v = F.linear(x, v_w, v_b)
    sh = lambda t: t.view(n, TOKENS, HEADS, HEAD_DIM).transpose(1, 2)
    q, k, v = sh(q), sh(k), sh(v)
    if sdpa:
        o = F.scaled_dot_product_attention(q, k, v, scale=HEAD_DIM ** -0.5)
    else:
        p = torch.softmax((q * HEAD_DIM ** -0.5) @ k.transpose(-1, -2), dim=-1)
        o = p @ v
    return o.transpose(1, 2).reshape(n, TOKENS, HIDDEN)


def forward(w, images, n_layers: int = 23, dtype=torch.float64):
    """hidden_states[0 .. n_layers], every op in ``dtype``."""
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
                       k["self_attn.v_proj.weight"], k["self_attn.v_proj.bias"], sdpa=False)
        h = h + F.linear(a, k["self_attn.out_proj.weight"], k["self_attn.out_proj.bias"])
        y = F.layer_norm(h, (HIDDEN,), k["layer_norm2.weight"], k["layer_norm2.bias"], 1e-5)
        h = h + F.linear(quick_gelu(F.linear(y, k["mlp.fc1.weight"], k["mlp.fc1.bias"])), k["mlp.fc2.weight"], k["mlp.fc2.bias"])
        out.append(h)
    return out


def forward_bf16_eager(w, images, n_layers: int = 23):
    """transformers' bf16 tower: bf16 tensors between ops, so every linear output, residual add and the embedding sum round to bf16;
    LayerNorm and softmax compute inside in fp32 (as torch does for bf16 inputs); attention through SDPA."""
    W = {k: v.to(torch.bfloat16) for k, v in w.items()}
    x = images.to(torch.bfloat16)
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


class FakeCLIPVisionModel(torch.nn.Module):
    """Parameters under CLIPVisionModel's names (``vision_model.`` prefix) and a config object: what CLIPVisionTowerB200 wraps, without
    transformers."""

    class Config:
        hidden_size, intermediate_size, num_attention_heads, num_hidden_layers = HIDDEN, INTER, HEADS, 24
        patch_size, image_size, hidden_act, layer_norm_eps, num_channels = PATCH, IMAGE, "quick_gelu", 1e-5, 3

    def __init__(self, w):
        super().__init__()
        self.config = self.Config()
        self.params = torch.nn.ParameterDict({k.replace(".", "__"): torch.nn.Parameter(v, requires_grad=False) for k, v in w.items()})

    def named_parameters(self, *args, **kwargs):
        for k, v in self.params.items():
            yield "vision_model." + k.replace("__", "."), v
