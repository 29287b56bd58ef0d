"""Executable statement of the DEVICE numerics plan (DESIGN.md §3-4) in numpy, on the CPU: the re-associations the CUDA path
makes — k/v first layers as one GEMM, LayerNorm folded into the following linear with statistics taken from the ROUNDED
activations, 1/sqrt(128) applied in the in-projection epilogue, out_proj folded into mlp.0 — with a bf16 rounding at every point
where the device stores bf16 and float32 arithmetic in between.  Held to the float64 oracle at the same gates the GPU parity
tests use (rel-RMS <= 3e-3, max-abs <= 5e-3): the algebra and the rounding plan meet the tolerance by construction, whatever
the kernels do.  (The kernels themselves are held to the oracle on the GPU: tests/test_projector_gpu.py.)"""
import numpy as np
import pytest

from oracle import tokenpacker_oracle as tpo

f32 = np.float32
bf = tpo.round_bf16


def _lin(x, w, b=None):
    y = x.astype(f32) @ w.astype(f32).T
    return y if b is None else y + b.astype(f32)


def _gelu32(x):
    return tpo.gelu_erf(x.astype(np.float64)).astype(f32)


def _fold(w, b, gamma, beta):
    """fold_layernorm_kernel: W' = bf16(W * gamma); wsum = row sums of the ROUNDED W'; c = W . beta + b (float32)."""
    wf = bf(w.astype(f32) * gamma.astype(f32)[None, :])
    return wf, wf.astype(f32).sum(axis=1), (w.astype(f32) @ beta.astype(f32) + b.astype(f32))


def _ln_folded_linear(y, wf, wsum, c, alpha=1.0):
    """Epilogue of GEMM [3]: statistics of the rounded y; v = fma(rstd, acc - mu * wsum, c); then alpha; then bf16."""
    y32 = y.astype(f32)
    mu = y32.sum(axis=1) / f32(1024)
    var = np.maximum((y32 * y32).sum(axis=1) / f32(1024) - mu * mu, 0)
    rstd = (1.0 / np.sqrt(var + f32(1e-6))).astype(f32)
    acc = y32 @ wf.astype(f32).T
    v = rstd[:, None] * (acc - mu[:, None] * wsum[None, :]) + c[None, :]
    return bf((f32(alpha) * v).astype(f32))


def device_plan_forward(p, x0, xm, s):
    n = x0.shape[0]
    g = 24 // s
    q = bf(tpo.point_queries(x0.astype(f32), s).astype(f32)).reshape(n * g * g, 1024)                    # [S]
    wkv0 = np.concatenate([p["k_proj_1.0.weight"], p["v_proj_1.0.weight"]], 0)
    bkv0 = np.concatenate([p["k_proj_1.0.bias"], p["v_proj_1.0.bias"]], 0)
    h_kv = bf(_gelu32(_lin(xm.reshape(-1, 4096), wkv0, bkv0)))                                           # [1]
    y_k = bf(_lin(h_kv[:, :1024], p["k_proj_1.2.weight"], p["k_proj_1.2.bias"]))                         # [2]
    y_v = bf(_lin(h_kv[:, 1024:], p["v_proj_1.2.weight"], p["v_proj_1.2.bias"]))
    y_q = bf(_lin(q, p["q_proj_1.weight"]))
    in_w, in_b = p["clip_attn.in_proj_weight"], p["clip_attn.in_proj_bias"]
    qp = _ln_folded_linear(y_q, *_fold(in_w[:1024], in_b[:1024], p["ln_q_1.weight"], p["ln_q_1.bias"]), alpha=128 ** -0.5)   # [3]
    kp = _ln_folded_linear(y_k, *_fold(in_w[1024:2048], in_b[1024:2048], p["ln_k_1.weight"], p["ln_k_1.bias"]))
    vp = _ln_folded_linear(y_v, *_fold(in_w[2048:], in_b[2048:], p["ln_v_1.weight"], p["ln_v_1.bias"]))
    # [A] window attention by address arithmetic: query (n, hb, wb) attends to fine tokens (hb*s+hi, wb*s+wi), 8 heads x 128
    kp = kp.reshape(n, g, s, g, s, 8, 128).transpose(0, 1, 3, 5, 2, 4, 6).reshape(n * g * g, 8, s * s, 128).astype(f32)
    vp = vp.reshape(n, g, s, g, s, 8, 128).transpose(0, 1, 3, 5, 2, 4, 6).reshape(n * g * g, 8, s * s, 128).astype(f32)
    sc = np.einsum("qhd,qhjd->qhj", qp.reshape(-1, 8, 128).astype(f32), kp)
    pr = np.exp(sc - sc.max(axis=-1, keepdims=True))
    pr /= pr.sum(axis=-1, keepdims=True)
    ctx = bf(np.einsum("qhj,qhjd->qhd", pr, vp).reshape(-1, 1024).astype(f32))
    w_om = bf(p["mlp.0.weight"].astype(f32) @ p["clip_attn.out_proj.weight"].astype(f32))               # pack time: one GEMM
    b_om = p["mlp.0.weight"].astype(f32) @ p["clip_attn.out_proj.bias"].astype(f32) + p["mlp.0.bias"].astype(f32)
    h_m = bf(_gelu32(_lin(ctx, w_om, b_om)))                                                              # [4]
    out = bf(_lin(h_m, p["mlp.2.weight"], p["mlp.2.bias"]))                                               # [5]
    return out.reshape(n, g * g, -1)


def _stencil_f32(a, b, c, d):
    """point_query_kernel's even-s sequence in float32 (numpy rounds every operation, no FMA): (0.25a + 0.25b) + (0.25c + 0.25d)"""
    q = f32(0.25)
    return (q * a + q * b) + (q * c + q * d)


def _bf16_bits(rng, shape):
    """random finite bf16 values over every binade, both signs, subnormals and zeros included"""
    bits = rng.integers(0, 1 << 16, size=shape, dtype=np.uint32)
    bits = np.where((bits & 0x7F80) == 0x7F80, bits & 0x807F, bits)        # inf / nan -> a subnormal of the same sign
    return (bits << 16).view(np.float32)


@pytest.mark.parametrize("s", [2, 4])
def test_point_query_stencil_matches_interpolate_bits(s):
    """The even-s stencil against torch's bilinear F.interpolate (the reference, builder.py:117-118): bit for bit, before and after
    the bf16 rounding, on windows of subnormal taps and windows whose taps lie in bf16's top binade (|x| >= 2^127) with equal and
    mixed signs; within two fp32 roundings on random bf16 taps from every binade.  Adding the taps before scaling them,
    0.25 ((a + b) + (c + d)), overflows to inf on the top-binade windows and gives the same bits everywhere else: checked too, so
    the inputs really reach the range the sequence is for."""
    import torch
    import torch.nn.functional as F
    g, c = 24 // s, 64
    rng = np.random.default_rng(7 + s)
    img = _bf16_bits(rng, (c, 24, 24))
    lo = s // 2 - 1                                              # first centre tap of a window
    top = (rng.integers(0x7F00, 0x7F80, size=(c, 4), dtype=np.uint32) << 16).view(np.float32)     # [2^127, max bf16]
    signs = np.array([[1, 1, 1, 1], [-1, -1, -1, -1], [1, -1, 1, -1], [1, 1, -1, 1]], dtype=np.float32)
    sub = _bf16_bits(rng, (c, 4)).view(np.uint32) & np.uint32(0x807F0000)                          # subnormals and zeros
    special = {(0, 0): top * signs[0], (0, 1): top * signs[1], (1, 0): top * signs[2], (1, 1): top * signs[3],
               (2, 2): sub.view(np.float32), (g - 1, g - 1): np.full((c, 4), 2.0 ** 127, dtype=np.float32)}
    for (hb, wb), taps in special.items():
        r, cc = hb * s + lo, wb * s + lo
        img[:, r, cc], img[:, r, cc + 1], img[:, r + 1, cc], img[:, r + 1, cc + 1] = taps.T
    ref = F.interpolate(torch.from_numpy(img)[None], size=(g, g), mode="bilinear", align_corners=False)[0].numpy()
    i = np.arange(g) * s + lo
    a, b = img[:, i][:, :, i], img[:, i][:, :, i + 1]
    cq, d = img[:, i + 1][:, :, i], img[:, i + 1][:, :, i + 1]
    got = _stencil_f32(a, b, cq, d)
    assert np.isfinite(got).all()
    for hb, wb in special:
        assert np.array_equal(got[:, hb, wb].view(np.uint32), ref[:, hb, wb].view(np.uint32)), (hb, wb)
        assert np.array_equal(bf(got[:, hb, wb]).view(np.uint32), bf(ref[:, hb, wb]).view(np.uint32)), (hb, wb)
    # elsewhere the taps span many binades, the fp32 sums round, and ATen adds in another order: both are within two roundings
    mag = sum(np.abs(t.astype(np.float64)) for t in (a, b, cq, d)) * 0.25
    assert (np.abs(got.astype(np.float64) - ref) <= 4 * 2.0 ** -24 * mag).all()
    with np.errstate(over="ignore"):
        old = f32(0.25) * ((a + b) + (cq + d))
    assert np.isinf(old[:, 0, 0]).all() and np.isinf(old[:, g - 1, g - 1]).all()
    fin = np.isfinite(old)                                       # elsewhere the two sequences give the same bits
    assert np.array_equal(old[fin].view(np.uint32), got[fin].view(np.uint32))


@pytest.mark.parametrize("s", [2, 3, 4, 6])
def test_device_plan_meets_the_gpu_gates(s):
    hidden, n = 128, 2
    params = {k: bf(v) for k, v in tpo.make_params(hidden, seed=300 + s).items()}
    x0, xm = tpo.make_inputs(n, seed=400 + s)
    x0, xm = bf(x0), bf(xm)
    ref = tpo.tokenpacker_forward(params, x0, xm, s)
    out = device_plan_forward(params, x0, xm, s).astype(np.float64)
    rel = float(np.sqrt(((out - ref) ** 2).mean()) / np.sqrt((ref ** 2).mean()))
    mx = float(np.abs(out - ref).max())
    assert rel <= 3e-3 and mx <= 5e-3, (rel, mx)
    assert rel >= 2e-4          # sanity: the model really rounds to bf16 (a pure-fp32 pipeline would sit at ~1e-6)
