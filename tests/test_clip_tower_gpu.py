"""The CLIP vision tower on the H100: the engine's residual / quick_gelu epilogue on its own, the attention kernel against fp64, and
the whole 23-layer tower against the fp64 oracle, gated by the error transformers' bf16 tower (the oracle's bf16 eager restatement)
makes on the same inputs.  Plus the bitwise properties: batch invariance, run-to-run determinism, strided crops."""
import ctypes as C
import os

import pytest
import torch

from oracle import clip_tower_oracle as cto

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_clip_tower_hooks.so")
DEV = "cuda:0"


@pytest.fixture(scope="module")
def hooks():
    lib = C.CDLL(HOOKS)
    lib.tpc_gemm.restype = C.c_int
    lib.tpc_gemm.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                             C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p]
    lib.tpc_workspace_offsets.restype = C.c_int
    lib.tpc_workspace_offsets.argtypes = [C.c_int64, C.POINTER(C.c_int64)]
    lib.tpc_layer.restype = C.c_int
    lib.tpc_layer.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.tpc_attention.restype = C.c_int
    lib.tpc_attention.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


def _ptr(t):
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------------------------------------
# epilogue additions
# ------------------------------------------------------------------------------------------------------------------------------
E, U = 2.0 ** -24, 2.0 ** -8          # fp32 and bf16 unit roundoff
QG_LIP = 1.13                         # max |quick_gelu'(z)| = 1.0998 (below GELU's 1.1289)


def _gemm_bound(a, b, bias=None, resid=None, gelu=0, out_bf16=True):
    """(reference, elementwise bound) of bf16(epilogue(a . b^T)) from the bf16 operands in fp64: the fp32 accumulation is off by
    <= (K + 1) E sum_k |a b|, the bias and residual adds by one rounding each (2 E |v|), quick_gelu carries that error with slope <= 1.13
    and adds its own <= (|t| / 16 + 8) 2^-23 relative (tp_ptx.cuh, t = 2.4555 v); the stored result one bf16 rounding (U |ref|) unless
    it is stored in fp32."""
    a, b = a.double(), b.double()
    v = a @ b.T
    floor = (a.shape[1] + 1) * E * (a.abs() @ b.abs().T)
    if bias is not None:
        v = v + bias.double()
    if resid is not None:
        v = v + resid.double()
    floor = floor + 2 * E * v.abs()
    if gelu == 2:
        ref = v * torch.sigmoid(1.702 * v)
        floor = QG_LIP * floor + ref.abs() * (2.46 * v.abs() / 16 + 8) * 2.0 ** -23
    else:
        ref = v
    if not out_bf16:
        return ref, floor + 1e-30
    return ref, U * ref.abs() + (1 + U) * floor + 1e-30


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    assert torch.isfinite(got.double()).all(), what
    assert (err <= bound).all(), (what, float((err / bound).max()))


@pytest.mark.parametrize("bias,resid,gelu", [(True, True, 0), (False, True, 0), (True, False, 2), (False, False, 2)])
def test_residual_and_quick_gelu_epilogue(hooks, bias, resid, gelu):
    g = torch.Generator(device=DEV).manual_seed(3)
    M, N, K = 577 * 3, 1024, 1024                          # ragged: 1731 rows are no multiple of 128 or 256
    a = (torch.randn(M, K, generator=g, device=DEV)).bfloat16()
    b = (torch.randn(N, K, generator=g, device=DEV) * 0.05).bfloat16()
    bv = torch.randn(N, generator=g, device=DEV) if bias else None
    r = (torch.randn(M, N, generator=g, device=DEV) * 4).bfloat16() if resid else None
    outs = []
    for mode in (1, 2):                                    # one-CTA 128 x 256 tiles, then the pair kernel
        frame = torch.full((M + 4, N + 64), float("nan"), device=DEV).bfloat16()   # guard rows / columns stay NaN
        c = frame[2:M + 2, :N]
        assert hooks.tpc_gemm(_ptr(a), K, _ptr(b), K, _ptr(c), N + 64, M, N, K, _ptr(bv), _ptr(r), N, gelu, mode, None) == 0
        torch.cuda.synchronize()
        assert torch.isnan(frame[:2].float()).all() and torch.isnan(frame[M + 2:].float()).all() and torch.isnan(frame[:, N:].float()).all()
        outs.append(c.clone())
    assert torch.equal(outs[0], outs[1]), "one-CTA and pair kernels differ"
    ref, bound = _gemm_bound(a, b, bv, r, gelu)
    _check(outs[0], ref, bound, "epilogue")


# ------------------------------------------------------------------------------------------------------------------------------
# attention kernel
# ------------------------------------------------------------------------------------------------------------------------------
def _attention_ref(qkv, n):
    x = qkv[: n * 577].double().view(n, 577, 3, 16, 64)
    q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)
    p = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
    return (p @ v).transpose(1, 2).reshape(n * 577, 1024), v


def test_attention_against_fp64(hooks):
    g = torch.Generator(device=DEV).manual_seed(5)
    n = 3
    qkv = torch.randn(n * 577 + 64, 3072, generator=g, device=DEV)
    x = qkv[: n * 577].view(n, 577, 3, 16, 64)
    x[0, :, 0, 1] *= 6.0                                   # head 1 of crop 0: saturated logits (scores in the hundreds)
    x[0, :, 0, 2] = 0.0                                    # head 2: all-equal logits -> the mean of v
    x[0, :, 1, 3] *= 0.01                                  # head 3: one dominant key
    x[0, 123, 1, 3] = 40.0
    x[1] *= 0.3
    x[1, :, 0, 4] = 0.0                                    # head 4 of crop 1: all-equal logits and v = 1: the result is exactly 1.  The 63
    x[1, :, 2, 4] = 1.0                                    # zero-filled keys 577..639 would score 0 too: unmasked they take 63/640 of the
                                                           # weight and give 577/640 = 0.90, 5x the bound below
    x[2, :, 2] *= 1e3                                      # crop 2's values are huge: crop 1's padded keys read zeros, never these rows
    qkv[n * 577:] = 3e4                                    # rows after the last crop (outside the map's crop extent: never read)
    qkv = qkv.bfloat16()
    ctx = torch.full((n * 577 + 8, 1024), float("nan"), device=DEV).bfloat16()
    assert hooks.tpc_attention(_ptr(qkv), _ptr(ctx), n, None) == 0
    torch.cuda.synchronize()
    assert torch.isnan(ctx[n * 577:].float()).all()
    ref, v = _attention_ref(qkv, n)
    out = ctx[: n * 577].double()
    # P is rounded to bf16 (2^-8) before P V and the row sum, ex2.approx adds 2^-22: each weight is off by d <= 2^-8 (1 + 2^-13)
    # relative, so the normalised sum is off by <= 2 d / (1 - d) max|v - o| <= 2^-6 max|v| of its (crop, head); the stored result adds
    # one rounding (2^-8 relative)
    vmax = v.abs().amax(dim=(2, 3))                                         # [n, 16]
    vmax = vmax[:, None, :, None].expand(n, 577, 16, 64).reshape(n * 577, 1024)
    bound = 2.0 ** -6 * vmax + 2.0 ** -8 * ref.abs() + 1e-30
    err = (out - ref).abs()
    assert (err <= bound).all(), float((err / bound).max())
    assert (out.view(n, 577, 16, 64)[1, :, 4] == 1.0).all()


# ------------------------------------------------------------------------------------------------------------------------------
# the whole tower
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[False, True], ids=["standard", "outlier"])
def tower(request):
    from tokenpacker_b200 import CLIPVisionTowerB200
    w = cto.round_bf16(cto.make_weights(23, seed=11, outlier=request.param, device=DEV))
    model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    return w, CLIPVisionTowerB200(model)


def _errors(got, ref):
    d = got.double() - ref
    return float(d.norm() / ref.norm()), float(d.abs().max())


@pytest.mark.parametrize("n", [1, 5])
def test_tower_against_oracle(tower, n):
    w, t = tower
    images = cto.make_images(n, seed=n, device=DEV).bfloat16()
    with torch.no_grad():
        ours = t.hidden_states(images)
        ref = cto.forward(w, images.double(), 23, torch.float64)
        hf = cto.forward_bf16_eager(w, images, 23)
    torch.cuda.synchronize()
    for got, layer in zip(ours, cto.OUT_LAYERS):
        assert got.shape == (n, 577, 1024) and got.dtype == torch.bfloat16
        rms, mx = _errors(got, ref[layer])
        rms_hf, mx_hf = _errors(hf[layer], ref[layer])
        # the gate is transformers' own bf16 tower on the same inputs (one rounding per stored tensor here, against its rounding of every
        # linear output and residual add): neither the rel-RMS nor the largest error may exceed its own
        assert rms <= rms_hf, (layer, rms, rms_hf)
        assert mx <= mx_hf, (layer, mx, mx_hf)


def test_batch_invariance_determinism_and_strided_crops(tower):
    _, t = tower
    images = cto.make_images(4, seed=9, device=DEV).bfloat16()
    with torch.no_grad():
        full = t.hidden_states(images)
        again = t.hidden_states(images)
        single = t.hidden_states(images[2:3])
        big = torch.full((4, 3 * 336 * 336 + 4096), float("nan"), device=DEV).bfloat16()
        strided = big[:, :3 * 336 * 336].view(4, 3, 336, 336)
        strided.copy_(images)
        from_strided = t.hidden_states(strided)
    torch.cuda.synchronize()
    for a, b, s, c in zip(full, again, single, from_strided):
        assert torch.equal(a, b)
        assert torch.equal(a[2:3], s)
        assert torch.equal(a, c)
        assert torch.isfinite(a.float()).all()


def test_refuses_gradients_and_cpu(tower):
    _, t = tower
    x = torch.zeros(1, 3, 336, 336, device=DEV, requires_grad=True)
    with pytest.raises(NotImplementedError, match="forward only"):
        t.hidden_states(x)
    with pytest.raises(RuntimeError, match="no CPU path"):
        with torch.no_grad():
            t.hidden_states(torch.zeros(1, 3, 336, 336))


# ------------------------------------------------------------------------------------------------------------------------------
# one layer, stage by stage
# ------------------------------------------------------------------------------------------------------------------------------
def _ln_ref(x, gamma, beta):
    """(reference, bound) of bf16(LayerNorm(x) gamma + beta) in fp32 from bf16 x.  The mean is an fp32 sum of 1024 terms: off by
    <= 1025 E mean|x| (absolute); the variance a sum of 1024 squares: <= 1026 E relative, so rstd (with rsqrt's 2^-22) is off by
    <= 2^-12 relative, as is the normalised value; the affine step and the bf16 rounding of the result follow."""
    x = x.double()
    g = gamma.double()
    mu = x.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
    xh = (x - mu) * rstd
    ref = xh * g + beta.double()
    floor = g.abs() * (2.0 ** -12 * xh.abs() + rstd * 1025 * E * x.abs().mean(-1, keepdim=True)) + 2 * E * ref.abs()
    return ref, U * ref.abs() + (1 + U) * floor + 1e-30


def test_one_layer_stage_by_stage(hooks, tower):
    """Layer 1 alone (its input, hidden_states[1], carries the outlier channels in the outlier variant) on a workspace poisoned with
    NaN: every stage against fp64 of that stage computed from the bf16 values the kernels stored before it."""
    w, t = tower
    n = 2
    images = cto.make_images(n, seed=21, device=DEV).bfloat16()
    with torch.no_grad():
        x = cto.forward(w, images.float(), 1, torch.float64)[1].bfloat16().reshape(n * 577, 1024).contiguous()
        packed, (cw, _) = t._packed_weights(torch.device(DEV))
    offs = (C.c_int64 * 7)()
    assert hooks.tpc_workspace_offsets(n, offs) == 0
    ws = torch.full((offs[6],), 0xFF, dtype=torch.uint8, device=DEV)        # bf16 0xFFFF: NaN everywhere
    out = torch.full((n * 577, 1024), float("nan"), device=DEV).bfloat16()
    assert hooks.tpc_layer(packed.data_ptr(), C.addressof(cw), 1, x.data_ptr(), out.data_ptr(), n, ws.data_ptr(), offs[6], None) == 0
    torch.cuda.synchronize()
    M = n * 577

    def region(i, cols, dtype=torch.bfloat16):
        size = 4 if dtype == torch.float32 else 2
        return ws[offs[i]: offs[i] + M * cols * size].view(dtype).view(M, cols)

    y1, qkv, ctx, y2, h = region(0, 1024), region(1, 3072), region(2, 1024), region(4, 1024), region(5, 4096)
    xp = region(3, 1024, torch.float32)                                       # the mid-layer residual stays unrounded
    k = {a: w[b].to(DEV) for a, b in cto.layer_keys(1).items()}
    bf = lambda v: v.bfloat16()
    ref, bound = _ln_ref(x, bf(k["layer_norm1.weight"]), bf(k["layer_norm1.bias"]))
    _check(y1, ref, bound, "y1 = layer_norm1(x)")
    wq = torch.cat([k["self_attn.q_proj.weight"] / 8, k["self_attn.k_proj.weight"], k["self_attn.v_proj.weight"]])
    bq = torch.cat([k["self_attn.q_proj.bias"] / 8, k["self_attn.k_proj.bias"], k["self_attn.v_proj.bias"]])
    ref, bound = _gemm_bound(y1, bf(wq), bf(bq).float())
    _check(qkv, ref, bound, "qkv")
    ref, v = _attention_ref(qkv, n)
    vmax = v.abs().amax(dim=(2, 3))[:, None, :, None].expand(n, 577, 16, 64).reshape(M, 1024)
    _check(ctx, ref, 2.0 ** -6 * vmax + U * ref.abs() + 1e-30, "ctx")
    ref, bound = _gemm_bound(ctx, bf(k["self_attn.out_proj.weight"]), bf(k["self_attn.out_proj.bias"]).float(), x, out_bf16=False)
    _check(xp, ref, bound, "x' = x + out_proj(ctx)")
    ref, bound = _ln_ref(xp, bf(k["layer_norm2.weight"]), bf(k["layer_norm2.bias"]))
    _check(y2, ref, bound, "y2 = layer_norm2(x')")
    ref, bound = _gemm_bound(y2, bf(k["mlp.fc1.weight"]), bf(k["mlp.fc1.bias"]).float(), None, 2)
    _check(h, ref, bound, "h = quick_gelu(fc1(y2))")
    ref, bound = _gemm_bound(h, bf(k["mlp.fc2.weight"]), bf(k["mlp.fc2.bias"]).float(), xp)
    _check(out, ref, bound, "x'' = x' + fc2(h)")


# ------------------------------------------------------------------------------------------------------------------------------
# end to end: decoded images -> HD crops -> tower -> projector
# ------------------------------------------------------------------------------------------------------------------------------
def test_uint8_images_to_packed_projector_output(tower):
    from tokenpacker_b200 import TokenPackerB200, hd_preprocess_batch
    w, t = tower
    g = torch.Generator(device=DEV).manual_seed(31)
    images = [torch.randint(0, 256, (h_, w_, 3), generator=g, device=DEV, dtype=torch.uint8) for h_, w_ in ((336, 336), (500, 700))]
    torch.manual_seed(7)
    proj = TokenPackerB200(hidden_size=1024, scale_factor=2).to(DEV, torch.bfloat16).eval()
    sep = torch.randn(1024, device=DEV).bfloat16()
    ret = torch.randn(1024, device=DEV).bfloat16()
    with torch.no_grad():
        crops, hb, wb = hd_preprocess_batch(images, patch_num=9, dtype=torch.bfloat16)
        ours = t.hidden_states(crops)                                     # the preprocessing output, read in place
        copy = t.hidden_states(crops.clone())
        for a, b in zip(ours, copy):
            assert torch.equal(a, b)
        ref_hs = cto.forward(w, crops.double(), 23, torch.float64)
        eager_hs = cto.forward_bf16_eager(w, crops, 23)
        run = lambda hs: proj.forward_hidden_states_packed(list(hs), hb, wb, sep, ret)[0].double()
        out = run(ours)
        ref = run([ref_hs[i].bfloat16() for i in cto.OUT_LAYERS])
        eager = run([eager_hs[i] for i in cto.OUT_LAYERS])
    torch.cuda.synchronize()
    # the same projector on both sides: what differs is the tower.  Ours must not be further from the fp64 tower's result than
    # transformers' bf16 tower is (rel-RMS and largest error).
    rms, mx = _errors(out, ref)
    rms_e, mx_e = _errors(eager, ref)
    assert torch.isfinite(out).all()
    assert rms <= rms_e and mx <= mx_e, (rms, rms_e, mx, mx_e)
