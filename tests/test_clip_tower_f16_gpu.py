"""The fp16 CLIP vision tower on the H100 (CLIPVisionTowerB200(model, dtype=torch.float16), the precision the reference's evaluation
and serving scripts run the tower in): the tile engine's f16 instantiations on their own, the f16 attention kernel and one layer stage
by stage against fp64, and the whole 23-layer tower against the fp64 oracle, gated by the error transformers' fp16 tower (the oracle's
fp16 eager restatement) makes on the same inputs.  Plus the bitwise properties and the whole path into the bf16 projector."""
import ctypes as C
import os

import pytest
import torch

from oracle import clip_tower_f16_oracle as ct16
from oracle import clip_tower_oracle as cto

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_clip_tower_f16_hooks.so")
DEV = "cuda:0"
F16 = torch.float16


@pytest.fixture(scope="module")
def hooks():
    lib = C.CDLL(HOOKS)
    lib.tpc_gemm_f16.restype = C.c_int
    lib.tpc_gemm_f16.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                 C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int,
                                 C.c_void_p]
    lib.tpc_workspace_offsets_f16.restype = C.c_int
    lib.tpc_workspace_offsets_f16.argtypes = [C.c_int64, C.POINTER(C.c_int64)]
    lib.tpc_layer_f16.restype = C.c_int
    lib.tpc_layer_f16.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.tpc_attention_f16.restype = C.c_int
    lib.tpc_attention_f16.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


def _ptr(t):
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------------------------------------
# the engine's f16 instantiations
# ------------------------------------------------------------------------------------------------------------------------------
E, U = 2.0 ** -24, 2.0 ** -11         # fp32 and fp16 unit roundoff
QG_LIP = 1.13                         # max |quick_gelu'(z)| = 1.0998


def _gemm_bound(a, b, bias=None, resid=None, gelu=0, alpha=1.0, out_f16=True):
    """(reference, elementwise bound) of f16(alpha * epilogue(a . b^T)) from the f16 operands in fp64, derived as in
    test_clip_tower_gpu.py: the fp32 accumulation is off by <= (K + 1) E sum_k |a b|, the bias and residual adds by one rounding each
    (2 E |v|), quick_gelu carries that error with slope <= 1.13 and adds its own <= (|t| / 16 + 8) 2^-23 relative; alpha (a power of two)
    is exact; the stored result one f16 rounding (U |ref|) unless it is stored in fp32."""
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
    ref, floor = ref * alpha, floor * abs(alpha)
    if not out_f16:
        return ref, floor + 1e-30
    return ref, U * ref.abs() + (1 + U) * floor + 1e-30


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    assert torch.isfinite(got.double()).all(), what
    assert (err <= bound).all(), (what, float((err / bound).max()))


def _run_gemm(hooks, a, b, M, N, K, bias, r, resid_f32, gelu, out_f32, alpha, mode, seg=None):
    """C in a NaN frame (2 guard rows above and below, 64 guard columns): returns (C, frame)"""
    dt = torch.float32 if out_f32 else F16
    rows = M if seg is None else M // seg[0] * seg[1]
    frame = torch.full((rows + 4, N + 64), float("nan"), device=DEV, dtype=dt)
    c = frame[2:rows + 2, :N]
    ldr = 0 if r is None else r.stride(0)
    seg_len, seg_stride = seg if seg is not None else (0, 0)
    assert hooks.tpc_gemm_f16(_ptr(a), a.stride(0), _ptr(b), b.stride(0), _ptr(c), N + 64, M, N, K, _ptr(bias), _ptr(r), ldr, resid_f32,
                              gelu, out_f32, alpha, seg_len, seg_stride, mode, None) == 0
    torch.cuda.synchronize()
    assert torch.isnan(frame[:2].float()).all() and torch.isnan(frame[rows + 2:].float()).all()
    assert torch.isnan(frame[:, N:].float()).all()
    return c.clone(), frame


@pytest.mark.parametrize("bias,resid,gelu,out_f32,alpha", [
    (True, "f16", 0, 0, 1.0),          # fc2 with an f16 residual
    (True, "f32", 0, 0, 1.0),          # fc2 of the tower: the fp32 mid-layer residual
    (True, "f16", 0, 1, 1.0),          # out_proj: f16 residual, fp32 output
    (False, "f16", 0, 1, 1.0),
    (True, None, 2, 0, 1.0),           # fc1: quick_gelu
    (False, None, 2, 0, 1.0),
    (True, None, 0, 0, 1.0),           # k | v: bias only (a plain item: the f16 instantiations run it all the same)
    (True, None, 0, 0, 0.125),         # q: alpha after the bias, one rounding
], ids=["f16resid", "f32resid", "f16resid-f32out", "nobias-f32out", "gelu", "nobias-gelu", "bias", "bias-alpha"])
def test_f16_epilogue(hooks, bias, resid, gelu, out_f32, alpha):
    g = torch.Generator(device=DEV).manual_seed(3)
    M, N, K = 577 * 3, 1024, 1024                          # ragged: 1731 rows are no multiple of 128 or 256
    a = torch.randn(M, K, generator=g, device=DEV).to(F16)
    b = (torch.randn(N, K, generator=g, device=DEV) * 0.05).to(F16)
    bv = torch.randn(N, generator=g, device=DEV) if bias else None
    r = None
    if resid is not None:
        r = torch.randn(M, N, generator=g, device=DEV) * 4
        r = r if resid == "f32" else r.to(F16)
    outs = [_run_gemm(hooks, a, b, M, N, K, bv, r, int(resid == "f32"), gelu, out_f32, alpha, mode)[0] for mode in (1, 2)]
    assert torch.equal(outs[0], outs[1]), "one-CTA and pair kernels differ"
    ref, bound = _gemm_bound(a, b, bv, r, gelu, alpha, out_f16=not out_f32)
    _check(outs[0], ref, bound, "epilogue")


def test_f16_patch_gemm_segmented_store(hooks):
    """The patch GEMM's uniform-stride store (576 rows per crop, 577 apart: token rows 1..576) on both f16 kernels; the rows between the
    segments (each crop's CLS row) are never written."""
    g = torch.Generator(device=DEV).manual_seed(4)
    n, N, K = 3, 1024, 588
    M = 576 * n
    a = torch.zeros(M, 592, device=DEV, dtype=F16)
    a[:, :K] = torch.randn(M, K, generator=g, device=DEV).to(F16)
    b = torch.zeros(N, 592, device=DEV, dtype=F16)
    b[:, :K] = (torch.randn(N, K, generator=g, device=DEV) * 0.05).to(F16)
    outs = []
    for mode in (1, 2):
        c, frame = _run_gemm(hooks, a[:, :K], b[:, :K], M, N, K, None, None, 0, 0, 0, 1.0, mode, seg=(576, 577))
        sep = c.view(n, 577, N)[:, 576]
        assert torch.isnan(sep.float()).all(), "separator rows written"
        outs.append(c.view(n, 577, N)[:, :576].reshape(M, N))
    assert torch.equal(outs[0], outs[1])
    ref, bound = _gemm_bound(a[:, :K], b[:, :K])
    _check(outs[0], ref, bound, "segmented store")


@pytest.mark.parametrize("mode", [1, 2])
def test_f16_integer_operands_are_exact(hooks, mode):
    """Small integers in A, B, the bias and an f16 residual: every product and partial sum is an integer of at most 2^11, so the fp32
    accumulation and the f16 result are exact.  K = 200 is no multiple of 64 and M = 300 no multiple of 128 or 256: the zero fill TMA
    puts into the ragged tiles of f16 operands through the (bf16-typed) tensor maps adds +0, as it must."""
    g = torch.Generator(device=DEV).manual_seed(6)
    M, N, K = 300, 512, 200
    a = torch.randint(-2, 3, (M, K), generator=g, device=DEV).to(F16)
    b = torch.randint(-2, 3, (N, K), generator=g, device=DEV).to(F16)
    bias = torch.randint(-64, 65, (N,), generator=g, device=DEV).float()
    r = torch.randint(-256, 257, (M, N), generator=g, device=DEV).to(F16)
    c, _ = _run_gemm(hooks, a, b, M, N, K, bias, r, 0, 0, 0, 1.0, mode)
    ref = a.double() @ b.double().T + bias.double() + r.double()
    assert ref.abs().max() <= 2048
    assert torch.equal(c.double(), ref)


# ------------------------------------------------------------------------------------------------------------------------------
# attention kernel
# ------------------------------------------------------------------------------------------------------------------------------
def _attention_ref(qkv, n):
    x = qkv[: n * 577].double().view(n, 577, 3, 16, 64)
    q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)
    p = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
    return (p @ v).transpose(1, 2).reshape(n * 577, 1024), v


def _attention_bound(ref, v, n):
    """P is rounded to f16 before P V and the row sum: a normal weight is off by <= 2^-11 (1 + 2^-11) relative, so the normalised sum is
    off by <= 2^-9 max|v| of its (crop, head); a weight below 2^-14 lands in f16's subnormals and is off by up to 2^-25 absolute, at most
    640 of them over a row sum l >= 1: <= 640 2^-25 2 max|v| < 2^-13 max|v|; the stored result adds one rounding (2^-11 relative)."""
    vmax = v.abs().amax(dim=(2, 3))[:, None, :, None].expand(n, 577, 16, 64).reshape(n * 577, 1024)
    return (2.0 ** -9 + 2.0 ** -13) * vmax + U * ref.abs() + 1e-30


def test_attention_against_fp64(hooks):
    g = torch.Generator(device=DEV).manual_seed(5)
    n = 3
    qkv = torch.randn(n * 577 + 64, 3072, generator=g, device=DEV)
    x = qkv[: n * 577].view(n, 577, 3, 16, 64)
    x[0, :, 0, 1] *= 6.0                                   # head 1 of crop 0: saturated logits (scores in the hundreds)
    x[0, :, 0, 2] = 0.0                                    # head 2: all-equal logits -> the mean of v
    x[0, :, 1, 3] *= 0.01                                  # head 3: one dominant key, every other weight deep in f16's subnormals
    x[0, 123, 1, 3] = 40.0
    x[1] *= 0.3
    x[1, :, 0, 4] = 0.0                                    # head 4 of crop 1: all-equal logits and v = 1: the result is exactly 1, and
    x[1, :, 2, 4] = 1.0                                    # only if the 63 zero-filled keys 577..639 are masked (unmasked: 577/640)
    x[2, :, 2] *= 1e3                                      # crop 2's values are huge: crop 1's padded keys read zeros, never these rows
    qkv[n * 577:] = 3e4                                    # rows after the last crop (outside the map's crop extent: never read)
    qkv = qkv.to(F16)
    ctx = torch.full((n * 577 + 8, 1024), float("nan"), device=DEV, dtype=F16)
    assert hooks.tpc_attention_f16(_ptr(qkv), _ptr(ctx), n, None) == 0
    torch.cuda.synchronize()
    assert torch.isnan(ctx[n * 577:].float()).all()
    ref, v = _attention_ref(qkv, n)
    out = ctx[: n * 577].double()
    _check(out, ref, _attention_bound(ref, v, n), "attention")
    assert (out.view(n, 577, 16, 64)[1, :, 4] == 1.0).all()


# ------------------------------------------------------------------------------------------------------------------------------
# the whole tower
# ------------------------------------------------------------------------------------------------------------------------------
def _f16_weights(outlier):
    """seeded weights rounded to fp16: the fp16 towers (ours and the eager one) and the fp64 one compute from the same values"""
    return {k: v.half().float() for k, v in cto.make_weights(23, seed=11, outlier=outlier, device=DEV).items()}


@pytest.fixture(scope="module", params=[False, True], ids=["standard", "outlier"])
def tower(request):
    from tokenpacker_b200 import CLIPVisionTowerB200
    w = _f16_weights(request.param)
    model = cto.FakeCLIPVisionModel({k: v.half() for k, v in w.items()}).to(DEV)
    return w, model, CLIPVisionTowerB200(model, dtype=F16)


def _errors(got, ref):
    d = got.double() - ref
    return float(d.norm() / ref.norm()), float(d.abs().max())


@pytest.mark.parametrize("n", [1, 5])
def test_tower_against_oracle(tower, n):
    w, _, t = tower
    images = cto.make_images(n, seed=n, device=DEV).bfloat16()
    with torch.no_grad():
        ours = t.hidden_states(images)
        ref = cto.forward(w, images.half().double(), 23, torch.float64)
        hf = ct16.forward_f16_eager(w, images, 23)
    torch.cuda.synchronize()
    for got, layer in zip(ours, cto.OUT_LAYERS):
        assert got.shape == (n, 577, 1024) and got.dtype == F16
        rms, mx = _errors(got, ref[layer])
        rms_hf, mx_hf = _errors(hf[layer], ref[layer])
        # the gate is transformers' own fp16 tower on the same inputs: neither the rel-RMS nor the largest error may exceed its own
        assert rms <= rms_hf, (layer, rms, rms_hf)
        assert mx <= mx_hf, (layer, mx, mx_hf)


def test_bitwise_properties(tower):
    """batch invariance, run-to-run determinism, strided crops (bf16 and f16), and bf16 crops give the bits of crops.half()"""
    _, _, t = tower
    images = cto.make_images(4, seed=9, device=DEV).bfloat16()
    with torch.no_grad():
        full = t.hidden_states(images)
        again = t.hidden_states(images)
        single = t.hidden_states(images[2:3])
        halves = t.hidden_states(images.half())
        from_fp32 = t.hidden_states(images.float())                          # other dtypes are cast to f16 first
        strided = []
        for dt in (torch.bfloat16, F16):
            big = torch.full((4, 3 * 336 * 336 + 4096), float("nan"), device=DEV, dtype=dt)
            view = big[:, :3 * 336 * 336].view(4, 3, 336, 336)
            view.copy_(images)
            strided.append(t.hidden_states(view))
    torch.cuda.synchronize()
    for i, a in enumerate(full):
        assert a.dtype == F16 and torch.isfinite(a.float()).all()
        assert torch.equal(a, again[i])
        assert torch.equal(a[2:3], single[i])
        assert torch.equal(a, halves[i])
        assert torch.equal(a, from_fp32[i])
        assert torch.equal(a, strided[0][i]) and torch.equal(a, strided[1][i])


def test_precisions_never_share_a_cache(tower):
    """A dtype=None module and a dtype=torch.float16 one over the same model, called in turn: each gives the bits of a fresh module of
    its own precision."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    _, model, _ = tower
    images = cto.make_images(2, seed=13, device=DEV).bfloat16()
    with torch.no_grad(), pytest.warns(UserWarning, match="cast to bf16"):
        t_bf, t_16 = CLIPVisionTowerB200(model), CLIPVisionTowerB200(model, dtype=F16)
        runs = [t_bf.hidden_states(images), t_16.hidden_states(images), t_bf.hidden_states(images), t_16.hidden_states(images)]
        fresh_bf = CLIPVisionTowerB200(model).hidden_states(images)
        fresh_16 = CLIPVisionTowerB200(model, dtype=F16).hidden_states(images)
    torch.cuda.synchronize()
    for i in range(4):
        assert runs[0][i].dtype == torch.bfloat16 and runs[1][i].dtype == F16
        assert torch.equal(runs[0][i], fresh_bf[i]) and torch.equal(runs[2][i], fresh_bf[i])
        assert torch.equal(runs[1][i], fresh_16[i]) and torch.equal(runs[3][i], fresh_16[i])


def test_refuses_gradients_and_cpu(tower):
    _, _, t = tower
    x = torch.zeros(1, 3, 336, 336, device=DEV, requires_grad=True)
    with pytest.raises(NotImplementedError, match="forward only"):
        t.hidden_states(x)
    with pytest.raises(RuntimeError, match="no CPU path"):
        with torch.no_grad():
            t.hidden_states(torch.zeros(1, 3, 336, 336, dtype=F16))


# ------------------------------------------------------------------------------------------------------------------------------
# one layer, stage by stage
# ------------------------------------------------------------------------------------------------------------------------------
def _ln_ref(x, gamma, beta):
    """(reference, bound) of f16(LayerNorm(x) gamma + beta) in fp32, derived as in test_clip_tower_gpu.py with the f16 rounding"""
    x = x.double()
    g = gamma.double()
    mu = x.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
    xh = (x - mu) * rstd
    ref = xh * g + beta.double()
    floor = g.abs() * (2.0 ** -12 * xh.abs() + rstd * 1025 * E * x.abs().mean(-1, keepdim=True)) + 2 * E * ref.abs()
    return ref, U * ref.abs() + (1 + U) * floor + 1e-30


def test_one_layer_stage_by_stage(hooks, tower):
    """Layer 1 alone on a workspace poisoned with 0xFF bytes (0xFFFF is NaN in f16 too): every stage against fp64 of that stage computed
    from the f16 values the kernels stored before it.  q is scaled by 1/8 after its bias with one rounding (the packed f16 weights are
    unscaled)."""
    _one_layer_stages(hooks, tower, 2)


def _one_layer_stages(hooks, tower, n):
    """the stages of test_one_layer_stage_by_stage over n crops (tests/test_clip_tower_batches_gpu.py runs the other plans' n)"""
    w, _, t = tower
    images = cto.make_images(n, seed=21, device=DEV).half()
    with torch.no_grad():
        x = cto.forward(w, images.float(), 1, torch.float64)[1].half().reshape(n * 577, 1024).contiguous()
        packed, (cw, _) = t._packed_weights(torch.device(DEV))
    offs = (C.c_int64 * 7)()
    assert hooks.tpc_workspace_offsets_f16(n, offs) == 0
    ws = torch.full((offs[6],), 0xFF, dtype=torch.uint8, device=DEV)
    out = torch.full((n * 577, 1024), float("nan"), device=DEV, dtype=F16)
    assert hooks.tpc_layer_f16(packed.data_ptr(), C.addressof(cw), 1, x.data_ptr(), out.data_ptr(), n, ws.data_ptr(), offs[6], None) == 0
    torch.cuda.synchronize()
    M = n * 577

    def region(i, cols, dtype=F16):
        size = 4 if dtype == torch.float32 else 2
        return ws[offs[i]: offs[i] + M * cols * size].view(dtype).view(M, cols)

    y1, qkv, ctx, y2, h = region(0, 1024), region(1, 3072), region(2, 1024), region(4, 1024), region(5, 4096)
    xp = region(3, 1024, torch.float32)
    k = {a: w[b].to(DEV) for a, b in cto.layer_keys(1).items()}
    hf = lambda v: v.half()
    ref, bound = _ln_ref(x, hf(k["layer_norm1.weight"]), hf(k["layer_norm1.bias"]))
    _check(y1, ref, bound, "y1 = layer_norm1(x)")
    ref, bound = _gemm_bound(y1, hf(k["self_attn.q_proj.weight"]), hf(k["self_attn.q_proj.bias"]).float(), alpha=0.125)
    _check(qkv[:, :1024], ref, bound, "q = q_proj(y1) / 8")
    wkv = torch.cat([k["self_attn.k_proj.weight"], k["self_attn.v_proj.weight"]])
    bkv = torch.cat([k["self_attn.k_proj.bias"], k["self_attn.v_proj.bias"]])
    ref, bound = _gemm_bound(y1, hf(wkv), hf(bkv).float())
    _check(qkv[:, 1024:], ref, bound, "k | v")
    ref, v = _attention_ref(qkv, n)
    _check(ctx, ref, _attention_bound(ref, v, n), "ctx")
    ref, bound = _gemm_bound(ctx, hf(k["self_attn.out_proj.weight"]), hf(k["self_attn.out_proj.bias"]).float(), x, out_f16=False)
    _check(xp, ref, bound, "x' = x + out_proj(ctx)")
    ref, bound = _ln_ref(xp, hf(k["layer_norm2.weight"]), hf(k["layer_norm2.bias"]))
    _check(y2, ref, bound, "y2 = layer_norm2(x')")
    ref, bound = _gemm_bound(y2, hf(k["mlp.fc1.weight"]), hf(k["mlp.fc1.bias"]).float(), None, 2)
    _check(h, ref, bound, "h = quick_gelu(fc1(y2))")
    ref, bound = _gemm_bound(h, hf(k["mlp.fc2.weight"]), hf(k["mlp.fc2.bias"]).float(), xp)
    _check(out, ref, bound, "x'' = x' + fc2(h)")


# ------------------------------------------------------------------------------------------------------------------------------
# end to end: decoded images -> HD crops (bf16) -> fp16 tower -> bf16 -> projector, as the evaluation scripts run it
# ------------------------------------------------------------------------------------------------------------------------------
def test_uint8_images_to_packed_projector_output(tower):
    from tokenpacker_b200 import CLIPVisionTowerB200, TokenPackerB200, hd_preprocess_batch
    w, model, t = tower
    g = torch.Generator(device=DEV).manual_seed(31)
    images = [torch.randint(0, 256, (h_, w_, 3), generator=g, device=DEV, dtype=torch.uint8) for h_, w_ in ((336, 336), (500, 700))]
    torch.manual_seed(7)
    proj = TokenPackerB200(hidden_size=1024, scale_factor=2).to(DEV, torch.bfloat16).eval()
    sep = torch.randn(1024, device=DEV).bfloat16()
    ret = torch.randn(1024, device=DEV).bfloat16()
    bf_model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    t_bf = CLIPVisionTowerB200(bf_model)                              # the drop-in as it computes without dtype=
    bf16 = lambda hs: [h.to(torch.bfloat16) for h in hs]              # clip_encoder.py:62
    with torch.no_grad():
        crops, hb, wb = hd_preprocess_batch(images, patch_num=9, dtype=torch.bfloat16)
        ours = t.hidden_states(crops)                                 # the preprocessing output, read in place
        assert all(h.dtype == F16 for h in ours)
        ref_hs = cto.forward(w, crops.half().double(), 23, torch.float64)
        eager_hs = ct16.forward_f16_eager(w, crops, 23)
        run = lambda hs: proj.forward_hidden_states_packed(bf16(hs), hb, wb, sep, ret)[0].double()
        out = run(ours)
        ref = run([ref_hs[i] for i in cto.OUT_LAYERS])
        eager = run([eager_hs[i] for i in cto.OUT_LAYERS])
        out_bf = run(t_bf.hidden_states(crops))
    torch.cuda.synchronize()
    # the same projector on every side: what differs is the tower.  Ours must not be further from the fp64 tower's result than
    # transformers' fp16 tower (the reference's evaluation setting) is.
    rms, mx = _errors(out, ref)
    rms_e, mx_e = _errors(eager, ref)
    assert torch.isfinite(out).all()
    assert rms <= rms_e and mx <= mx_e, (rms, rms_e, mx, mx_e)
    # the gap this closes: against the composition the reference evaluates with, the bf16 drop-in and the fp16 one
    gap_bf, gap_bf_mx = _errors(out_bf, eager)
    gap_16, gap_16_mx = _errors(out, eager)
    print(f"\nprojector output vs the fp16-eager composition: bf16 tower rel-RMS {gap_bf:.3e} "
          f"max {gap_bf_mx:.3e}; fp16 tower rel-RMS {gap_16:.3e} max {gap_16_mx:.3e}; vs fp64: fp16 tower {rms:.3e}, fp16 eager {rms_e:.3e}")
    assert gap_16 < gap_bf, (gap_16, gap_bf)
