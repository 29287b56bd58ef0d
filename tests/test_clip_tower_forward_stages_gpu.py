"""The CLIP tower's forward pieces that the per-layer stage tests do not reach, each on its own against fp64 or bit for bit:
  * the derived weight cache (tp_clip_tower_pack_weights / _f16) of all 23 layers, with q weights at bf16's subnormals and near its max;
  * the embedding stage (run_clip_embed: im2col -> patch GEMM -> class / position embedding + pre_layrnorm) step by step, in the bf16
    tower, the fp16 tower on bf16 crops and the fp16 tower on fp16 crops, from strided crops at an odd element offset;
  * every LayerNorm instantiation of the forward (layer_norm1 / layer_norm2 in both precisions, both pre_layrnorms) on adversarial rows;
  * quick_gelu at every finite bf16 and fp16 input: the fused fc1 epilogue of both kernels and precisions, the training forward's
    elementwise pass, and the backward's derivative and bias column sums.
Hooks: tests/csrc/tp_clip_tower_hooks.cu (tpc_embed, tpc_layernorm, tpc_packed_layout, tpc_gemm), tp_clip_tower_f16_hooks.cu
(tpc_embed_f16, tpc_gemm_f16) and tp_clip_tower_train_hooks.cu (tptt_quick_gelu_fwd, tptt_quick_gelu_bwd); each calls the product's own
launch code.

Every bound is derived from the kernel's operation order (fp32 unit roundoff E = 2^-24; the stored result one rounding, U = 2^-8 in bf16,
2^-11 in fp16, plus half the spacing of the subnormals it can land in).  Workspaces start as 0xFF bytes (NaN in bf16 and fp16) and
outputs sit between NaN guard rows: each step must leave everything outside its own regions as it was.  The worst error / bound ratio
of each check is recorded as a property."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import clip_tower_oracle as cto
from test_clip_tower_train_stages_gpu import _quick_gelu_grad_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "tokenpacker_b200")
BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
E = 2.0 ** -24                                     # fp32 unit roundoff
UNIT = {BF: 2.0 ** -8, F16: 2.0 ** -11}            # unit roundoff of the stored result
SUB = {BF: 2.0 ** -134, F16: 2.0 ** -25}           # half the spacing of its subnormals
CROP = 3 * 336 * 336
STRIDE = CROP + 8                                  # the crops' stride: 8 elements between crops
CROPS_BF16, CROPS_F16 = 1, 2
INF16 = 65520.0                                    # the smallest magnitude f16 rounds to inf


def _lib(name, sigs):
    import tokenpacker_b200  # noqa: F401  (the product library is loaded next to these)
    lib = C.CDLL(os.path.join(LIBDIR, name))
    for fn, args in sigs.items():
        getattr(lib, fn).restype = C.c_int
        getattr(lib, fn).argtypes = args
    return lib


p, i64, i32 = C.c_void_p, C.c_int64, C.c_int


@pytest.fixture(scope="module")
def ct():
    return _lib("libtokenpacker_b200_clip_tower_hooks.so", {
        "tpc_embed_offsets": [i64, C.POINTER(i64)], "tpc_embed": [p, p, p, i32, i64, i64, p, C.c_size_t, i32, p],
        "tpc_layernorm": [p, i32, i64, p, p, p, i32, p], "tpc_packed_layout": [C.POINTER(i64)],
        "tpc_gemm": [p, i64, p, i64, p, i64, i64, i64, i64, p, p, i64, i32, i32, p]})


@pytest.fixture(scope="module")
def ct16():
    return _lib("libtokenpacker_b200_clip_tower_f16_hooks.so", {
        "tpc_embed_f16": [p, p, p, i32, i64, i64, p, C.c_size_t, i32, p],
        "tpc_gemm_f16": [p, i64, p, i64, p, i64, i64, i64, i64, p, p, i64, i32, i32, i32, C.c_float, i32, i32, i32, p]})


@pytest.fixture(scope="module")
def ctt():
    return _lib("libtokenpacker_b200_clip_tower_train_hooks.so", {
        "tptt_quick_gelu_fwd": [p, p, p, i64, p], "tptt_quick_gelu_bwd": [p, p, i64, p, p, p],
        "tptt_saved_offsets": [i64, C.POINTER(i64)]})


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Worst:
    """the largest error / bound ratio of each named check, recorded as a test property"""

    def __init__(self, record_property):
        self.record, self.seen = record_property, {}

    def check(self, name, got, ref, bound, zero_ok=None):
        """|got - ref| <= bound elementwise (NaN and inf fail); zero_ok: where a ±0 result is accepted as well"""
        got = got.double()
        ratio = (got - ref).abs() / bound
        if zero_ok is not None:
            ratio = torch.where(zero_ok & (got == 0), torch.zeros_like(ratio), ratio)
        bad = ~(ratio <= 1)
        assert not bool(bad.any()), (name, float(ratio[bad].nan_to_num(float("inf")).max()), int(bad.sum()))
        self.seen[name] = max(self.seen.get(name, 0.0), float(ratio.max()) if ratio.numel() else 0.0)
        self.record(f"worst_{name}", f"{self.seen[name]:.3f}")


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------------------------------------
# LayerNorm: fp64 reference and the bound of clip_ln_row_store's fp32 arithmetic
# ------------------------------------------------------------------------------------------------------------------------------
def _warp_mean(x32):
    """clip_ln_row_store's mean in its own fp32 order: lane l adds its 32 columns 256 j + 8 l + m (j = 0..3, m = 0..7) in sequence,
    five xor-shuffle levels (16, 8, 4, 2, 1) add the lanes, and the sum is scaled by 1/1024 (exact)"""
    rows = x32.shape[0]
    v = x32.reshape(rows, 4, 32, 8).permute(0, 2, 1, 3).reshape(rows, 32, 32)
    acc = torch.zeros(rows, 32, dtype=F32, device=x32.device)
    for i in range(32):
        acc = acc + v[:, :, i]
    lanes = torch.arange(32, device=x32.device)
    for off in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ off]
    return acc[:, 0] * (1.0 / 1024)


def _ln_expect(x32, gamma, beta, dtype):
    """(reference, bound) of dtype(LayerNorm(x) gamma + beta) from the fp32 row values x32 the kernel holds.  The mean's rounding
    error d = |mean32 - mean| is taken from the kernel's own summation order (_warp_mean), since it is the one error that is not small
    relative to the row's spread when |mean| >> std.  With the mean off by d the deviations' mean square is var + d^2, so rstd is off
    by <= d^2 / (2 (var + eps)) relative, plus 2^-12 for the fp32 sum of 1024 squares (<= 1026 E) and rsqrtf; the deviation e - mean32
    rounds once (E |e - mean32|), the product with rstd once, the fma once; the stored result one more rounding."""
    x = x32.double()
    g, b = gamma.double(), beta.double()
    mu = x.mean(-1, keepdim=True)
    dev = x - mu
    var = (dev * dev).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + 1e-5)
    xh = dev * rstd
    ref = xh * g + b
    d = (_warp_mean(x32).double()[:, None] - mu).abs()
    rel = 2.0 ** -12 + d * d / (2 * (var + 1e-5))
    floor = g.abs() * (xh.abs() * (rel + 2 * E) + rstd * (d + E * (dev.abs() + d))) + 2 * E * ref.abs()
    u = UNIT[dtype]
    return ref, u * ref.abs() + (1 + u) * floor + SUB[dtype]


def _check_ln(worst, name, got, x32, gamma, beta, dtype, exact_beta=False):
    """got (dtype) against _ln_expect; f16 results past 65504 must be ±inf exactly where the fp64 result rounds to inf in f16 (and no
    fp64 result may lie within its bound of that threshold, so the comparison is exact); exact_beta: every row must equal beta"""
    ref, bound = _ln_expect(x32, gamma, beta, dtype)
    g = got.double()
    assert not bool(torch.isnan(g).any()), name
    if exact_beta:
        assert bool((got.float() == beta.float()[None]).all()), name
        return
    if dtype == F16:
        over = ref.abs() >= INF16
        assert not bool(((ref.abs() - INF16).abs() <= bound).any()), f"{name}: a result on the f16 overflow threshold"
        assert torch.equal(torch.isinf(g), over), name
        assert torch.equal(torch.sign(g[over]), torch.sign(ref[over])), name
        keep = ~over
        worst.check(name, g[keep], ref[keep], bound[keep])
    else:
        worst.check(name, g, ref, bound)


OUTLIERS = list(cto.OUTLIER_CHANNELS)


def _row_sets(x_dtype, dtype, rows, seed):
    """[(name, x (x_dtype) [rows, 1024], gamma, beta, exact_beta)]: the adversarial row sets of one LayerNorm instantiation"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    f32_in = x_dtype == F32
    gamma = (1 + 0.1 * rn(1024)).to(dtype)
    beta = (0.05 * rn(1024)).to(dtype)
    beta = torch.where(beta == 0, torch.full_like(beta, 0.01), beta)          # no ±0: the exact cases compare values
    big = 6e4 if x_dtype == F16 else 3e4
    out = [("normal", rn(rows, 1024) * 2 + 0.3, gamma, beta, False)]
    # constant rows: every partial sum is exact (16-bit inputs, or fp32 of <= 19 significant bits), the deviations are 0 and the
    # output is beta itself
    consts = [0.0, 1.5, -7.25, big, -big] + ([30000.125, -1234.5625] if f32_in else [])
    c = torch.tensor([consts[i % len(consts)] for i in range(rows)], device=DEV)
    out.append(("constant", c[:, None].expand(rows, 1024).clone(), gamma, beta, True))
    if f32_in:                                    # |mean| >> std: E[x^2] - mean^2 in fp32 would lose the variance entirely
        out.append(("offset1e4", 1e4 + 1e-2 * rn(rows, 1024), gamma, beta, False))
    out.append(("std1e-4", (0.5 if f32_in else 0.0) + 1e-4 * rn(rows, 1024), gamma, beta, False))
    x = rn(rows, 1024)
    x[:, OUTLIERS] = torch.tensor([1.0, -1.0, 1.0, -1.0], device=DEV) * (3e4 if dtype == F16 and not f32_in else 1e3)
    out.append(("outliers", x, gamma, beta, False))
    out.append(("gamma0", rn(rows, 1024) * 2, torch.zeros_like(gamma), beta, True))
    if dtype == F16:                              # five channels scaled by 4e4: three of them past 65504
        x = rn(rows, 1024)
        ch = [5, 77, 400, 700, 1023]
        x[:, ch] = torch.tensor([3.0, -3.0, 1.0, 1.4, -2.0], device=DEV)
        gam = gamma.clone()
        gam[ch] = 4e4
        out.append(("overflow", x, gam, beta, False))
    return [(n, v.to(x_dtype), gm, bt, ex) for n, v, gm, bt, ex in out]


@pytest.mark.parametrize("x_dtype,dtype", [(BF, BF), (F32, BF), (F16, F16), (F32, F16)],
                         ids=["bf16-layer_norm1", "fp32-layer_norm2", "f16-layer_norm1", "fp32-f16-layer_norm2"])
def test_layernorm_adversarial(ct, record_property, x_dtype, dtype):
    """clip_layernorm_kernel, as launch_clip_ln runs it, on 1, 7 and 3 x 577 rows of every adversarial set; NaN rows above and below
    both the input and the output: none is read, none is written"""
    worst = Worst(record_property)
    for rows in (1, 7, 3 * 577):
        for name, x, gamma, beta, exact in _row_sets(x_dtype, dtype, rows, rows + 11):
            xf = torch.full((rows + 2, 1024), float("nan"), dtype=x_dtype, device=DEV)
            xf[1:rows + 1] = x
            y = torch.full((rows + 2, 1024), float("nan"), dtype=dtype, device=DEV)
            assert ct.tpc_layernorm(_ptr(xf[1:]), int(x_dtype == F32), rows, _ptr(gamma), _ptr(beta), _ptr(y[1:]), int(dtype == F16),
                                    _stream()) == 0
            torch.cuda.synchronize()
            assert bool(torch.isnan(y[0].float()).all()) and bool(torch.isnan(y[rows + 1].float()).all()), name
            _check_ln(worst, f"{name}", y[1:rows + 1], x.float(), gamma, beta, dtype, exact)
    x = torch.zeros(8, 1024, device=DEV)
    assert ct.tpc_layernorm(_ptr(x), 2, 8, _ptr(x), _ptr(x), _ptr(x), 0, _stream()) != 0         # no other instantiation


# ------------------------------------------------------------------------------------------------------------------------------
# towers, crops and the embedding stage's runs
# ------------------------------------------------------------------------------------------------------------------------------
def _embed_weights(dtype):
    """seeded weights in the tower's precision, with four huge position-embedding channels (the pre-LN input's hard case)"""
    w = cto.round_bf16(cto.make_weights(23, seed=21, device=DEV))
    pos = w["embeddings.position_embedding.weight"]
    pos[:, OUTLIERS] += torch.tensor([70.0, -60.0, 90.0, -50.0], device=DEV)
    return {k: v.to(dtype) for k, v in w.items()}


class Tower:
    def __init__(self, dtype, w=None):
        from tokenpacker_b200 import CLIPVisionTowerB200
        self.dtype = dtype
        self.w = _embed_weights(dtype) if w is None else w
        self.model = cto.FakeCLIPVisionModel(dict(self.w)).to(DEV)
        self.tower = CLIPVisionTowerB200(self.model, dtype=dtype)
        with torch.no_grad():
            self.packed, (self.cw, self.keep) = self.tower._packed_weights(torch.device(DEV))
        torch.cuda.synchronize()


@pytest.fixture(scope="module")
def towers():
    return {BF: Tower(BF), F16: Tower(F16)}


def _crops(n, dtype, seed):
    """n crops of cto.make_images in dtype, STRIDE elements apart from an odd element offset, NaN between them"""
    base = torch.full((n * STRIDE + 16,), float("nan"), dtype=dtype, device=DEV)
    view = base.as_strided((n, 3, 336, 336), (STRIDE, 336 * 336, 336, 1), 1)
    view.copy_(cto.make_images(n, seed=seed, device=DEV))
    return base, view


def _offsets(ct, n):
    out = (C.c_int64 * 3)()
    assert ct.tpc_embed_offsets(n, out) == 0
    return dict(zip(("h", "xa", "total"), list(out)))


def _embed(ct, ct16, tw, cw, crops, crops_dtype, n, step):
    """a fresh 0xFF workspace, then run_clip_embed up to step; returns (workspace, patch rows [576 n, 592], xa [n, 577, 1024])"""
    off = _offsets(ct, n)
    ws = torch.full((off["total"],), 0xFF, dtype=torch.uint8, device=DEV)
    args = (_ptr(tw.packed), C.byref(cw), _ptr(crops), crops_dtype, n, STRIDE, _ptr(ws), ws.numel(), step, _stream())
    assert (ct16.tpc_embed_f16(*args) if tw.dtype == F16 else ct.tpc_embed(*args)) == 0
    torch.cuda.synchronize()
    R, M = 576 * n, 577 * n
    patches = ws[off["h"]:off["h"] + R * 592 * 2].view(tw.dtype).view(R, 592)
    xa = ws[off["xa"]:off["xa"] + M * 2048].view(tw.dtype).view(n, 577, 1024)
    return ws, patches, xa


def _only_owned(ct, ws, n, step):
    """everything but the step's own regions still holds the 0xFF poison: patch columns 0..587 (step 1), token rows 1..576 of xa
    (step 2), every row of xa (step 3)"""
    off = _offsets(ct, n)
    rest = ws.clone()
    R, M = 576 * n, 577 * n
    rest[off["h"]:off["h"] + R * 592 * 2].view(torch.int16).view(R, 592)[:, :588] = -1
    if step >= 2:
        rest[off["xa"]:off["xa"] + M * 2048].view(torch.int16).view(n, 577, 1024)[:, 0 if step == 3 else 1:] = -1
    return bool((rest == 0xFF).all())


def _unfold(crops, dtype):
    """the patch rows [576 n, 588] in the conv weight's (c, ky, kx) order, from the crops converted to dtype (bf16 -> f16 on the CPU:
    one round-to-nearest-even through fp32, as crops.half() rounds)"""
    c = crops if crops.dtype == dtype else crops.cpu().float().to(dtype).to(DEV)
    n = c.shape[0]
    return F.unfold(c, 14, stride=14).transpose(1, 2).reshape(576 * n, 588)


def _special_bf16():
    """bf16 values whose f16 conversions tell round-to-nearest-even from truncation and saturation: ties at the f16 subnormal
    spacing ((2k + 1) 2^-25), other values in [2^-30, 2^-14], and magnitudes around f16's largest finite value"""
    g = torch.Generator().manual_seed(99)
    ties = (2 * torch.arange(128, dtype=F64) + 1) * 2.0 ** -25
    tiny = torch.exp2(-30 + 16 * torch.rand(1024, generator=g, dtype=F64))
    huge = torch.tensor([65280.0, 65504.0, 65519.0, 65520.0, 1e5, 2.0 ** 15 * 1.99], dtype=F64)
    v = torch.cat([ties, tiny, huge])
    return torch.cat([v, -v]).to(BF)


CASES = [(BF, BF), (F16, BF), (F16, F16)]


@pytest.mark.parametrize("n", [1, 3, 29])
@pytest.mark.parametrize("tower_dtype,crops_dtype", CASES, ids=["bf16-tower", "f16-tower-bf16-crops", "f16-tower-f16-crops"])
def test_embedding_stage(ct, ct16, ctt, towers, record_property, tower_dtype, crops_dtype, n):
    worst = Worst(record_property)
    tw = towers[tower_dtype]
    T = tower_dtype
    code = CROPS_F16 if crops_dtype == F16 else CROPS_BF16
    R, M = 576 * n, 577 * n
    base, crops = _crops(n, crops_dtype, seed=40 + n)

    # ---- step 1: im2col, bit for bit F.unfold of the crops in the tower's type
    if (T, crops_dtype) == (F16, BF):
        sbase, scrops = _crops(n, BF, seed=40 + n)
        sp = _special_bf16()
        scrops[0, 0].view(-1)[:sp.numel()] = sp.to(DEV)
        scrops[n - 1, 2].view(-1)[-sp.numel():] = sp.flip(0).to(DEV)
        ws, patches, _ = _embed(ct, ct16, tw, tw.cw, scrops, code, n, 1)
        want = _unfold(scrops, T)
        assert bool(torch.isinf(want.float()).any()) and bool((want.float().abs() == 2.0 ** -24).any())
        assert torch.equal(_bits(patches[:, :588]), _bits(want)), "bf16 -> f16 patch rows"
        assert _only_owned(ct, ws, n, 1)
    ws, patches, _ = _embed(ct, ct16, tw, tw.cw, crops, code, n, 1)
    rows1 = patches[:, :588].clone()
    assert torch.equal(_bits(rows1), _bits(_unfold(crops, T))), "patch rows"
    assert _only_owned(ct, ws, n, 1)

    # ---- step 2: the patch GEMM into token rows 1..576 of every crop; row 0 keeps the poison
    ws, patches, xa = _embed(ct, ct16, tw, tw.cw, crops, code, n, 2)
    assert torch.equal(_bits(patches[:, :588]), _bits(rows1))
    assert _only_owned(ct, ws, n, 2)
    wp = tw.w["embeddings.patch_embedding.weight"].reshape(1024, 588).double()
    a = rows1.double()
    ref = a @ wp.T
    u = UNIT[T]
    bound = u * ref.abs() + (1 + u) * 589 * E * (a.abs() @ wp.abs().T) + SUB[T]
    rows2 = xa[:, 1:].reshape(R, 1024)
    worst.check("patch_gemm", rows2, ref, bound)
    xa2 = xa.clone()

    # ---- step 3: + class / position embedding (one fp32 add, as torch adds), pre_layrnorm -> hidden_states[0]
    ws, patches, xa = _embed(ct, ct16, tw, tw.cw, crops, code, n, 3)
    assert _only_owned(ct, ws, n, 3)
    e = xa2.float()
    e[:, 0] = tw.w["embeddings.class_embedding"].float()
    e = (e + tw.w["embeddings.position_embedding.weight"].float()).reshape(M, 1024)
    _check_ln(worst, "pre_layrnorm", xa.reshape(M, 1024), e, tw.w["pre_layrnorm.weight"], tw.w["pre_layrnorm.bias"], T)
    hs0 = xa.clone()

    if T == BF:                         # the product's own hidden_states[0]: layer 0's input in a whole-tower training forward
        from tokenpacker_b200 import CLIPVisionTowerB200
        model = cto.FakeCLIPVisionModel(dict(tw.w)).to(DEV)
        for name, prm in model.named_parameters():
            prm.requires_grad_("encoder.layers." not in name)
        model.gradient_checkpointing = True
        t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
        outs = t.hidden_states(crops)
        torch.cuda.synchronize()
        so = (C.c_int64 * 12)()
        assert ctt.tptt_saved_offsets(n, so) == 0
        saved = outs[3].grad_fn.saved
        x0 = saved[so[1]:so[1] + M * 2048].view(BF).view(n, 577, 1024)
        assert torch.equal(_bits(x0), _bits(hs0)), "hidden_states[0] of the training forward"


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
def test_embed_preln_adversarial(ct, ct16, towers, record_property, dtype, n):
    """clip_embed_preln_kernel on the adversarial row sets: zero crops make every patch row +0, so e = position_embedding[t] (class
    embedding 0 at token 0), and the position embedding carries the rows"""
    from tokenpacker_b200 import _lib
    worst = Worst(record_property)
    tw = towers[dtype]
    base, crops = _crops(n, dtype, seed=1)
    crops.zero_()
    code = CROPS_F16 if dtype == F16 else CROPS_BF16
    for name, x, gamma, beta, exact in _row_sets(dtype, dtype, 577, 5 + n):
        cls = torch.zeros(1024, dtype=dtype, device=DEV)
        cw = _lib.TpClipTowerWeights.from_buffer_copy(tw.cw)
        cw.pos_emb, cw.class_emb = x.data_ptr(), cls.data_ptr()
        cw.pre_ln_w, cw.pre_ln_b = gamma.data_ptr(), beta.data_ptr()
        _, _, xa2 = _embed(ct, ct16, tw, cw, crops, code, n, 2)
        rows = xa2[:, 1:].float()
        assert bool((rows == 0).all())
        ws, _, xa = _embed(ct, ct16, tw, cw, crops, code, n, 3)
        assert _only_owned(ct, ws, n, 3)
        e = torch.cat([torch.zeros(n, 1, 1024, device=DEV), rows], 1) + x.float()[None]
        _check_ln(worst, name, xa.reshape(577 * n, 1024), e.reshape(577 * n, 1024), gamma, beta, dtype, exact)


# ------------------------------------------------------------------------------------------------------------------------------
# the derived weight cache
# ------------------------------------------------------------------------------------------------------------------------------
def _pack_weights(dtype):
    """seeded weights with q weights and biases at the type's subnormals and near its largest finite value, in every layer"""
    w = _embed_weights(dtype)
    info = torch.finfo(dtype)
    g = torch.Generator(device=DEV).manual_seed(5)
    sub = torch.arange(1, 129, device=DEV, dtype=F32) * info.smallest_normal / 128       # subnormals: bf16 has 7 fraction bits,
    sub = sub.to(dtype)                                                                   # f16 10 (these are exact in both)
    top = torch.tensor([info.max, info.max * 0.75, info.max / 2, info.smallest_normal], device=DEV).to(dtype)
    for i in range(23):
        k = cto.layer_keys(i)
        q, qb = w[k["self_attn.q_proj.weight"]], w[k["self_attn.q_proj.bias"]]
        r = int(torch.randint(0, 1000, (1,), generator=g, device=DEV))
        q[r, :128], q[r + 1, :128] = sub, -sub
        q[r + 2, :4], q[r + 3, :4] = top, -top
        qb[:128] = sub if i % 2 == 0 else -sub
        qb[200:204] = top
    return w


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
def test_pack(ct, dtype):
    """tp_clip_tower_pack_weights(_f16) of all 23 layers: q|k|v (bf16: q times 1/8, rounded once), every bias as fp32 (the bf16 q bias
    times 1/8), the patch weight in 592-element rows.  Bit for bit."""
    tw = Tower(dtype, _pack_weights(dtype))
    lay = (C.c_int64 * 9)()
    assert ct.tpc_packed_layout(lay) == 0
    patch_w, layer0, layer_bytes, w_qkv, b_qkv, b_o, b_fc1, b_fc2, total = list(lay)
    P = tw.packed
    assert P.numel() == total
    pw = P[patch_w:patch_w + 1024 * 592 * 2].view(dtype).view(1024, 592)[:, :588]
    assert torch.equal(_bits(pw), _bits(tw.w["embeddings.patch_embedding.weight"].reshape(1024, 588)))
    vec = lambda B, off, n: B[off:off + 4 * n].view(F32)
    for i in range(23):
        k = {a: tw.w[b] for a, b in cto.layer_keys(i).items()}
        B = P[layer0 + i * layer_bytes:layer0 + (i + 1) * layer_bytes]
        q, qb = k["self_attn.q_proj.weight"], k["self_attn.q_proj.bias"].float()
        if dtype == BF:                                          # bf16(q * 0.125), rounded to nearest even, on the CPU
            q = (q.cpu().float() * 0.125).to(BF).to(DEV)
            qb = (qb.cpu() * 0.125).to(DEV)
        want = torch.cat([q, k["self_attn.k_proj.weight"], k["self_attn.v_proj.weight"]])
        got = B[w_qkv:w_qkv + 3 * 1024 * 1024 * 2].view(dtype).view(3072, 1024)
        assert torch.equal(_bits(got), _bits(want)), (i, "w_qkv")
        bq = torch.cat([qb, k["self_attn.k_proj.bias"].float(), k["self_attn.v_proj.bias"].float()])
        for name, off, ref in (("b_qkv", b_qkv, bq), ("b_o", b_o, k["self_attn.out_proj.bias"].float()),
                               ("b_fc1", b_fc1, k["mlp.fc1.bias"].float()), ("b_fc2", b_fc2, k["mlp.fc2.bias"].float())):
            assert torch.equal(vec(B, off, ref.numel()).view(torch.int32), ref.contiguous().view(torch.int32)), (i, name)


# ------------------------------------------------------------------------------------------------------------------------------
# quick_gelu at every finite input
# ------------------------------------------------------------------------------------------------------------------------------
def _all_finite(dtype):
    bits = np.arange(65536, dtype=np.uint16)
    exp = 0x7F80 if dtype == BF else 0x7C00
    bits = bits[(bits & exp) != exp]
    return torch.from_numpy(bits.view(np.int16)).to(DEV).view(dtype).view(-1, 256)      # bf16: [255, 256]; f16: [248, 256]


K_T = 2.45546696                                   # |t| / |x| in quick_gelu_pk: 1.702 / ln 2


def _quick_gelu_expect(x, dtype):
    """(reference, bound, zero_ok, saturated_pos, saturated_neg) of dtype(quick_gelu(x)) from the fp32 value x: the documented error
    (|t| / 16 + 8) 2^-23 relative (tp_ptx.cuh) with |t| capped at 128; past the cap the result must be x itself (x > 0) or ±0 (x < 0);
    ±0 is accepted wherever |quick_gelu(x)| < 2^-120 (the flush region)"""
    xd = x.double()
    ref = xd * torch.sigmoid(1.702 * xd)
    t = (K_T * xd).abs()
    floor = ref.abs() * (t.clamp(max=128) / 16 + 8) * 2.0 ** -23
    u = UNIT[dtype]
    bound = u * ref.abs() + (1 + u) * floor + SUB[dtype]
    return ref, bound, ref.abs() < 2.0 ** -120, (t > 128) & (xd > 0), (t > 128) & (xd < 0)


def _check_quick_gelu(worst, name, x, h, dtype):
    ref, bound, zero_ok, sat_pos, sat_neg = _quick_gelu_expect(x, dtype)
    hd = h.double()
    assert bool((hd[sat_pos] == x.to(dtype).double()[sat_pos]).all()), name
    assert bool((hd[sat_neg] == 0).all()), name
    keep = ~(sat_pos | sat_neg)
    worst.check(name, hd[keep], ref[keep], bound[keep], zero_ok[keep])


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
def test_quick_gelu_every_input(ct, ct16, ctt, record_property, dtype):
    """The fused fc1 epilogue (gelu = 2) on A = every finite value, B = I: C = A exactly in fp32, so quick_gelu_pk sees every value;
    both kernels give the same bits.  bf16: clip_quick_gelu_fwd_kernel on the same values gives those bits too, and holds the bound on
    fp32 values bf16 cannot represent."""
    worst = Worst(record_property)
    a = _all_finite(dtype)
    M = a.shape[0]
    eye = torch.eye(256, device=DEV).to(dtype)
    outs = []
    for mode in (1, 2):
        frame = torch.full((M + 4, 256 + 64), float("nan"), dtype=dtype, device=DEV)
        c = frame[2:M + 2, :256]
        if dtype == BF:
            st = ct.tpc_gemm(_ptr(a), 256, _ptr(eye), 256, _ptr(c), 256 + 64, M, 256, 256, None, None, 0, 2, mode, _stream())
        else:
            st = ct16.tpc_gemm_f16(_ptr(a), 256, _ptr(eye), 256, _ptr(c), 256 + 64, M, 256, 256, None, None, 0, 0, 2, 0, 1.0, 0, 0, mode,
                                   _stream())
        assert st == 0
        torch.cuda.synchronize()
        assert bool(torch.isnan(frame[:2].float()).all()) and bool(torch.isnan(frame[M + 2:].float()).all())
        assert bool(torch.isnan(frame[:, 256:].float()).all())
        outs.append(c.clone())
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "one-CTA and pair kernels differ"
    h = outs[0]
    _check_quick_gelu(worst, "epilogue", a.float(), h, dtype)
    if dtype != BF:
        return

    # the training forward's elementwise pass on the same fp32 values: z = bf16(z32) and the epilogue's bits (zeros: the GEMM's sum
    # of -0 is +0, so only their value is compared)
    z32 = a.float().contiguous()
    z = torch.full_like(a, float("nan"))
    hz = torch.full_like(a, float("nan"))
    assert ctt.tptt_quick_gelu_fwd(_ptr(z32), _ptr(z), _ptr(hz), z32.numel(), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(_bits(z), _bits(a))
    nz = a.float() != 0
    assert torch.equal(_bits(hz)[nz], _bits(h)[nz]) and bool((hz.float()[~nz] == 0).all())
    # and on fp32 values between bf16's: h is quick_gelu of the unrounded value
    g = torch.Generator(device=DEV).manual_seed(17)
    z32 = torch.randn(64, 4096, generator=g, device=DEV) * torch.exp2(torch.linspace(-20, 6, 64, device=DEV))[:, None]
    z32[0, :8] = torch.tensor([-51.0, -52.5, 60.0, 1e30, -1e30, 3.0e-39, -1e-40, 52.2], device=DEV)
    z = torch.empty(64, 4096, dtype=BF, device=DEV)
    hz = torch.empty_like(z)
    assert ctt.tptt_quick_gelu_fwd(_ptr(z32), _ptr(z), _ptr(hz), z32.numel(), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(_bits(z), _bits(z32.bfloat16()))
    _check_quick_gelu(worst, "train_fwd_fp32", z32, hz, BF)


def _colsum_emulated(dz, chunks):
    """quick_gelu_bwd_colsum_kernel's per-chunk row sums (chunk c: rows c per .. c per + per - 1, in order) and colsum_reduce_kernel's
    fixed order (lane j: chunks j, j + 16, ...; then the 16 lanes in order), in fp32, rounded to bf16"""
    rows = dz.shape[0]
    per = (rows + chunks - 1) // chunks
    d = dz.float()
    part = torch.zeros(chunks, dz.shape[1], device=DEV)
    full = torch.zeros(chunks * per, dz.shape[1], device=DEV)
    full[:rows] = d
    full = full.view(chunks, per, -1)
    for r in range(per):
        part = part + full[:, r]
    lanes = torch.zeros(16, dz.shape[1], device=DEV)
    for i in range(0, chunks, 16):
        blk = part[i:i + 16]
        lanes[:blk.shape[0]] = lanes[:blk.shape[0]] + blk
    t = torch.zeros(dz.shape[1], device=DEV)
    for j in range(16):
        t = t + lanes[j]
    return t.bfloat16()


def test_quick_gelu_backward_every_input(ctt, record_property):
    """dz = dh quick_gelu'(z) at every finite bf16 z (16 rows of 4096 with 256 zeros after them) for dh = 1 and powers of two, against
    fp64 within _quick_gelu_grad_ref's bound and one bf16 rounding; ±0 is accepted where |quick_gelu'(z)| < 2^-120 (z < -52.1, where
    __expf overflows and s = 0, as in the forward's flush region).  fc1's bias gradient bit for bit against the fixed-order fp32 sums of
    the stored dz, also over 1200 rows (3 per chunk)."""
    worst = Worst(record_property)
    z = torch.zeros(16 * 4096, dtype=BF, device=DEV)
    z[:65280] = _all_finite(BF).reshape(-1)
    z = z.view(16, 4096)
    part = torch.empty(592 * 4096, device=DEV)
    gp, f_gp = _quick_gelu_grad_ref(z)
    for k in (0, -40, -7, 5, 40):
        s = 2.0 ** k
        dz = torch.full((16, 4096), s, dtype=BF, device=DEV)
        db = torch.empty(4096, dtype=BF, device=DEV)
        assert ctt.tptt_quick_gelu_bwd(_ptr(dz), _ptr(z), 16, _ptr(db), _ptr(part), _stream()) == 0
        torch.cuda.synchronize()
        worst.check("dz", dz, s * gp, UNIT[BF] * s * gp.abs() + (1 + UNIT[BF]) * s * f_gp + SUB[BF], gp.abs() < 2.0 ** -120)
        assert torch.equal(_bits(db), _bits(_colsum_emulated(dz, 16))), k
    g = torch.Generator(device=DEV).manual_seed(23)
    rows = 1200
    zz = z.repeat(75, 1)
    dh = torch.randn(rows, 4096, generator=g, device=DEV).bfloat16()
    dz = dh.clone()
    db = torch.empty(4096, dtype=BF, device=DEV)
    assert ctt.tptt_quick_gelu_bwd(_ptr(dz), _ptr(zz), rows, _ptr(db), _ptr(part), _stream()) == 0
    torch.cuda.synchronize()
    gp, f_gp = _quick_gelu_grad_ref(zz)
    hd = dh.double()
    worst.check("dz_randn", dz, hd * gp, UNIT[BF] * (hd * gp).abs() + (1 + UNIT[BF]) * hd.abs() * (f_gp + 2 * E * gp.abs()) + SUB[BF],
                gp.abs() < 2.0 ** -120)
    assert torch.equal(_bits(db), _bits(_colsum_emulated(dz, 592)))
