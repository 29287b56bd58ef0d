"""The pair kernel's fragment-direct epilogue (tiles stored through the TMA slabs: every value computed where the wgmma fragment holds
it, 16-bit values written to the slabs with stmatrix, row statistics re-read from the slabs) against the one-CTA kernel, whose epilogue
turns the fragments into one-row-per-thread form through shared memory: for every epilogue kind both store the same bits.

Items and their NaN-sentinel output frames are those of tests/test_gemm_engine_gpu.py.  The pair kernel takes plain-form items
only at N % 256 == 0 (narrower N runs on the one-CTA kernels alone), so N sweeps 256, 512 and 1024; M sweeps a single row, ragged
row tiles and 36864 + 64 rows (the benchmarked batch's token count and a partial last row tile).  Window-major row statistics exist
only inside the fused forward and are checked by tests/test_forward_stages_gpu.py.

The CLIP tower's instantiations (bias, bf16 / f16 / fp32 residual, quick_gelu, alpha, f16 output, the patch GEMM's segmented store) go
through the same comparison with the tower's own test hooks (tpc_gemm_resid, tpc_gemm_f16), from one row to the 64-crop batch's token
count plus a partial row tile, at the tower's widths N = 1024 and 4096.
"""
import ctypes as C

import pytest
import torch

from test_clip_tower_forward_stages_gpu import F16, _lib, _ptr, i32, i64, p
from test_gemm_engine_gpu import BF, GUARD, ONE_256, PAIR, Item, _bits, _run, _same_bits, hk  # noqa: F401  (hk: fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

KINDS = {
    "bias": dict(bias=True),
    "bias_gelu": dict(bias=True, gelu=True),
    "alpha_half": dict(bias=True, alpha=0.5),
    "gelu_alpha_half": dict(bias=True, gelu=True, alpha=0.5),
    "gelu_alpha_m3": dict(bias=True, gelu=True, alpha=-3.0),
    "no_bias": dict(),
    "ln_fold": dict(bias=True, ln=True),
    "ln_fold_gelu": dict(bias=True, ln=True, gelu=True),
    "stats": dict(bias=True, gelu=True, stats=True),
    "ln_fold_stats": dict(bias=True, ln=True, stats=True),
}
SHAPES = [(1, 256, 384), (129, 512, 256), (300, 1024, 640), (36864 + 64, 1024, 256)]


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("kind", list(KINDS))
def test_pair_epilogue_same_bits_as_one_cta(hk, kind, m, n, k):
    """C (and the row-statistics slots) of the pair kernel equal the one-CTA kernel's bit for bit; guards keep their sentinels."""
    it = Item(0, m, n, k, seed=101 + m + n + k, **KINDS[kind])
    _run(hk, [it], mode="1", expect=ONE_256)
    one = it.snapshot()
    it.check_guards()
    it.reset()
    _run(hk, [it], mode="2", expect=PAIR)
    it.check_guards()
    assert _same_bits(it.snapshot(), one)


DUAL_WITH = {"plain": dict(), "ln_fold": dict(ln=True), "stats": dict(stats=True), "ln_fold_stats": dict(ln=True, stats=True)}


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("alpha", [1.0, 0.5, -3.0])
@pytest.mark.parametrize("with_", list(DUAL_WITH))
def test_pair_dual_same_bits_as_one_cta(hk, record_property, with_, alpha, m, n, k):
    """dual (pair kernel only), alone and with the LayerNorm fold and / or row statistics: the pre-activation output equals the
    one-CTA kernel's result without GELU and alpha, the activation output and the statistics slots its result with them, bit for bit,
    from the same operands; all of them also hold their fp64 bounds."""
    seed = 211 + m + n + k
    kw = DUAL_WITH[with_]
    dual = Item(0, m, n, k, seed=seed, bias=True, gelu=True, alpha=alpha, dual=True, **kw)
    _run(hk, [dual], expect=PAIR)
    dual.check(record_property, f"dual_{with_}")
    act = Item(0, m, n, k, seed=seed, bias=True, gelu=True, alpha=alpha, **kw)
    pre = Item(0, m, n, k, seed=seed, bias=True, ln=kw.get("ln", False))
    for ref in (act, pre):
        _run(hk, [ref], mode="1", expect=ONE_256)
        ref.check_guards()
    assert act.bt.equal(dual.bt) and act.at.equal(dual.at) and pre.at.equal(dual.at)
    assert _bits(dual.c().contiguous()).equal(_bits(act.c().contiguous()))
    assert dual.pre.dtype == BF
    assert _bits(dual.pre[GUARD:GUARD + m, :n].contiguous()).equal(_bits(pre.c().contiguous()))
    if dual.stats:
        assert _bits(dual.st).equal(_bits(act.st))


@pytest.mark.parametrize("kind", ["bias", "ln_fold"])
def test_pair_unaligned_column_vectors(hk, kind):
    """Column vectors whose address is not 16-byte aligned (4-byte copies instead of 16-byte ones) give the same bits as the
    one-CTA kernel."""
    it = Item(0, 300, 512, 256, seed=307, **KINDS[kind])
    keep = []
    for name in ("bias", "col_a"):
        v = getattr(it, name, None)
        if v is not None:
            buf = torch.empty(v.numel() + 1, dtype=v.dtype, device=v.device)
            buf[1:] = v
            keep.append(buf)
            setattr(it.desc, name, buf[1:].data_ptr())
            assert buf[1:].data_ptr() % 16 != 0
    _run(hk, [it], mode="1", expect=ONE_256)
    one = it.snapshot()
    it.reset()
    _run(hk, [it], mode="2", expect=PAIR)
    it.check_guards()
    assert _same_bits(it.snapshot(), one)


TOWER_KINDS = {
    "bf16_bias_resid": dict(dtype=BF, bias=True, resid="x"),
    "bf16_bias_resid_f32": dict(dtype=BF, bias=True, resid="f32"),
    "bf16_quick_gelu": dict(dtype=BF, bias=True, gelu=2),
    "bf16_quick_gelu_no_bias": dict(dtype=BF, gelu=2),
    "f16_bias_resid": dict(dtype=F16, bias=True, resid="x"),
    "f16_bias_resid_f32": dict(dtype=F16, bias=True, resid="f32"),
    "f16_quick_gelu": dict(dtype=F16, bias=True, gelu=2),
    "f16_quick_gelu_no_bias": dict(dtype=F16, gelu=2),
    "f16_bias_alpha": dict(dtype=F16, bias=True, alpha=0.125),
    "f16_patch_store": dict(dtype=F16, seg=(576, 577)),
}
TOWER_SHAPES = [(m, n) for m in (1, 129, 1731, 36864 + 64) for n in (1024, 4096)]
PATCH_SHAPES = [(576 * crops, n) for crops in (1, 3, 64) for n in (1024, 4096)]     # the patch GEMM's rows are whole crops
TOWER_CASES = [(kind, m, n) for kind, kw in TOWER_KINDS.items() for m, n in (PATCH_SHAPES if "seg" in kw else TOWER_SHAPES)]


@pytest.fixture(scope="module")
def ct():
    return _lib("libtokenpacker_b200_clip_tower_hooks.so", {
        "tpc_gemm_resid": [p, i64, p, i64, p, i64, i64, i64, i64, p, p, i64, i32, i32, i32, p]})


@pytest.fixture(scope="module")
def ct16():
    return _lib("libtokenpacker_b200_clip_tower_f16_hooks.so", {
        "tpc_gemm_f16": [p, i64, p, i64, p, i64, i64, i64, i64, p, p, i64, i32, i32, i32, C.c_float, i32, i32, i32, p]})


def _tower_gemm(ct, ct16, kw, a, b, bias, r, m, n, k, mode):
    """C of tpc_gemm_resid / tpc_gemm_f16 in a NaN frame of GUARD rows above and below and 64 columns to the right: returns the frame"""
    dtype = kw["dtype"]
    seg_len, seg_stride = kw.get("seg", (0, 0))
    rows = m if seg_len == 0 else m // seg_len * seg_stride
    frame = torch.full((rows + 2 * GUARD, n + 64), float("nan"), dtype=dtype, device=DEV)
    c = frame[GUARD:GUARD + rows, :n]
    ldr, resid_f32 = (0, 0) if r is None else (r.stride(0), int(r.dtype == torch.float32))
    gelu = kw.get("gelu", 0)
    if dtype == BF:
        st = ct.tpc_gemm_resid(_ptr(a), k, _ptr(b), k, _ptr(c), n + 64, m, n, k, _ptr(bias), _ptr(r), ldr, resid_f32, gelu, mode, None)
    else:
        st = ct16.tpc_gemm_f16(_ptr(a), k, _ptr(b), k, _ptr(c), n + 64, m, n, k, _ptr(bias), _ptr(r), ldr, resid_f32, gelu, 0,
                               kw.get("alpha", 1.0), seg_len, seg_stride, mode, None)
    assert st == 0
    torch.cuda.synchronize()
    guards = [frame[:GUARD], frame[GUARD + rows:], frame[:, n:]]
    if seg_len != 0:
        guards.append(c.view(m // seg_len, seg_stride, n)[:, seg_len:])      # the rows between the segments are never written
    assert all(bool(torch.isnan(x.float()).all()) for x in guards)
    return frame


@pytest.mark.parametrize("kind,m,n", TOWER_CASES)
def test_tower_epilogue_same_bits_as_one_cta(ct, ct16, kind, m, n):
    """The tower's epilogue kinds on the pair kernel (slabs written from the wgmma fragments) store the one-CTA kernel's bits, NaN
    guards included.  The residual's row stride is wider than N."""
    kw = TOWER_KINDS[kind]
    dtype, k = kw["dtype"], 320
    g = torch.Generator(device=DEV).manual_seed(401 + m + n)
    a = torch.randn(m, k, generator=g, device=DEV).to(dtype)
    b = (torch.randn(n, k, generator=g, device=DEV) * 0.05).to(dtype)
    bias = torch.randn(n, generator=g, device=DEV) if kw.get("bias") else None
    r = None
    if "resid" in kw:
        r = torch.randn(m, n + 8, generator=g, device=DEV) * 4
        r = (r if kw["resid"] == "f32" else r.to(dtype))[:, :n]
    one, pair = (_tower_gemm(ct, ct16, kw, a, b, bias, r, m, n, k, mode) for mode in (1, 2))
    assert pair.view(torch.int16).equal(one.view(torch.int16)), "one-CTA and pair kernels differ"
