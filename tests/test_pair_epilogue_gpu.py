"""The pair kernel's fragment-direct epilogue (tiles stored through the TMA slabs: every value computed where the wgmma fragment holds
it, bf16 written to the slabs with stmatrix, row statistics re-read from the slabs) against the one-CTA kernel, whose epilogue still
turns the fragments into one-row-per-thread form through shared memory: for every epilogue kind both store the same bits.

Items and their NaN-sentinel output frames are those of tests/test_gemm_engine_gpu.py.  The pair kernel takes plain-form items
only at N % 256 == 0 (narrower N runs on the one-CTA kernels alone), so N sweeps 256, 512 and 1024; M sweeps a single row, ragged
row tiles and 36864 + 64 rows (the benchmarked batch's token count and a partial last row tile).  Window-major row statistics exist
only inside the fused forward and are checked by tests/test_forward_stages_gpu.py.
"""
import pytest
import torch

from test_gemm_engine_gpu import BF, GUARD, ONE_256, PAIR, Item, _bits, _run, _same_bits, hk  # noqa: F401  (hk: fixture)

pytestmark = pytest.mark.gpu

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
