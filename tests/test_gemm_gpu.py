"""wgmma GEMM (tp_gemm_bf16 / tp_gemm_tn_bf16 / tp_gemm_nn_bf16 through the C ABI) against float64 products of the same bf16
operands.  The plain A . B^T cases run on every kernel the form allows: the one-CTA kernels (TP_GEMM_MODE=1), the CTA-pair
kernel (=2, where N % 256 == 0) and the cost-based choice; the TN / NN forms exist on the pair kernel only."""
import contextlib
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

E = 2.0 ** -24            # fp32 unit roundoff
U = 2.0 ** -8             # bf16 unit roundoff
F64 = torch.float64


@contextlib.contextmanager
def _mode(mode):
    """TP_GEMM_MODE for the calls inside (read per call); None: the cost-based choice"""
    old = os.environ.get("TP_GEMM_MODE")
    if mode is None:
        os.environ.pop("TP_GEMM_MODE", None)
    else:
        os.environ["TP_GEMM_MODE"] = mode
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("TP_GEMM_MODE", None)
        else:
            os.environ["TP_GEMM_MODE"] = old


def _modes(n):
    """every kernel choice the plain form allows at this N"""
    return ["1", None] + (["2"] if n % 256 == 0 else [])


def _assert_close(out, ref, floor):
    """Elementwise |out - ref| <= U |ref| + (1 + U) floor: the bf16 rounding of the stored result is within U = 2^-8 of the value it
    rounds, and floor bounds the kernel's fp32 error in that value (derived from the arithmetic, see _ref)."""
    err = (out.to(F64) - ref).abs()
    bound = U * ref.abs() + (1 + U) * floor
    ratio = float((err / bound.clamp_min(1e-300)).max())
    assert torch.isfinite(out).all() and ratio <= 1.0, (ratio, err.max().item(), ref.abs().max().item())


def _ref(a, b, bias, gelu, alpha):
    """fp64 alpha GELU(a b^T + bias) and its floor: (K + 1) E sum|a||b| for the fp32 accumulation, one rounding for the bias add,
    GELU's derivative bound 1.13 plus the 1e-6 |z| of its erf approximation, one rounding for alpha"""
    ad, bd = a.to(F64), b.to(F64)
    y = ad @ bd.t()
    f = (a.shape[1] + 1) * E * (ad.abs() @ bd.abs().t())
    if bias is not None:
        y = y + bias.to(F64)
    f = f + E * y.abs()
    if gelu:
        z = y
        y = torch.nn.functional.gelu(z)          # exact erf form
        f = 1.13 * f + 1e-6 * z.abs() + 4 * E * y.abs() + 2.0 ** -133
    if alpha != 1.0:
        y = y * alpha
        f = abs(alpha) * f + E * y.abs()
    return y, f


@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (128, 256, 64), (256, 256, 128), (128, 128, 1024), (384, 1024, 1024),
                                   (576, 2048, 4096), (144, 4096, 1024), (64, 128, 128), (200, 160, 72), (1000, 5120, 1024),
                                   (36864, 1024, 1024)])
def test_gemm_shapes(m, n, k):
    from tokenpacker_b200.kernels import gemm_bf16
    g = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k)
    a = torch.randn(m, k, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    ref, floor = _ref(a, b, None, False, 1.0)
    for mode in _modes(n):
        with _mode(mode):
            out = gemm_bf16(a, b)
        _assert_close(out, ref, floor)


@pytest.mark.parametrize("gelu", [False, True])
def test_gemm_epilogue_bias_gelu_alpha(gelu):
    from tokenpacker_b200.kernels import gemm_bf16
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(300, 1024, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(512, 1024, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    bias = torch.randn(512, device="cuda", generator=g)
    ref, floor = _ref(a, b, bias, gelu, 0.5)
    for mode in _modes(512):
        with _mode(mode):
            out = gemm_bf16(a, b, bias=bias, gelu=gelu, alpha=0.5)
        _assert_close(out, ref, floor)


def test_gemm_strided_operands_and_identity():
    """A with a row stride larger than K (the h_kv[:, 1024:] view) and an exactly representable product."""
    from tokenpacker_b200.kernels import gemm_bf16
    big = torch.zeros(256, 2048, device="cuda", dtype=torch.bfloat16)
    big[:, 1024:] = torch.randint(-4, 5, (256, 1024), device="cuda").to(torch.bfloat16)
    eye = torch.eye(1024, device="cuda", dtype=torch.bfloat16)
    for mode in _modes(1024):
        with _mode(mode):
            out = gemm_bf16(big[:, 1024:], eye)
        assert torch.equal(out, big[:, 1024:])        # A @ I^T == A, bit-exact


def test_gemm_linearity():
    """Small integers: every product and partial sum is exact in fp32 (9 K < 2^24), so the only rounding is the final fp32 -> bf16,
    also at K = 36864, where the derived bound of the random-operand cases is loose and only this exactness sees a lost k-block."""
    from tokenpacker_b200.kernels import gemm_bf16
    g = torch.Generator(device="cuda").manual_seed(9)
    for m, n, k in ((512, 384, 256), (257, 512, 36864)):
        a = torch.randint(-3, 4, (m, k), device="cuda", generator=g).to(torch.bfloat16)
        b = torch.randint(-3, 4, (n, k), device="cuda", generator=g).to(torch.bfloat16)
        exact = (a.to(F64) @ b.to(F64).t()).to(torch.bfloat16)
        for mode in _modes(n):
            with _mode(mode):
                out = gemm_bf16(a, b)
            assert torch.equal(out, exact), (m, n, k, mode)


@pytest.mark.parametrize("m,n,k", [(256, 256, 64), (256, 256, 512), (1024, 1024, 9216), (128, 256, 300), (1024, 4096, 1000), (4096, 1024, 36864)])
def test_gemm_tn_wgrad_form(m, n, k):
    """C = A^T B with row-major [K,M] / [K,N] operands: MN-major UMMA descriptors, contraction over rows (wgrad)."""
    from tokenpacker_b200.kernels import gemm_tn_bf16
    g = torch.Generator(device="cuda").manual_seed(m + n + k)
    a = torch.randn(k, m, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(k, n, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    out = gemm_tn_bf16(a, b)
    ref, floor = _ref(a.t(), b.t(), None, False, 1.0)
    _assert_close(out, ref, floor)


def test_gemm_tn_exact_small_integers():
    """exact fp32 sums (see test_gemm_linearity), also over the 36864 rows of the largest wgrad case"""
    from tokenpacker_b200.kernels import gemm_tn_bf16
    g = torch.Generator(device="cuda").manual_seed(3)
    for m, n, k in ((512, 256, 640), (512, 1024, 36864)):
        a = torch.randint(-3, 4, (k, m), device="cuda", generator=g).to(torch.bfloat16)
        b = torch.randint(-3, 4, (k, n), device="cuda", generator=g).to(torch.bfloat16)
        assert torch.equal(gemm_tn_bf16(a, b), (a.to(F64).t() @ b.to(F64)).to(torch.bfloat16)), (m, n, k)


@pytest.mark.parametrize("m,n,k", [(256, 256, 64), (512, 1024, 1024), (1000, 1024, 4096), (9216, 4096, 4096), (300, 256, 200)])
def test_gemm_nn_dgrad_form(m, n, k):
    """C = A B with B a row-major [K,N] matrix (a weight as stored): K-major A tiles, MN-major B tiles, no transposed copy (dgrad)."""
    from tokenpacker_b200.kernels import gemm_nn_bf16
    g = torch.Generator(device="cuda").manual_seed(m + n + k + 1)
    a = torch.randn(m, k, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(k, n, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    out = gemm_nn_bf16(a, b, alpha=0.5)
    ref, floor = _ref(a, b.t(), None, False, 0.5)
    _assert_close(out, ref, floor)


def test_gemm_nn_exact_small_integers():
    """exact fp32 sums (see test_gemm_linearity), also at K = 36864"""
    from tokenpacker_b200.kernels import gemm_nn_bf16
    g = torch.Generator(device="cuda").manual_seed(4)
    for m, n, k in ((384, 512, 640), (300, 512, 36864)):
        a = torch.randint(-3, 4, (m, k), device="cuda", generator=g).to(torch.bfloat16)
        b = torch.randint(-3, 4, (k, n), device="cuda", generator=g).to(torch.bfloat16)
        assert torch.equal(gemm_nn_bf16(a, b), (a.to(F64) @ b.to(F64)).to(torch.bfloat16)), (m, n, k)
