"""wgmma GEMM (tp_gemm_bf16 through the C ABI) against a plain PyTorch fp32 reference of the same op."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _assert_close(out, ref):
    """Elementwise: bf16 rounding of the stored result is at most half an ulp = 2^-9 |ref| (gate 2^-8 |ref|), plus a floor of
    2e-4 of the matrix scale for fp32 accumulation-order differences between the two GEMMs (K up to 36864)."""
    err = (out.float() - ref).abs()
    bound = ref.abs() * 2.0 ** -8 + 2e-4 * ref.abs().max()
    worst = (err - bound).max().item()
    assert worst <= 0, (worst, err.max().item(), ref.abs().max().item())


def _ref(a, b, bias, gelu, alpha):
    y = a.float() @ b.float().t()
    if bias is not None:
        y = y + bias.float()
    if gelu:
        y = torch.nn.functional.gelu(y)          # exact erf form
    return y * alpha


@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (128, 256, 64), (256, 256, 128), (128, 128, 1024), (384, 1024, 1024),
                                   (576, 2048, 4096), (144, 4096, 1024), (64, 128, 128), (200, 160, 72), (1000, 5120, 1024),
                                   (36864, 1024, 1024)])
def test_gemm_shapes(m, n, k):
    from tokenpacker_b200.kernels import gemm_bf16
    g = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k)
    a = torch.randn(m, k, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(n, k, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    out = gemm_bf16(a, b)
    ref = _ref(a, b, None, False, 1.0)
    _assert_close(out, ref)


@pytest.mark.parametrize("gelu", [False, True])
def test_gemm_epilogue_bias_gelu_alpha(gelu):
    from tokenpacker_b200.kernels import gemm_bf16
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(300, 1024, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(512, 1024, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    bias = torch.randn(512, device="cuda", generator=g)
    out = gemm_bf16(a, b, bias=bias, gelu=gelu, alpha=0.5)
    ref = _ref(a, b, bias, gelu, 0.5)
    _assert_close(out, ref)


def test_gemm_strided_operands_and_identity():
    """A with a row stride larger than K (the h_kv[:, 1024:] view) and an exactly representable product."""
    from tokenpacker_b200.kernels import gemm_bf16
    big = torch.zeros(256, 2048, device="cuda", dtype=torch.bfloat16)
    big[:, 1024:] = torch.randint(-4, 5, (256, 1024), device="cuda").to(torch.bfloat16)
    eye = torch.eye(1024, device="cuda", dtype=torch.bfloat16)
    out = gemm_bf16(big[:, 1024:], eye)
    assert torch.equal(out, big[:, 1024:])            # A @ I^T == A, bit-exact


def test_gemm_linearity():
    from tokenpacker_b200.kernels import gemm_bf16
    g = torch.Generator(device="cuda").manual_seed(9)
    a = torch.randint(-3, 4, (512, 256), device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randint(-3, 4, (384, 256), device="cuda", generator=g).to(torch.bfloat16)
    # small integers: every product and partial sum is exact in fp32, so the only rounding is the final fp32 -> bf16
    out = gemm_bf16(a, b)
    assert torch.equal(out, (a.float() @ b.float().t()).to(torch.bfloat16))


@pytest.mark.parametrize("m,n,k", [(256, 256, 64), (256, 256, 512), (1024, 1024, 9216), (128, 256, 300), (1024, 4096, 1000), (4096, 1024, 36864)])
def test_gemm_tn_wgrad_form(m, n, k):
    """C = A^T B with row-major [K,M] / [K,N] operands: MN-major UMMA descriptors, contraction over rows (wgrad)."""
    from tokenpacker_b200.kernels import gemm_tn_bf16
    g = torch.Generator(device="cuda").manual_seed(m + n + k)
    a = torch.randn(k, m, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(k, n, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    out = gemm_tn_bf16(a, b)
    ref = a.float().t() @ b.float()
    _assert_close(out, ref)


def test_gemm_tn_exact_small_integers():
    from tokenpacker_b200.kernels import gemm_tn_bf16
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randint(-3, 4, (640, 512), device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randint(-3, 4, (640, 256), device="cuda", generator=g).to(torch.bfloat16)
    assert torch.equal(gemm_tn_bf16(a, b), (a.float().t() @ b.float()).to(torch.bfloat16))


@pytest.mark.parametrize("m,n,k", [(256, 256, 64), (512, 1024, 1024), (1000, 1024, 4096), (9216, 4096, 4096), (300, 256, 200)])
def test_gemm_nn_dgrad_form(m, n, k):
    """C = A B with B a row-major [K,N] matrix (a weight as stored): K-major A tiles, MN-major B tiles, no transposed copy (dgrad)."""
    from tokenpacker_b200.kernels import gemm_nn_bf16
    g = torch.Generator(device="cuda").manual_seed(m + n + k + 1)
    a = torch.randn(m, k, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(k, n, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    out = gemm_nn_bf16(a, b, alpha=0.5)
    ref = 0.5 * (a.float() @ b.float())
    _assert_close(out, ref)


def test_gemm_nn_exact_small_integers():
    from tokenpacker_b200.kernels import gemm_nn_bf16
    g = torch.Generator(device="cuda").manual_seed(4)
    a = torch.randint(-3, 4, (384, 640), device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randint(-3, 4, (640, 512), device="cuda", generator=g).to(torch.bfloat16)
    assert torch.equal(gemm_nn_bf16(a, b), (a.float() @ b.float()).to(torch.bfloat16))
