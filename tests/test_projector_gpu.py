"""Parity of the CUDA projector (through the nn.Module -> C ABI -> sm_90a kernels) with the oracle and the
reference-generated golden fixtures.  Tolerances (stated per SURVEY.md §8c): bf16 storage / fp32 accumulation vs the
fp32|fp64 oracle on identical bf16-rounded weights and inputs: rel-RMS <= 4e-3 and max-abs <= 5e-3 (measured on an H100: 2.0e-3 / 1.3e-3 at
hidden 256; the error grows with the width of the last two linears) at output
RMS ~0.1 (the reference's own bf16-vs-fp32 gap at these inputs is rel-RMS 4.6e-3..5.3e-3, max-abs up to 4.9e-3)."""
import os

import numpy as np
import pytest
import torch

from oracle import tokenpacker_oracle as tpo

pytestmark = pytest.mark.gpu

REL_RMS_TOL = 4e-3
MAX_ABS_TOL = 5e-3


def make_module(hidden, s, seed):
    from tokenpacker_b200 import TokenPackerB200
    params = {k: tpo.round_bf16(v) for k, v in tpo.make_params(hidden, seed=seed).items()}
    m = TokenPackerB200(hidden_size=hidden, scale_factor=s)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    return m.to(device="cuda", dtype=torch.bfloat16).eval(), params


def errors(out, ref):
    out = out.astype(np.float64)
    ref = ref.astype(np.float64)
    rms = np.sqrt((ref ** 2).mean())
    return float(np.sqrt(((out - ref) ** 2).mean()) / rms), float(np.abs(out - ref).max())


@pytest.mark.parametrize("s", [2, 3, 4, 1, 6, 8, 12, 24])       # 2/3/4: released models; the rest: the other divisors of 24
def test_against_oracle_small_hidden(s):
    hidden, n = 128, 3
    m, params = make_module(hidden, s, seed=100 + s)
    x0, xm = tpo.make_inputs(n, seed=200 + s)
    x0, xm = tpo.round_bf16(x0), tpo.round_bf16(xm)
    ref = tpo.tokenpacker_forward(params, x0, xm, s)
    with torch.no_grad():
        out = m((torch.from_numpy(x0).cuda().bfloat16(), torch.from_numpy(xm).cuda().bfloat16()))
    assert out.shape == (n, (24 // s) ** 2, hidden) and out.dtype == torch.bfloat16 and out.is_contiguous()
    rel, mx = errors(out.float().cpu().numpy(), ref)
    assert rel <= REL_RMS_TOL and mx <= MAX_ABS_TOL, (rel, mx)


@pytest.mark.parametrize("s", [2, 3, 4])
def test_against_reference_golden_full_width(golden_dir, s):
    """hidden=4096, N=1: the committed fixture is the REFERENCE module's fp32 output on these bf16-rounded tensors."""
    g = np.load(os.path.join(golden_dir, f"projector_s{s}_h4096_bf16in.npz"))
    m, _ = make_module(4096, s, seed=int(g["param_seed"]))
    x0, xm = tpo.make_inputs(1, seed=int(g["input_seed"]))
    x0, xm = tpo.round_bf16(x0), tpo.round_bf16(xm)
    with torch.no_grad():
        out = m((torch.from_numpy(x0).cuda().bfloat16(), torch.from_numpy(xm).cuda().bfloat16())).float().cpu().numpy()
    sub = out[0, ::int(g["row_stride"]), ::int(g["col_stride"])]
    rel, mx = errors(sub, g["out_sub"])
    assert rel <= REL_RMS_TOL and mx <= MAX_ABS_TOL, (rel, mx)
    assert abs(float(np.sqrt((out.astype(np.float64) ** 2).mean())) - float(g["out_rms"])) < 2e-3 * float(g["out_rms"]) + 1e-4


@pytest.mark.parametrize("s", [1, 6, 8, 12, 24])
def test_against_reference_golden_other_scale_factors(golden_dir, s):
    """The scale factors no released model uses but the reference constructor accepts (builder.py:51-52): streamed-window
    attention kernel, generic point-query stencil; fixture = the REFERENCE module's fp32 output (fp32 weights and inputs, so the
    gap includes the bf16 rounding of both: the reference's own bf16 gap, see the header)."""
    g = np.load(os.path.join(golden_dir, f"projector_s{s}_h128.npz"))
    hidden, n = int(g["hidden"]), int(g["n"])
    from tokenpacker_b200 import TokenPackerB200
    params = tpo.make_params(hidden, seed=int(g["param_seed"]))
    m = TokenPackerB200(hidden_size=hidden, scale_factor=s)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    x0, xm = tpo.make_inputs(n, seed=int(g["input_seed"]))
    with torch.no_grad():
        out = m((torch.from_numpy(x0).cuda().bfloat16(), torch.from_numpy(xm).cuda().bfloat16()))
    assert out.shape == (n, (24 // s) ** 2, hidden)
    rel, mx = errors(out.float().cpu().numpy(), g["out"])
    assert rel <= 1.2e-2 and mx <= 2e-2, (rel, mx)


def test_batch_invariance_and_strided_views():
    """Crops are independent: row n of a batched call equals the single-crop call bit for bit, and the [:,1:]
    views CLIPVisionTower hands over in training (crop stride 577*C) give the same bits as contiguous copies."""
    s, hidden, n = 2, 256, 5
    m, _ = make_module(hidden, s, seed=7)
    g = torch.Generator(device="cuda").manual_seed(3)
    full0 = torch.randn(n, 577, 1024, device="cuda", generator=g).bfloat16()
    fullm = torch.randn(n, 577, 4096, device="cuda", generator=g).bfloat16()
    v0, vm = full0[:, 1:], fullm[:, 1:]
    assert not v0.is_contiguous()
    with torch.no_grad():
        a = m((v0, vm))
        b = m((v0.contiguous(), vm.contiguous()))
        c = m((v0[2:3].contiguous(), vm[2:3].contiguous()))
    assert torch.equal(a, b)
    assert torch.equal(a[2:3], c)


def test_window_locality_full_size():
    """Size-independent property at BASELINE configs[1] scale (N=64, s=2, H=4096): perturbing one fine token of one
    crop changes exactly one output row of that crop."""
    s, hidden, n = 2, 4096, 64
    m, _ = make_module(hidden, s, seed=0)
    g = torch.Generator(device="cuda").manual_seed(11)
    x0 = torch.randn(n, 576, 1024, device="cuda", generator=g).bfloat16()
    xm = torch.randn(n, 576, 4096, device="cuda", generator=g).bfloat16()
    with torch.no_grad():
        base = m((x0, xm))
        xm2 = xm.clone()
        crop, tok = 37, 5 * 24 + 9                       # fine token (5, 9) -> query (2, 4) -> row 2*12+4 = 28
        xm2[crop, tok] += 1.0
        pert = m((x0, xm2))
    assert torch.isfinite(base).all()
    diff = (pert.float() - base.float()).abs().amax(dim=-1)        # [N, M]
    changed = diff > 0
    assert changed[crop, 28] and int(changed.sum()) == 1
    # x0 only feeds the queries: changing token (5,9) of x0 changes query 28 only (s=2 stencil covers its window)
    with torch.no_grad():
        x02 = x0.clone()
        x02[crop, tok] += 1.0
        pert = m((x02, xm))
    changed = (pert.float() - base.float()).abs().amax(dim=-1) > 0
    assert changed[crop, 28] and int(changed.sum()) == 1


def test_weight_cache_invalidation():
    s, hidden = 4, 128
    m, _ = make_module(hidden, s, seed=1)
    g = torch.Generator(device="cuda").manual_seed(2)
    x0 = torch.randn(2, 576, 1024, device="cuda", generator=g).bfloat16()
    xm = torch.randn(2, 576, 4096, device="cuda", generator=g).bfloat16()
    with torch.no_grad():
        a = m((x0, xm))
        m.mlp[2].bias.add_(1.0)
        b = m((x0, xm))
    assert (b.float() - a.float() - 1.0).abs().max().item() < 2e-2


def test_dtype_roundtrip_and_errors():
    s, hidden = 3, 128
    m, _ = make_module(hidden, s, seed=1)
    x0 = torch.randn(1, 576, 1024, device="cuda")
    xm = torch.randn(1, 576, 4096, device="cuda")
    with torch.no_grad():
        out16 = m((x0.half(), xm.half()))
    assert out16.dtype == torch.float16 and out16.shape == (1, 64, hidden)
    with pytest.raises(ValueError):
        m((x0[:, :100].bfloat16(), xm.bfloat16()))
    with pytest.raises(NotImplementedError):
        m((x0.bfloat16().requires_grad_(True), xm.bfloat16()))     # gradients w.r.t. the CLIP features are not provided


def test_kernel_variants_agree_bitwise(monkeypatch):
    """The one-CTA (cta_group::1) and CTA-pair (cta_group::2, grouped or not) GEMM kernels are interchangeable bit for bit
    through the whole forward (explicit-intrinsic epilogue math), so the automatic size-based selection cannot make a
    crop's result depend on how many crops share its call."""
    s, hidden, n = 4, 256, 10
    monkeypatch.setenv("TP_FUSE_ATTN", "0")          # this test is about the GEMM kernels: keep the attention core a kernel of its own
    m, _ = make_module(hidden, s, seed=3)
    g = torch.Generator(device="cuda").manual_seed(7)
    x0 = torch.randn(n, 576, 1024, device="cuda", generator=g).bfloat16()
    xm = torch.randn(n, 576, 4096, device="cuda", generator=g).bfloat16()
    outs = {}
    with torch.no_grad():
        for mode in ("0", "1", "2", "3"):
            monkeypatch.setenv("TP_GEMM_MODE", mode)
            outs[mode] = m((x0, xm)).clone()
            outs["half" + mode] = m((x0[5:], xm[5:])).clone()
    for mode in ("1", "2", "3"):
        assert torch.equal(outs["0"], outs[mode]), mode
        assert torch.equal(outs["0"][5:], outs["half" + mode]), mode
    assert torch.equal(outs["0"][5:], outs["half0"])       # Q=180 (one-CTA kernels) vs Q=360 (pair kernels) under auto selection


@pytest.mark.parametrize("s,hidden,n", [(2, 256, 5), (4, 512, 9), (2, 4096, 3)])
def test_fused_single_launch_vs_separate_kernels(s, hidden, n, monkeypatch):
    """scale_factor 2 / 4 with hidden % 256 == 0 run as ONE persistent launch (window-major y_k / y_v, K/V in-projections fused with
    the window attention: k', v' stay in fp32 registers).  TP_FUSE_ATTN=0 / TP_CHAIN=0 select the separate-kernel plans: same
    math, k' / v' additionally rounded to bf16 — the two must agree to rounding, and each must meet the oracle gate; the fused
    plan must not depend on the batch (row n of a batched call == the single-crop call, bit for bit)."""
    from tokenpacker_b200._lib import lib
    m, params = make_module(hidden, s, seed=21)
    x0, xm = tpo.make_inputs(n, seed=22)
    x0, xm = tpo.round_bf16(x0), tpo.round_bf16(xm)
    ref = tpo.tokenpacker_forward(params, x0, xm, s, dtype=np.float32)
    t0, tm = torch.from_numpy(x0).cuda().bfloat16(), torch.from_numpy(xm).cuda().bfloat16()
    with torch.no_grad():
        m((t0, tm))                                                 # first call packs the weights (its own launches)
        l0 = lib.tp_launch_count()
        fused = m((t0, tm)).clone()
        assert lib.tp_launch_count() - l0 == 1                      # the whole forward is one kernel
        single = m((t0[n - 1:], tm[n - 1:])).clone()
        monkeypatch.setenv("TP_FUSE_ATTN", "0")
        chained = m((t0, tm)).clone()
        monkeypatch.setenv("TP_CHAIN", "0")
        l0 = lib.tp_launch_count()
        plain = m((t0, tm)).clone()
        assert lib.tp_launch_count() - l0 >= 7                      # [S] + 5 GEMM stages + attention, one launch each (or more)
    assert torch.equal(fused[n - 1:], single)
    assert torch.equal(chained, plain)                              # chaining changes scheduling, never bits
    for name, out in (("fused", fused), ("plain", plain)):
        rel, mx = errors(out.float().cpu().numpy(), ref)
        assert rel <= REL_RMS_TOL and mx <= MAX_ABS_TOL, (name, rel, mx)
    d = (fused.float() - plain.float())
    # the two plans differ by the bf16 rounding of k' / v' (and the summation order inside a window)
    assert float(d.pow(2).mean().sqrt() / plain.float().pow(2).mean().sqrt()) < 4e-3


@pytest.mark.parametrize("n,s,hidden", [(1, 2, 5120), (3, 3, 5120), (7, 4, 4096)])
def test_other_shapes_against_oracle(n, s, hidden):
    """13B hidden size (5120 = 20 x 256), odd crop counts, single crop: M/N tails of every kernel."""
    m, params = make_module(hidden, s, seed=11)
    x0, xm = tpo.make_inputs(n, seed=12)
    x0, xm = tpo.round_bf16(x0), tpo.round_bf16(xm)
    ref = tpo.tokenpacker_forward(params, x0, xm, s, dtype=np.float32)
    with torch.no_grad():
        out = m((torch.from_numpy(x0).cuda().bfloat16(), torch.from_numpy(xm).cuda().bfloat16()))
    assert out.shape == (n, (24 // s) ** 2, hidden)
    rel, mx = errors(out.float().cpu().numpy(), ref)
    assert rel <= REL_RMS_TOL and mx <= MAX_ABS_TOL, (rel, mx)


def test_empty_batch_and_bad_inputs():
    m, _ = make_module(128, 2, seed=1)
    with torch.no_grad():
        out = m((torch.zeros(0, 576, 1024, device="cuda", dtype=torch.bfloat16), torch.zeros(0, 576, 4096, device="cuda", dtype=torch.bfloat16)))
    assert out.shape == (0, 144, 128)
    with pytest.raises(TypeError):
        m(torch.zeros(1, 576, 1024, device="cuda"))
    with pytest.raises(ValueError):
        with torch.no_grad():
            m((torch.zeros(2, 576, 1024, device="cuda"), torch.zeros(3, 576, 4096, device="cuda")))


def test_full_size_sweep_properties():
    """BASELINE configs[2] sizes (batch 128, s in {2,3,4}, H=4096): finite, deterministic, and every crop equals its own
    single-crop forward (checked on 3 crops) — size-independent properties where the oracle would take minutes."""
    for s in (2, 3, 4):
        m, _ = make_module(4096, s, seed=0)
        g = torch.Generator(device="cuda").manual_seed(100 + s)
        x0 = torch.randn(128, 576, 1024, device="cuda", generator=g).bfloat16()
        xm = torch.randn(128, 576, 4096, device="cuda", generator=g).bfloat16()
        with torch.no_grad():
            a = m((x0, xm))
            b = m((x0, xm))
            assert torch.isfinite(a).all() and torch.equal(a, b)
            for c in (0, 77, 127):
                assert torch.equal(a[c:c + 1], m((x0[c:c + 1], xm[c:c + 1])))
        del m


def test_cuda_graph_capture_and_replay():
    """Serving path: the 7-launch forward (PDL launches, TMA tensor maps baked into kernel parameters) is capturable in a CUDA
    graph; replays on new inputs match eager execution bit for bit."""
    s, hidden, n = 2, 4096, 2
    m, _ = make_module(hidden, s, seed=0)
    g = torch.Generator(device="cuda").manual_seed(5)
    sx0 = torch.randn(n, 576, 1024, device="cuda", generator=g).bfloat16()
    sxm = torch.randn(n, 576, 4096, device="cuda", generator=g).bfloat16()
    with torch.no_grad():
        m((sx0, sxm))                                   # packs the weights outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            sout = m((sx0, sxm))
        for seed in (11, 12):
            g2 = torch.Generator(device="cuda").manual_seed(seed)
            x0 = torch.randn(n, 576, 1024, device="cuda", generator=g2).bfloat16()
            xm = torch.randn(n, 576, 4096, device="cuda", generator=g2).bfloat16()
            sx0.copy_(x0)
            sxm.copy_(xm)
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(sout, m((x0, xm)))


def test_randomised_configurations_against_oracle():
    """Seeded sweep over crop counts, scale factors, hidden sizes, input scales and memory layouts (contiguous / [:,1:] views)."""
    rng = np.random.default_rng(2024)
    for trial in range(10):
        n = int(rng.integers(1, 10))
        s = int(rng.choice([2, 3, 4]))
        hidden = int(rng.choice([128, 256, 384, 512]))
        scale = float(rng.choice([0.3, 1.0, 2.5]))
        m, params = make_module(hidden, s, seed=1000 + trial)
        x0 = tpo.round_bf16(rng.standard_normal((n, 577, 1024)).astype(np.float32) * scale)
        xm = tpo.round_bf16(rng.standard_normal((n, 577, 4096)).astype(np.float32) * scale)
        t0, tm = torch.from_numpy(x0).cuda().bfloat16(), torch.from_numpy(xm).cuda().bfloat16()
        v0, vm = (t0[:, 1:], tm[:, 1:]) if trial % 2 == 0 else (t0[:, 1:].contiguous(), tm[:, 1:].contiguous())
        ref = tpo.tokenpacker_forward(params, x0[:, 1:], xm[:, 1:], s, dtype=np.float32)
        with torch.no_grad():
            out = m((v0, vm)).float().cpu().numpy()
        rel, mx = errors(out, ref)
        rms = float(np.sqrt((ref.astype(np.float64) ** 2).mean()))
        assert rel <= REL_RMS_TOL and mx <= MAX_ABS_TOL * max(1.0, rms / 0.1), (trial, n, s, hidden, scale, rel, mx)


@pytest.mark.parametrize("chunk", [1, 3, 64])
def test_host_buffer_path_matches_device_path(chunk):
    """tp_forward_host (pinned host tensors in and out, chunked H2D | compute | D2H pipeline) == device-resident forward, bitwise."""
    s, hidden, n = 3, 256, 7
    m, _ = make_module(hidden, s, seed=4)
    g = torch.Generator().manual_seed(8)
    hx0 = torch.randn(n, 576, 1024, generator=g).bfloat16().pin_memory()
    hxm = torch.randn(n, 576, 4096, generator=g).bfloat16().pin_memory()
    with torch.no_grad():
        ref = m((hx0.cuda(), hxm.cuda())).cpu()
        out = m.forward_host((hx0, hxm), chunk_crops=chunk)
    assert out.shape == ref.shape and not out.is_cuda
    assert torch.equal(out, ref)
    with pytest.raises(TypeError):
        m.forward_host((hx0.float(), hxm))


def test_forward_from_clip_layers_equals_forward_on_concatenation():
    """tp_forward_layers reads the four hidden states through four tensor maps: same bits as feature_select's cat + forward."""
    s, hidden, n = 2, 256, 3
    m, _ = make_module(hidden, s, seed=6)
    g = torch.Generator(device="cuda").manual_seed(9)
    hs = [torch.randn(n, 577, 1024, device="cuda", generator=g).bfloat16() for _ in range(4)]     # layers 12, 16, 22, 23 with CLS
    x0 = hs[3][:, 1:]
    xm = torch.cat(hs, dim=-1)[:, 1:]                                                             # clip_encoder.py:39-43
    with torch.no_grad():
        ref = m((x0, xm))
        out = m.forward_layers(hs)
        out2 = m.forward_layers([h[:, 1:].contiguous() for h in hs])
    assert torch.equal(out, ref) and torch.equal(out2, ref)
