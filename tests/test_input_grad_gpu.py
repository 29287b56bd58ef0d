"""Gradients w.r.t. the CLIP features (TokenPackerB200.input_grad, tp_backward_inputs) on the GPU.

1. The point-query stencil backwards (tpt_point_query_bwd) against the numpy transpose of the stencil, bit for bit.
2. The two new dgrads against float64 references computed from the bf16 values the backward stored (tpt_bwd_layout), with the
   tolerance idiom of tests/test_train_kernels_gpu.py (bf16 rounding of the result plus an fp32 accumulation floor derived from
   K, never fitted); d_x0 = stencil^T(stored dq) exactly; the launch count of each variant.
3. End to end: x0.grad / xm.grad against autograd over oracle/torch_port.forward in fp32, <= 1.5 % rel-RMS per tensor and per crop
   (the gate the parameter gradients meet in tests/test_backward_gpu.py).
4. Bitwise properties: parameter gradients unchanged by asking for input gradients, run-to-run identity, batch invariance per crop.
5. Plumbing through autograd: which gradients are asked for, dtypes, [:,1:] CLIP views, forward_packed, the switch off.
The worst measured ratios are recorded as test properties (``pytest -o junit_family=legacy --junitxml``).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import hd_oracle as hdo
from oracle import tokenpacker_oracle as tpo
from oracle import torch_port
from test_input_grad_host import stencil_t

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_input_grad_hooks.so")
E = 2.0 ** -24            # fp32 unit roundoff
U = 2.0 ** -8             # bf16 unit roundoff
F64 = torch.float64
BF = torch.bfloat16
DIVISORS = [1, 2, 3, 4, 6, 8, 12, 24]


@pytest.fixture(scope="module")
def hk():
    import tokenpacker_b200  # noqa: F401  (the product library is loaded next to this one, as in a real process)
    assert os.path.exists(HOOKS), f"{HOOKS} missing: build with `make -C tokenpacker_b200/csrc`"
    lib = C.CDLL(HOOKS)
    lib.tpt_point_query_bwd.restype = C.c_int
    lib.tpt_point_query_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
    lib.tpt_bwd_layout.restype = C.c_int
    lib.tpt_bwd_layout.argtypes = [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int64)]
    return lib


@pytest.fixture(autouse=True)
def _fp32_exact():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    torch.cuda.empty_cache()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(torch.int16)


def _module(s, hidden, seed):
    from tokenpacker_b200 import TokenPackerB200
    params = {k: tpo.round_bf16(v) for k, v in tpo.make_params(hidden, seed=seed).items()}
    m = TokenPackerB200(hidden_size=hidden, scale_factor=s)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    return m.to("cuda", BF).train(), params


def _inputs(n, seed):
    x0, xm = tpo.make_inputs(n, seed=seed)
    return torch.from_numpy(tpo.round_bf16(x0)).cuda(), torch.from_numpy(tpo.round_bf16(xm)).cuda()     # fp32, bf16 values


def _grad_out(n, s, hidden, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, (24 // s) ** 2, hidden, device="cuda", generator=g).to(BF)


def _every_binade(shape, seed):
    """bf16 values with exponents from the subnormals (2^-133) to the top binade (2^127), random signs and mantissas"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    e = torch.randint(-133, 128, shape, device="cuda", generator=g).to(F64)
    mant = 1 + torch.rand(shape, device="cuda", generator=g, dtype=F64) * 0.99
    sign = torch.randint(0, 2, shape, device="cuda", generator=g).to(F64) * 2 - 1
    return (sign * mant * torch.exp2(e)).to(torch.float32).to(BF)


# ------------------------------------------------------------------------------------------------------------------------------
# 1. the stencil backwards, bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", DIVISORS)
def test_point_query_bwd_is_the_stencil_transpose_bit_for_bit(hk, s):
    n = 3
    g = 24 // s
    dq = _every_binade((n, g * g, 1024), 100 + s)
    assert torch.isfinite(dq.float()).all()
    assert (dq.float().abs() >= 2.0 ** 127).any() and ((dq.float() != 0) & (dq.float().abs() < 2.0 ** -126)).any()
    dx0 = torch.full((n + 1, 576, 1024), float("nan"), dtype=BF, device="cuda")       # crop n: a sentinel the call must not touch
    assert hk.tpt_point_query_bwd(dq.data_ptr(), dx0.data_ptr(), n, s, _stream()) == 0
    torch.cuda.synchronize()
    ref = torch.from_numpy(stencil_t(dq.float().cpu().numpy(), s)).to(BF)
    assert not torch.isnan(dx0[:n].float()).any()
    assert torch.equal(_bits(dx0[:n].cpu()), _bits(ref))
    assert torch.isnan(dx0[n].float()).all()
    taps = torch.from_numpy(stencil_t(np.ones((1, g * g, 1), np.float32), s)).reshape(576) != 0
    assert torch.equal(_bits(dx0[:n, ~taps.cuda()]), torch.zeros_like(_bits(dx0[:n, ~taps.cuda()])))   # +0.0 exactly off the taps
    assert int(taps.sum()) == (576 if s == 2 else g * g * (1 if s % 2 else 4))


# ------------------------------------------------------------------------------------------------------------------------------
# 2. stage checks through the C ABI on a workspace the test owns
# ------------------------------------------------------------------------------------------------------------------------------
def _train_step_c(m, x0b, xmb, gout, want_x0, want_xm, entry="inputs"):
    """tp_pack_weights_train + tp_forward_train + (tp_backward_inputs | tp_backward) on buffers owned here; the workspace and d_x0 /
    d_xm start as NaN bytes.  Returns (grads, d_x0, d_xm, workspace, launches of the backward)."""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    s, H, n = m.scale_factor, m.hidden_size, x0b.shape[0]
    bf = [p.detach().contiguous() for p in m._raw_params()]
    w = _lib.TpWeights(*[t.data_ptr() for t in bf])
    pbytes = lib.tp_packed_bytes(H)
    packed = torch.empty(pbytes, dtype=torch.uint8, device="cuda")
    _lib.check(lib.tp_pack_weights_train(C.byref(w), H, packed.data_ptr(), pbytes, _stream()), "pack")
    sbytes = lib.tp_train_saved_bytes(n, s, H)
    saved = torch.empty(sbytes, dtype=torch.uint8, device="cuda")
    out = torch.empty(n, m.num_queries, H, dtype=BF, device="cuda")
    _lib.check(lib.tp_forward_train(C.byref(w), packed.data_ptr(), x0b.data_ptr(), xmb.data_ptr(), n, 576 * 1024, 576 * 4096, s, H,
                                    out.data_ptr(), saved.data_ptr(), sbytes, _stream()), "tp_forward_train")
    grads = [torch.full_like(t, float("nan")) for t in bf]
    gs = _lib.TpWeights(*[t.data_ptr() for t in grads])
    wbytes = lib.tp_backward_workspace_bytes(n, s, H)
    ws = torch.full((wbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    d_x0 = torch.full((n, 576, 1024), float("nan"), dtype=BF, device="cuda") if want_x0 else None
    d_xm = torch.full((n, 576, 4096), float("nan"), dtype=BF, device="cuda") if want_xm else None
    torch.cuda.synchronize()
    before = lib.tp_launch_count()
    if entry == "inputs":
        _lib.check(lib.tp_backward_inputs(C.byref(w), packed.data_ptr() if want_xm else None, xmb.data_ptr(), 576 * 4096, n, s, H,
                                          gout.data_ptr(), saved.data_ptr(), C.byref(gs), d_x0.data_ptr() if want_x0 else None,
                                          d_xm.data_ptr() if want_xm else None, ws.data_ptr(), wbytes, _stream()), "tp_backward_inputs")
    else:
        _lib.check(lib.tp_backward(C.byref(w), xmb.data_ptr(), 576 * 4096, n, s, H, gout.data_ptr(), saved.data_ptr(), C.byref(gs),
                                   ws.data_ptr(), wbytes, _stream()), "tp_backward")
    launches = lib.tp_launch_count() - before
    torch.cuda.synchronize()
    return grads, d_x0, d_xm, ws, launches


def _check(record, name, got, ref, floor):
    """|got - ref| <= U |ref| + (1 + U) floor, elementwise; records the worst ratio error / bound."""
    got, ref = got.to(F64), ref.to(F64)
    assert torch.isfinite(got).all(), name
    bound = U * ref.abs() + (1 + U) * floor
    ratio = float(((got - ref).abs() / bound.clamp_min(1e-300)).max())
    record(name, f"{ratio:.3g}")
    assert ratio <= 1.0, (name, ratio)


@pytest.mark.parametrize("s,hidden,n", [(2, 4096, 2), (3, 256, 3), (24, 128, 2)])
def test_stages_against_fp64_and_launches(hk, record_property, s, hidden, n):
    m, params = _module(s, hidden, seed=40 + s)
    x0, xm = _inputs(n, seed=50 + s)
    x0b, xmb = x0.to(BF).contiguous(), xm.to(BF).contiguous()
    gout = _grad_out(n, s, hidden, 60 + s)
    base, _, _, _, l_base = _train_step_c(m, x0b, xmb, gout, False, False, entry="backward")
    none, _, _, _, l_none = _train_step_c(m, x0b, xmb, gout, False, False)
    grads, d_x0, d_xm, ws, l_both = _train_step_c(m, x0b, xmb, gout, True, True)
    _, _, _, _, l_x0 = _train_step_c(m, x0b, xmb, gout, True, False)
    _, _, _, _, l_xm = _train_step_c(m, x0b, xmb, gout, False, True)
    # each dgrad joins a launch the backward already makes; d_x0 adds the stencil kernel and nothing else
    assert l_none == l_base and l_xm == l_base and l_x0 == l_base + 1 and l_both == l_base + 1, (l_base, l_none, l_x0, l_xm, l_both)
    for a, b, c in zip(base, none, grads):                  # parameter gradients: exactly those of tp_backward
        assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(a), _bits(c))

    lay = (C.c_int64 * 4)()
    assert hk.tpt_bwd_layout(n, s, hidden, lay) == 0
    o_dzkv, o_dqh, o_dyq, total = (int(v) for v in lay)
    assert total == ws.numel()
    R, Q = n * 576, n * m.num_queries

    def region(off, rows, cols):
        return ws[off:off + rows * cols * 2].view(BF).view(rows, cols)
    dz, dq, dyq = region(o_dzkv, R, 2048), region(o_dqh, Q, 1024), region(o_dyq, Q, 1024)
    assert torch.isfinite(dz.float()).all() and torch.isfinite(dyq.float()).all()
    w_kv0 = torch.cat([torch.from_numpy(params["k_proj_1.0.weight"]), torch.from_numpy(params["v_proj_1.0.weight"])]).cuda().to(F64)
    w_q = torch.from_numpy(params["q_proj_1.weight"]).cuda().to(F64)
    dzd, dyqd = dz.to(F64), dyq.to(F64)
    _check(record_property, "dxm", d_xm.view(R, 4096), dzd @ w_kv0, 2048 * E * (dzd.abs() @ w_kv0.abs()))
    _check(record_property, "dq", dq, dyqd @ w_q, 1024 * E * (dyqd.abs() @ w_q.abs()))
    ref_x0 = torch.from_numpy(stencil_t(dq.float().view(n, -1, 1024).cpu().numpy(), s)).to(BF)
    assert torch.equal(_bits(d_x0.cpu()), _bits(ref_x0))


# ------------------------------------------------------------------------------------------------------------------------------
# 3. end to end against autograd over the reference's op sequence (fp32)
# ------------------------------------------------------------------------------------------------------------------------------
def _rel(got, ref):
    return float((got.float() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())


@pytest.mark.parametrize("s,hidden,n", [(2, 256, 2), (3, 128, 3), (4, 256, 4), (6, 256, 2), (24, 256, 3), (2, 4096, 8)])
def test_input_gradients_match_autograd_of_reference(record_property, s, hidden, n):
    m, params = _module(s, hidden, seed=21 + s)
    m.input_grad = True
    x0, xm = _inputs(n, seed=31 + s)
    gw = _grad_out(n, s, hidden, 5).float()
    a0 = x0.to(BF).requires_grad_(True)
    am = xm.to(BF).requires_grad_(True)
    out = m((a0, am))
    (out.float() * gw).sum().backward()

    ref_p = {k: torch.from_numpy(v).cuda() for k, v in params.items()}
    r0, rm = x0.clone().requires_grad_(True), xm.clone().requires_grad_(True)
    (torch_port.forward(ref_p, r0, rm, s) * gw).sum().backward()
    assert a0.grad.dtype == BF and am.grad.dtype == BF
    worst = {}
    for name, got, ref in (("x0", a0.grad, r0.grad), ("xm", am.grad, rm.grad)):
        assert torch.isfinite(got.float()).all(), name
        per = [_rel(got[i], ref[i]) for i in range(n)]
        worst[name] = max([_rel(got, ref)] + per)
        record_property(f"rel_rms_{name}", f"{_rel(got, ref):.3g}")
        record_property(f"rel_rms_{name}_worst_crop", f"{max(per):.3g}")
    assert max(worst.values()) <= 1.5e-2, worst


# ------------------------------------------------------------------------------------------------------------------------------
# 4. bitwise properties
# ------------------------------------------------------------------------------------------------------------------------------
def _step(m, x0, xm, gw, want=(True, True)):
    m.zero_grad(set_to_none=True)
    a0 = x0.detach().clone().requires_grad_(want[0])
    am = xm.detach().clone().requires_grad_(want[1])
    out = m((a0, am))
    (out.float() * gw).sum().backward()
    return a0.grad, am.grad, {k: p.grad.clone() for k, p in m.named_parameters()}


@pytest.mark.parametrize("s,hidden", [(2, 4096), (3, 256)])
def test_bitwise_properties(s, hidden):
    m, _ = _module(s, hidden, seed=7)
    m.input_grad = True
    n = 4
    x0, xm = _inputs(n, seed=8)
    x0, xm = x0.to(BF), xm.to(BF)
    gw = _grad_out(n, s, hidden, 9).float()
    g0, gm, gp = _step(m, x0, xm, gw)
    g0b, gmb, gpb = _step(m, x0, xm, gw)
    assert torch.equal(_bits(g0), _bits(g0b)) and torch.equal(_bits(gm), _bits(gmb))          # run to run
    for k in gp:
        assert torch.equal(_bits(gp[k]), _bits(gpb[k])), k
    m.input_grad = False
    _, _, gp_only = _step(m, x0, xm, gw, want=(False, False))
    for k in gp:
        assert torch.equal(_bits(gp[k]), _bits(gp_only[k])), k                                 # parameter gradients unchanged
    m.input_grad = True
    for i in (0, n - 1):                                                                         # crop i alone = crop i of the batch
        s0, sm, _ = _step(m, x0[i:i + 1], xm[i:i + 1], gw[i:i + 1])
        assert torch.equal(_bits(s0[0]), _bits(g0[i])), ("x0", i)
        assert torch.equal(_bits(sm[0]), _bits(gm[i])), ("xm", i)


# ------------------------------------------------------------------------------------------------------------------------------
# 5. plumbing
# ------------------------------------------------------------------------------------------------------------------------------
def test_only_x0_requires_grad_never_asks_for_xm(monkeypatch):
    from tokenpacker_b200 import projector
    m, _ = _module(2, 256, seed=11)
    m.input_grad = True
    n = 2
    x0, xm = _inputs(n, seed=12)
    gw = _grad_out(n, 2, 256, 13).float()
    calls = []
    orig = projector.lib.tp_backward_inputs

    def spy(*args):
        calls.append(args)
        return orig(*args)
    monkeypatch.setattr(projector.lib, "tp_backward_inputs", spy)
    a0 = x0.to(BF).requires_grad_(True)
    b_m = xm.to(BF)
    (m((a0, b_m)).float() * gw).sum().backward()
    assert len(calls) == 1 and calls[0][1] is None and calls[0][10] is not None and calls[0][11] is None   # no packed, no d_xm
    assert b_m.grad is None and a0.grad is not None
    g_x0 = a0.grad.clone()
    # frozen parameters: the input gradient alone still takes the training path, and gives the same bits
    for p in m.parameters():
        p.requires_grad_(False)
    a0 = x0.to(BF).requires_grad_(True)
    (m((a0, b_m)).float() * gw).sum().backward()
    assert len(calls) == 2 and torch.equal(_bits(a0.grad), _bits(g_x0))


def test_fp16_and_fp32_inputs_get_gradients_in_their_dtype():
    m, _ = _module(2, 256, seed=14)
    m.input_grad = True
    n = 2
    x0, xm = _inputs(n, seed=15)                  # bf16 values: every cast below is exact
    gw = _grad_out(n, 2, 256, 16).float()
    ref0, refm, _ = _step(m, x0.to(BF), xm.to(BF), gw)
    for dt in (torch.float16, torch.float32):
        a0, am = x0.to(dt).requires_grad_(True), xm.to(dt).requires_grad_(True)
        out = m((a0, am))
        (out.float() * gw).sum().backward()
        assert a0.grad.dtype == dt and am.grad.dtype == dt
        if dt == torch.float32:
            assert torch.equal(a0.grad, ref0.float()) and torch.equal(am.grad, refm.float())


def test_clip_view_gets_zero_gradient_in_cls_row():
    m, _ = _module(2, 256, seed=17)
    m.input_grad = True
    n = 2
    x0, xm = _inputs(n, seed=18)
    gw = _grad_out(n, 2, 256, 19).float()
    ref0, refm, _ = _step(m, x0.to(BF), xm.to(BF), gw)
    g = torch.Generator(device="cuda").manual_seed(20)
    f0 = torch.randn(n, 577, 1024, device="cuda", generator=g).to(BF)
    fm = torch.randn(n, 577, 4096, device="cuda", generator=g).to(BF)
    f0[:, 1:] = x0.to(BF)
    fm[:, 1:] = xm.to(BF)
    f0.requires_grad_(True)
    fm.requires_grad_(True)
    out = m((f0[:, 1:], fm[:, 1:]))
    (out.float() * gw).sum().backward()
    assert torch.equal(_bits(f0.grad[:, 0]), torch.zeros_like(_bits(f0.grad[:, 0])))
    assert torch.equal(_bits(fm.grad[:, 0]), torch.zeros_like(_bits(fm.grad[:, 0])))
    assert torch.equal(_bits(f0.grad[:, 1:]), _bits(ref0)) and torch.equal(_bits(fm.grad[:, 1:]), _bits(refm))


def test_forward_packed_carries_input_gradients():
    s, hidden = 4, 128
    grids = [(1, 1), (2, 3)]
    n = sum(hdo.n_crops(a, b) for a, b in grids)
    m, _ = _module(s, hidden, seed=22)
    m.input_grad = True
    x0, xm = _inputs(n, seed=23)
    g = torch.Generator(device="cuda").manual_seed(24)
    sep = torch.randn(hidden, device="cuda", generator=g).to(BF)
    ret = torch.randn(hidden, device="cuda", generator=g).to(BF)
    hb, wb = [a for a, _ in grids], [b for _, b in grids]
    a0, am = x0.to(BF).requires_grad_(True), xm.to(BF).requires_grad_(True)
    packed, cu = m.forward_packed((a0, am), hb, wb, sep, ret)
    gp = torch.randn(packed.shape, device="cuda", generator=g)
    (packed.float() * gp).sum().backward()
    assert a0.grad is not None and am.grad is not None
    # the same gradient through forward() + the scatter's transpose (rows of crop i start at i (M + 1))
    M = m.num_queries
    rows = (torch.arange(n, device="cuda")[:, None] * (M + 1) + torch.arange(M, device="cuda")[None, :]).reshape(-1)
    ref0, refm, _ = _step(m, x0.to(BF), xm.to(BF), gp.to(BF).float()[rows].view(n, M, hidden))
    assert torch.equal(_bits(a0.grad), _bits(ref0)) and torch.equal(_bits(am.grad), _bits(refm))
    # frozen parameters, separator rows not requiring grad: the input gradient alone selects the differentiable path
    for p in m.parameters():
        p.requires_grad_(False)
    a0 = x0.to(BF).requires_grad_(True)
    packed2, _ = m.forward_packed((a0, xm.to(BF)), hb, wb, sep, ret)
    assert packed2.requires_grad
    (packed2.float() * gp).sum().backward()
    assert torch.equal(_bits(a0.grad), _bits(ref0))


def test_switch_off_still_raises():
    m, _ = _module(2, 256, seed=25)
    x0, xm = _inputs(1, seed=26)
    assert m.input_grad is False
    with pytest.raises(NotImplementedError, match="input_grad"):
        m((x0.to(BF).requires_grad_(True), xm.to(BF)))
    with pytest.raises(NotImplementedError):
        m((x0.to(BF), xm.to(BF).requires_grad_(True)))
    m.input_grad = True
    for p in m.parameters():
        p.requires_grad_(False)
    with pytest.raises(NotImplementedError):                     # inference-only paths stay so
        m.forward_into_peers((x0.to(BF).requires_grad_(True), xm.to(BF)), [0], 0)
