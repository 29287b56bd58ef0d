"""The backward's kernels one by one, through the test-hook library (tests/csrc/tp_test_hooks.cu: the same launch functions
tp_backward calls), against plain float64 references computed from the same bf16 inputs.  Plus the whole backward at a batch
that takes the split-K weight-gradient path.

Tolerances are derived from the arithmetic, never fitted: a stored bf16 result is within U = 2^-8 of the value it rounds (8
significant bits), and an fp32 sum of n terms is within n * E * sum|terms| of the exact sum (E = 2^-24), with n the longest
chain of dependent additions the kernel performs.  Each check asserts |got - ref| <= U |ref| + (1 + U) * floor elementwise, the
floor being that fp32 bound.  The worst measured ratio error / bound of each check is recorded as a test property
(``pytest -o junit_family=legacy --junitxml``) and quoted in the docstrings, as measured on an H100 (80 GB HBM3, 400 W power
limit).  A ratio close to 1 is expected wherever the bf16 rounding of the result dominates: that rounding alone can take up the
whole U |ref| term.  The file runs in about 10 s on that H100 (plus the torch import).
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_testhooks.so")
E = 2.0 ** -24            # fp32 unit roundoff
U = 2.0 ** -8             # bf16 unit roundoff
F64 = torch.float64
BF = torch.bfloat16

_vp, _i64, _int, _f32, _sz = C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_size_t
_SIGNATURES = {
    "tpt_launch_count": (C.c_uint64, []),
    "tpt_constants": (_int, [C.POINTER(_i64)]),
    "tpt_wgrad_splitk": (_int, [_vp, _i64, _vp, _i64, _i64, _int, _int, _int, _vp, _sz, _vp, _i64, _vp, _i64, _vp, _i64, _i64, _int, _int,
                                _f32, _vp]),
    "tpt_splitk_reduce": (_int, [_vp, _int, _i64, _f32, _vp, _vp]),
    "tpt_ln_bwd": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _sz, _i64, _vp, _vp, _vp, _vp]),
    "tpt_ln_apply": (_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "tpt_window_attn_bwd": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _int, _vp]),
    "tpt_gelu_fwd": (_int, [_vp, _vp, _i64, _vp]),
    "tpt_gelu_bwd_bias": (_int, [_vp, _vp, _i64, _i64, _int, _vp, _vp, _vp, _sz, _vp]),
    "tpt_colsum": (_int, [_vp, _i64, _i64, _int, _f32, _vp, _sz, _vp, _vp]),
    "tpt_transpose": (_int, [_vp, _i64, _vp, _i64, _i64, _int, _vp]),
}


class Hooks:
    def __init__(self):
        import tokenpacker_b200  # noqa: F401  (the product library is loaded next to this one, as in a real process)
        assert os.path.exists(HOOKS), f"{HOOKS} missing: build with `make -C tokenpacker_b200/csrc`"
        self.lib = C.CDLL(HOOKS)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(self.lib, name)
            fn.restype, fn.argtypes = res, args
        c = (_i64 * 4)()
        assert self.lib.tpt_constants(c) == 0
        self.ln_blocks, self.col_chunks, self.splits, self.split_min_rows = (int(v) for v in c)

    def __getattr__(self, name):
        fn = getattr(self.lib, name)

        def call(*args):
            return fn(*args, torch.cuda.current_stream().cuda_stream)
        return call if name not in ("tpt_launch_count", "tpt_constants") else fn


@pytest.fixture(scope="module")
def hk():
    return Hooks()


@pytest.fixture(autouse=True)
def _fp64_and_fp32_exact():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    torch.cuda.empty_cache()


def P(t):
    return t.data_ptr() if t is not None else None


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(shape, seed, scale=1.0, mean=0.0):
    return (torch.randn(shape, device="cuda", generator=_gen(seed)) * scale + mean).to(BF)


def _check(record, name, got, ref, floor):
    """|got - ref| <= U |ref| + (1 + U) floor, elementwise (floor broadcasts); records the worst ratio error / bound."""
    got, ref = got.to(F64), ref.to(F64)
    assert torch.isfinite(got).all(), name
    bound = U * ref.abs() + (1 + U) * floor
    ratio = float(((got - ref).abs() / bound.clamp_min(1e-300)).max())
    record(name, f"{ratio:.3g}")
    assert ratio <= 1.0, (name, ratio)
    return ratio


def _check_f32(record, name, got, ref, floor):
    """an fp32 result (no bf16 rounding): |got - ref| <= floor elementwise"""
    ratio = float(((got.to(F64) - ref).abs() / floor.clamp_min(1e-300)).max())
    record(name, f"{ratio:.3g}")
    assert ratio <= 1.0, (name, ratio)


# ------------------------------------------------------------------------------------------------------------------------------
# split-K weight gradient (tp_backward's in_proj k/v and k_proj_1.2 / v_proj_1.2 wgrads once R >= 16384 rows)
# ------------------------------------------------------------------------------------------------------------------------------
def _slices(K, splits):
    kb = (K + 63) // 64
    per = (kb + splits - 1) // splits
    return [(s * per * 64, min(K, (s + 1) * per * 64)) for s in range(splits)]


def _reduce_emulated(part, alpha):
    """splitk_reduce_kernel's fixed order in float32: bf16_rn((((p0 + p1) + p2) + p3) * alpha)"""
    acc = part[0].clone()
    for s in range(1, part.shape[0]):
        acc = acc + part[s]
    return (acc * torch.tensor(alpha, dtype=torch.float32, device="cuda")).to(BF)


def _splitk(hk, dy, x, splits, dgrad=None):
    K, M = dy.shape
    N = x.shape[1]
    part = torch.full((splits, M, N), 7.0, dtype=torch.float32, device="cuda")
    d = dgrad or (None, None, None)
    st = hk.tpt_wgrad_splitk(P(dy), dy.stride(0), P(x), x.stride(0), K, M, N, splits, P(part), part.numel(), P(d[0]),
                             d[0].stride(0) if d[0] is not None else 0, P(d[1]), d[1].stride(0) if d[1] is not None else 0, P(d[2]),
                             d[2].stride(0) if d[2] is not None else 0, d[0].shape[0] if d[0] is not None else 0,
                             d[1].shape[1] if d[1] is not None else 0, d[1].shape[0] if d[1] is not None else 0, 1.0)
    return st, part


@pytest.mark.parametrize("K", [16384, 16704, 18432, 20000, 36864])
def test_wgrad_splitk_slices_and_reduce(hk, record_property, K):
    """Each fp32 slice against the fp64 product over its own rows (pins kb_per_split, the slice offsets and boundaries: K = 16704
    is n = 29 crops, slices of 66/66/66/63 k-blocks; 20000 ends in a half k-block), the reduce bit for bit against its float32
    emulation, and the reduced bf16 gradient against the fp64 product.  Floor: one fp32 chain per slice row, n E sum|dy x|.
    Measured on an H100: worst slice error / bound 0.0027 (the bound is a worst case), reduced output 0.12."""
    dy, x = _bf((K, 1024), 1 + K), _bf((K, 1024), 2 + K)
    st, part = _splitk(hk, dy, x, hk.splits)
    assert st == 0
    dyd, xd = dy.to(F64), x.to(F64)
    for s, (r0, r1) in enumerate(_slices(K, hk.splits)):
        ref = dyd[r0:r1].t() @ xd[r0:r1]
        _check_f32(record_property, f"slice{s}", part[s], ref, (r1 - r0) * E * (dyd[r0:r1].abs().t() @ xd[r0:r1].abs()))
    for alpha in (1.0, 0.08838834764831845):
        out = torch.empty(1024, 1024, dtype=BF, device="cuda")
        assert hk.tpt_splitk_reduce(P(part), hk.splits, part[0].numel(), alpha, P(out)) == 0
        assert torch.equal(out.view(torch.int16), _reduce_emulated(part, alpha).view(torch.int16))
    full = dyd.t() @ xd
    _check(record_property, "reduced", out, alpha * full, alpha * K * E * (dyd.abs().t() @ xd.abs()))


def test_wgrad_splitk_small_integers_exact(hk):
    """Integers in [-4, 4]: every product and partial sum (|.| <= 16 * 16704 < 2^24) is exact in fp32, so every slice must equal the
    exact product and the reduce must be the bf16 rounding of the exact total."""
    K = 16704
    dy = torch.randint(-4, 5, (K, 1024), device="cuda", generator=_gen(3)).to(BF)
    x = torch.randint(-4, 5, (K, 1024), device="cuda", generator=_gen(4)).to(BF)
    st, part = _splitk(hk, dy, x, hk.splits)
    assert st == 0
    dyd, xd = dy.to(F64), x.to(F64)
    for s, (r0, r1) in enumerate(_slices(K, hk.splits)):
        assert torch.equal(part[s].to(F64), dyd[r0:r1].t() @ xd[r0:r1]), s
    out = torch.empty(1024, 1024, dtype=BF, device="cuda")
    assert hk.tpt_splitk_reduce(P(part), hk.splits, part[0].numel(), 1.0, P(out)) == 0
    assert torch.equal(out.view(torch.int16), (dyd.t() @ xd).to(BF).view(torch.int16))


def test_wgrad_splitk_grouped_with_dgrad(hk, record_property):
    """The split-K item in one launch with an NN dgrad item (as tp_backward groups them): both outputs right.
    Measured on an H100: worst error / bound 0.0026 (slices), 0.92 (dgrad: its bf16 rounding)."""
    K = 16704
    dy, x = _bf((K, 1024), 5), _bf((K, 1024), 6)
    w = _bf((1024, 1024), 7, scale=0.03)
    dx = torch.full((K, 1024), float("nan"), dtype=BF, device="cuda")
    st, part = _splitk(hk, dy, x, hk.splits, dgrad=(dy, w, dx))
    assert st == 0
    dyd, xd, wd = dy.to(F64), x.to(F64), w.to(F64)
    for s, (r0, r1) in enumerate(_slices(K, hk.splits)):
        _check_f32(record_property, f"slice{s}", part[s], dyd[r0:r1].t() @ xd[r0:r1],
                   (r1 - r0) * E * (dyd[r0:r1].abs().t() @ xd[r0:r1].abs()))
    _check(record_property, "dgrad", dx, dyd @ wd, 1024 * E * (dyd.abs() @ wd.abs()))


@pytest.mark.parametrize("K,splits", [(320, 4), (576, 4), (1024, 20)])
def test_wgrad_splitk_empty_slice_refused(hk, K, splits):
    """A split count that leaves the last slice without k-blocks (5 blocks in slices of 2; 9 in slices of 3; 16 in slices of 1
    over 20 splits) is an invalid argument, and nothing is launched or written."""
    dy, x = _bf((K, 1024), 8), _bf((K, 1024), 9)
    torch.cuda.synchronize()
    n0 = hk.tpt_launch_count()
    st, part = _splitk(hk, dy, x, splits)
    torch.cuda.synchronize()
    assert st == 1 and hk.tpt_launch_count() == n0
    assert bool((part == 7.0).all())


# ------------------------------------------------------------------------------------------------------------------------------
# LayerNorm backward + parameter reduce, LayerNorm apply
# ------------------------------------------------------------------------------------------------------------------------------
def _ln_inputs(rows, seed):
    """rows of three kinds: ordinary; |mean| >> std (mean +-10..30, std 0.25: a few bf16 levels); std ~ 1e-3 (var ~ eps)"""
    kind = (torch.arange(rows, device="cuda") * 7 + 2) % 3
    g = _gen(seed)
    mean = torch.where(kind == 0, torch.randn(rows, device="cuda", generator=g) * 0.5,
                       torch.where(kind == 1, (10 + 20 * torch.rand(rows, device="cuda", generator=g)) *
                                   torch.sign(torch.randn(rows, device="cuda", generator=g)), torch.zeros(rows, device="cuda")))
    std = torch.where(kind == 0, torch.ones(rows, device="cuda"), torch.where(kind == 1, torch.full((rows,), 0.25, device="cuda"),
                                                                                torch.full((rows,), 1e-3, device="cuda")))
    y = (torch.randn(rows, 1024, device="cuda", generator=g) * std[:, None] + mean[:, None]).to(BF)
    yd = y.to(F64).view(rows, 8, 128)
    mb = yd.mean(-1)
    m2 = ((yd - mb[..., None]) ** 2).sum(-1)
    stats = torch.stack([mb, m2], -1).to(torch.float32).contiguous()          # the forward's per-128-column (mean, M2)
    gout = _bf((rows, 1024), seed + 1)
    gamma = _bf((1024,), seed + 2, scale=0.2, mean=1.0)
    beta = _bf((1024,), seed + 3, scale=0.2)
    return y, stats, gout, gamma, beta


def _ln_ref(y, stats, gamma):
    """fp64 mean / rstd from the fp32 stats the kernel reads, and per-row bounds of the kernel's fp32 error in yhat"""
    st = stats.to(F64)
    mb, m2 = st[..., 0], st[..., 1]
    mu = mb.mean(-1)
    d = mb - mu[:, None]
    between, m2t = (d * d).sum(-1), m2.sum(-1)
    var = (128 * between + m2t) / 1024
    rstd = 1 / torch.sqrt(var + 1e-6)
    yd = y.to(F64)
    yh = (yd - mu[:, None]) * rstd[:, None]
    dmu = 10 * E * mb.abs().amax(-1)
    dbet = (2 * d.abs() * (E * d.abs() + dmu[:, None])).sum(-1) + 8 * E * between
    dvar = (128 * dbet + 10 * E * m2t) / 1024 + 2 * E * var
    rho = 0.5 * dvar / (var + 1e-6) + 4 * E                                   # relative error of rstd (rsqrtf: 2 ulp)
    dyh = rstd * (E * (yd - mu[:, None]).abs().amax(-1) + dmu) + yh.abs().amax(-1) * (rho + 2 * E)
    return yh, rstd, rho, dyh


def _ln_bwd_ref(gout, y, stats, gamma, ln_blocks):
    """fp64 LayerNorm backward (ln_bwd_kernel + ln_param_reduce_kernel over ln_blocks CTAs) from the bf16 / fp32 values the kernels
    read: {name: (ref, floor)} for dy, dgamma and dbeta, and the length of the fp32 chain of the column sums (dbias, taken over the
    STORED dy, has the same chain).  Floors: 48 E per row sum (32 sequential lane adds + 5 shuffle levels), propagated through rstd
    and yhat; column sums: rows-per-warp + 8 warps + 19 + 16 lane partials."""
    rows = y.shape[0]
    yh, rstd, rho, dyh = _ln_ref(y, stats, gamma)
    g, gm = gout.to(F64), gamma.to(F64)
    gg = gm * g
    c1, c2 = gg.mean(-1), (gg * yh).mean(-1)
    ref = rstd[:, None] * (gg - c1[:, None] - yh * c2[:, None])
    A, B, Y = gg.abs().mean(-1), (gg * yh).abs().mean(-1), yh.abs().amax(-1)
    dc1 = 48 * E * A
    dc2 = 48 * E * B + A * dyh
    mag = gg.abs().amax(-1) + c1.abs() + Y * c2.abs()
    floor = rstd * (dc1 + Y * dc2 + c2.abs() * dyh) + (rho + 4 * E) * rstd * mag
    warps = ln_blocks * 8
    chain = (rows + warps - 1) // warps + 8 + (ln_blocks + 15) // 16 + 16 + 2
    return {"dy": (ref, floor[:, None]),
            "dgamma": ((g * yh).sum(0), chain * E * (g * yh).abs().sum(0) + (g.abs() * dyh[:, None]).sum(0)),
            "dbeta": (g.sum(0), chain * E * g.abs().sum(0))}, chain


def _ln_apply_ref(y, stats, gamma, beta):
    """fp64 LayerNorm output yhat gamma + beta (ln_apply_kernel) and its floor: the fp32 error of yhat, then one fma"""
    yh, _, _, dyh = _ln_ref(y, stats, gamma)
    gm, bt = gamma.to(F64), beta.to(F64)
    return yh * gm + bt, gm.abs() * dyh[:, None] + 2 * E * ((yh * gm).abs() + bt.abs())


@pytest.mark.parametrize("rows", [1, 7, 296 * 8 + 3, 16704])
def test_ln_bwd_and_param_reduce(hk, record_property, rows):
    """dy = rstd (gg - mean(gg) - yhat mean(gg yhat)) elementwise, dgamma / dbeta (column sums of g yhat / g) and dbias (column sums of
    the STORED bf16 dy) against fp64; LayerNorm apply against fp64.  1 row; 7 (a partial warp grid); 2371 (one row past the
    296 x 8 warps of the grid); 16704 (grid-stride wrap, n = 29 crops).  Rows with |mean| >> std and with var ~ eps = 1e-6.
    Floors: 48 E per row sum (32 sequential lane adds + 5 shuffle levels), propagated through rstd and yhat; column sums: one
    fp32 chain of rows-per-warp + 8 warps + 19 + 16 lane partials.
    Measured on an H100: worst error / bound: dy 0.994, dgamma 0.978, dbeta 0.995, dbias 0.977, LayerNorm apply 0.996 (the bf16
    rounding of the result takes up to U |ref|)."""
    y, stats, gout, gamma, beta = _ln_inputs(rows, 40 + rows)
    part = torch.empty(3 * hk.ln_blocks * 1024, dtype=torch.float32, device="cuda")
    dy = torch.empty(rows, 1024, dtype=BF, device="cuda")
    dgam, dbet, dbias = (torch.empty(1024, dtype=BF, device="cuda") for _ in range(3))
    assert hk.tpt_ln_bwd(P(gout), P(y), P(stats), P(gamma), P(dy), P(part), part.numel(), rows, P(dgam), P(dbet), P(dbias)) == 0
    lnout = torch.empty(rows, 1024, dtype=BF, device="cuda")
    assert hk.tpt_ln_apply(P(y), P(stats), P(gamma), P(beta), P(lnout), rows) == 0

    refs, chain = _ln_bwd_ref(gout, y, stats, gamma, hk.ln_blocks)
    _check(record_property, "dy", dy, *refs["dy"])
    _check(record_property, "dgamma", dgam, *refs["dgamma"])
    _check(record_property, "dbeta", dbet, *refs["dbeta"])
    dyk = dy.to(F64)
    _check(record_property, "dbias", dbias, dyk.sum(0), chain * E * dyk.abs().sum(0))
    _check(record_property, "ln_apply", lnout, *_ln_apply_ref(y, stats, gamma, beta))


# ------------------------------------------------------------------------------------------------------------------------------
# window-attention backward
# ------------------------------------------------------------------------------------------------------------------------------
_ATTN_CASES = {1: 1, 2: 2, 3: 2, 4: 3, 6: 4, 8: 5, 12: 6, 24: 13}     # s -> crops; the last 3 queries are dropped (partial last CTA)


def _window_rows(s, n_q):
    G = 24 // s
    q = torch.arange(n_q, device="cuda")
    n, m = q // (G * G), q % (G * G)
    hb, wb = m // G, m % G
    j = torch.arange(s * s, device="cuda")
    return n[:, None] * 576 + (hb[:, None] * s + j[None] // s) * 24 + wb[:, None] * s + j[None] % s     # [Q, W] token rows


def _attn_inputs(s, kind, seed):
    n = _ATTN_CASES[s]
    R, Q = n * 576, n * (24 // s) ** 2 - 3
    rows = _window_rows(s, Q)
    if kind == "random":
        qp, kp = _bf((Q, 1024), seed, scale=0.25), _bf((R, 1024), seed + 1)
    elif kind == "saturated":                      # every logit exactly +-50: 128 channels x 0.5 x 0.78125
        qp = torch.full((Q, 1024), 0.5, device="cuda").to(BF)
        sign = torch.sign(torch.randn(R, 8, 1, device="cuda", generator=_gen(seed)))
        kp = (sign * 0.78125).expand(R, 8, 128).reshape(R, 1024).to(BF)
    else:                                          # all keys of a window equal: uniform softmax, dq' = 0 analytically
        qp = _bf((Q, 1024), seed, scale=0.25)
        kp = torch.zeros(R, 1024, device="cuda").to(BF)
        kp[rows.reshape(-1)] = _bf((Q, 1, 1024), seed + 1).expand(Q, s * s, 1024).reshape(-1, 1024)
    vp, dctx = _bf((R, 1024), seed + 2), _bf((Q, 1024), seed + 3)
    return qp, kp, vp, dctx, rows


def _attn_ref(qp, kp, vp, dctx, rows):
    """fp64 autograd of 8-head single-query window attention, and per-element fp32 error floors of the kernel's formulas"""
    Q, W = rows.shape
    q = qp.to(F64).view(Q, 8, 128).requires_grad_(True)
    k = kp.to(F64)[rows].view(Q, W, 8, 128).requires_grad_(True)
    v = vp.to(F64)[rows].view(Q, W, 8, 128).requires_grad_(True)
    dc = dctx.to(F64).view(Q, 8, 128)
    logit = torch.einsum("qhc,qwhc->qhw", q, k)
    p = torch.softmax(logit, -1)
    ctx = torch.einsum("qhw,qwhc->qhc", p, v)
    dq, dk, dv = torch.autograd.grad((ctx * dc).sum(), (q, k, v))
    with torch.no_grad():
        q, k, v, p, logit = q.detach(), k.detach(), v.detach(), p.detach(), logit.detach()
        dp = torch.einsum("qhc,qwhc->qhw", dc, v)
        dot = (p * dp).sum(-1, keepdim=True)
        ds = p * (dp - dot)
        d_s = 20 * E * torch.einsum("qhc,qwhc->qhw", q.abs(), k.abs())            # logits: 8 fma + 4 shuffle levels (+ slack)
        d_dp = 20 * E * torch.einsum("qhc,qwhc->qhw", dc.abs(), v.abs())
        xr = (logit.amax(-1, keepdim=True) - logit).amax(-1, keepdim=True)      # largest exp argument
        rho = 2 * d_s.amax(-1, keepdim=True) + 2.0 ** -21 + 2 * xr * E + (W + 4) * E
        d_p = p * rho + 2.0 ** -120                                               # + exp results flushed to zero
        d_dot = (d_p * dp.abs() + p * d_dp).sum(-1, keepdim=True) + (W + 2) * E * (p * dp.abs()).sum(-1, keepdim=True)
        d_ds = d_p * (dp - dot).abs() + p * (d_dp + d_dot) + 2 * E * ds.abs()
        f_dv = torch.einsum("qhw,qhc->qwhc", d_p, dc.abs()) + E * torch.einsum("qhw,qhc->qwhc", p, dc.abs())
        f_dk = torch.einsum("qhw,qhc->qwhc", d_ds, q.abs()) + E * torch.einsum("qhw,qhc->qwhc", ds.abs(), q.abs())
        f_dq = torch.einsum("qhw,qwhc->qhc", d_ds, k.abs()) + (W + 1) * E * torch.einsum("qhw,qwhc->qhc", ds.abs(), k.abs())
    return (dq.reshape(Q, 1024), dk.reshape(Q * W, 1024), dv.reshape(Q * W, 1024),
            f_dq.reshape(Q, 1024), f_dk.reshape(Q * W, 1024), f_dv.reshape(Q * W, 1024))


@pytest.mark.parametrize("kind", ["random", "saturated", "equal"])
@pytest.mark.parametrize("s", [1, 2, 3, 4, 6, 8, 12, 24])
def test_window_attn_bwd(hk, record_property, s, kind):
    """dq', dk', dv' of window_attn_bwd_kernel<2|3|4> and window_attn_bwd_stream_kernel (s = 1, 6, 8, 12, 24) against fp64 autograd,
    for random inputs, a saturated softmax (logits +-50) and all-equal logits.  Q = crops x queries - 3: the last CTA is partial,
    and the key/value rows of the dropped queries must stay untouched.
    Measured on an H100: worst error / bound over all s and inputs: dq' 0.96, dk' 0.98, dv' 0.98."""
    qp, kp, vp, dctx, rows = _attn_inputs(s, kind, 100 + s)
    Q, R = qp.shape[0], kp.shape[0]
    dq = torch.full((Q, 1024), float("nan"), dtype=BF, device="cuda")
    dk = torch.full((R, 1024), float("nan"), dtype=BF, device="cuda")
    dv = torch.full((R, 1024), float("nan"), dtype=BF, device="cuda")
    assert hk.tpt_window_attn_bwd(P(qp), P(kp), P(vp), P(dctx), P(dq), P(dk), P(dv), Q, s) == 0
    rdq, rdk, rdv, fq, fk, fv = _attn_ref(qp, kp, vp, dctx, rows)
    flat = rows.reshape(-1)
    _check(record_property, "dq", dq, rdq, fq)
    _check(record_property, "dk", dk[flat], rdk, fk)
    _check(record_property, "dv", dv[flat], rdv, fv)
    untouched = torch.ones(R, dtype=torch.bool, device="cuda")
    untouched[flat] = False
    assert int(untouched.sum()) == 3 * s * s
    assert bool(dk[untouched].isnan().all()) and bool(dv[untouched].isnan().all())


# ------------------------------------------------------------------------------------------------------------------------------
# GELU forward / backward over every finite bf16 value
# ------------------------------------------------------------------------------------------------------------------------------
def _all_finite_bf16():
    bits = np.arange(65536, dtype=np.uint16)
    bits = bits[(bits & 0x7F80) != 0x7F80]                     # drop inf / nan
    z = torch.from_numpy(bits.view(np.int16)).cuda().view(BF)
    return z.view(-1, 256)                                      # 65280 values = [255, 256]


def _phi(zd):
    return torch.exp(-0.5 * zd * zd) / math.sqrt(2 * math.pi)


def _cdf(zd):
    return 0.5 * torch.special.erfc(-zd / math.sqrt(2))


def _gelu_grad_ref(zd):
    """fp64 GELU'(z) = Phi(z) + z phi(z) and the floor of gelu_grad's fp32 value: 1.5e-7 (erf) + a few E + |z phi| (__expf: 2^-21
    + z^2 E relative) + 2^-126 (exp flushed to zero)"""
    zphi = zd * _phi(zd)
    return _cdf(zd) + zphi, 1.5e-7 + 8 * E + zphi.abs() * (2.0 ** -21 + zd * zd * E + 4 * E) + 2.0 ** -126


def test_gelu_fwd_every_bf16(hk, record_property):
    """gelu_fwd_kernel against the fp64 erf GELU x Phi(x) at all 65280 finite bf16 inputs.  Floor: Abramowitz & Stegun 7.1.28
    (|erf error| <= 3e-7, so 1.5e-7 |x|) + a few fp32 roundings of |x|, + 2^-133 for results in bf16's subnormal range.
    Measured on an H100: worst error / bound 0.975."""
    z = _all_finite_bf16()
    h = torch.empty_like(z)
    assert hk.tpt_gelu_fwd(P(z), P(h), z.numel()) == 0
    zd = z.to(F64)
    ref = zd * _cdf(zd)
    _check(record_property, "gelu", h, ref, zd.abs() * (1.5e-7 + 4 * E) + 2.0 ** -133)


def test_gelu_grad_every_bf16(hk, record_property):
    """gelu_grad = Phi(z) + z phi(z), through gelu_bwd_colsum_kernel with dh = 1 (dz = bf16(gelu_grad(z)) exactly), against fp64 at
    all 65280 finite bf16 inputs.  Floor: 1.5e-7 (erf) + a few E + |z phi| (__expf: 2^-21 + 2 x E relative) + 2^-126 (exp flushed
    to zero).  Measured on an H100: worst error / bound 0.993."""
    z = _all_finite_bf16()
    dz = torch.ones_like(z)
    part = torch.empty(hk.col_chunks * 256, dtype=torch.float32, device="cuda")
    out = torch.empty(256, dtype=BF, device="cuda")
    assert hk.tpt_gelu_bwd_bias(P(dz), P(z), 256, z.shape[0], 256, P(out), None, P(part), part.numel()) == 0
    _check(record_property, "gelu_grad", dz, *_gelu_grad_ref(z.to(F64)))


@pytest.mark.parametrize("mode", ["1", "2"])
def test_gemm_gelu_epilogue_equals_gelu_kernel_bitwise(hk, monkeypatch, mode):
    """Z @ I is exact, so gemm_bf16(Z, I, gelu=True) runs the epilogue's gelu_erf_pk on exactly the values gelu_fwd_kernel runs
    gelu_erf on: the bits must agree at every finite bf16 value, under the one-CTA (TP_GEMM_MODE=1) and pair (=2) kernels."""
    from tokenpacker_b200.kernels import gemm_bf16
    monkeypatch.setenv("TP_GEMM_MODE", mode)
    z = _all_finite_bf16()
    eye = torch.eye(256, device="cuda").to(BF)
    same = gemm_bf16(z, eye)
    assert torch.equal(same.float(), z.float())                     # the identity product is exact (-0 becomes +0)
    got = gemm_bf16(z, eye, gelu=True)
    h = torch.empty_like(z)
    assert hk.tpt_gelu_fwd(P(z), P(h), z.numel()) == 0
    assert torch.equal(got.view(torch.int16), h.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------------------------
# column sums (bias gradients)
# ------------------------------------------------------------------------------------------------------------------------------
def _colsum_chain(rows, col_chunks):
    """longest fp32 chain of colsum_partial + colsum_reduce over rows: rows per chunk + 16 lanes of chunks + the 16 lane sums + 2"""
    chunks = min(rows, col_chunks)
    return (rows + chunks - 1) // chunks + (chunks + 15) // 16 + 16 + 2


@pytest.mark.parametrize("cols", [8, 1000, 2048, 5120])
@pytest.mark.parametrize("rows", [1, 591, 592, 593, 36864])
def test_colsum(hk, record_property, rows, cols):
    """colsum_partial + colsum_reduce against fp64 (rows around the 592 chunks: fewer rows than chunks, one row per chunk, a
    chunk of two), deterministic run to run; the fused gelu_bwd_colsum sums (with and without out_hi) equal colsum over the dz it
    stored, bit for bit.  Floor: one fp32 chain of rows-per-chunk + 37 + 16 adds.  Measured on an H100: worst error / bound 0.978."""
    ld = cols + 16 if rows == 593 else cols                    # a strided input
    x = _bf((rows, ld), rows * 7 + cols, mean=0.3)
    part = torch.empty(hk.col_chunks * cols, dtype=torch.float32, device="cuda")
    scale = 0.08838834764831845 if cols == 1000 else 1.0
    outs = []
    for _ in range(2):
        out = torch.empty(cols, dtype=BF, device="cuda")
        assert hk.tpt_colsum(P(x), ld, rows, cols, scale, P(part), part.numel(), P(out)) == 0
        outs.append(out)
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    xd = x[:, :cols].to(F64)
    chain = _colsum_chain(rows, hk.col_chunks)
    _check(record_property, "colsum", outs[0], scale * xd.sum(0), scale * chain * E * xd.abs().sum(0))

    z = _bf((rows, ld), rows + cols + 1, scale=2.0)
    for hi in (False, True):
        dz = x.clone()
        lo_out = torch.empty(cols // 2 if hi else cols, dtype=BF, device="cuda")
        hi_out = torch.empty(cols // 2, dtype=BF, device="cuda") if hi else None
        assert hk.tpt_gelu_bwd_bias(P(dz), P(z), ld, rows, cols, P(lo_out), P(hi_out), P(part), part.numel()) == 0
        fused = torch.cat([lo_out, hi_out]) if hi else lo_out
        plain = torch.empty(cols, dtype=BF, device="cuda")
        assert hk.tpt_colsum(P(dz), ld, rows, cols, 1.0, P(part), part.numel(), P(plain)) == 0
        assert torch.equal(fused.view(torch.int16), plain.view(torch.int16))
        if cols < ld:
            assert torch.equal(dz[:, cols:], x[:, cols:])          # columns past cols are not written


# ------------------------------------------------------------------------------------------------------------------------------
# transpose
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols", [(1, 7), (45, 33), (1000, 1030), (77, 1)])
def test_transpose_bitwise(hk, rows, cols):
    """out[c, r] = in[r, c] for sizes that are not multiples of the 32 x 32 tile, from a strided input into a strided output; the
    output's padding is left alone."""
    x = _bf((rows, cols + 5), 300 + rows)
    out = torch.full((cols, rows + 3), float("nan"), dtype=BF, device="cuda")
    assert hk.tpt_transpose(P(x), x.stride(0), P(out), out.stride(0), rows, cols) == 0
    assert torch.equal(out[:, :rows].view(torch.int16), x[:, :cols].t().contiguous().view(torch.int16))
    assert bool(out[:, rows:].isnan().all())


# ------------------------------------------------------------------------------------------------------------------------------
# the whole backward at a batch that takes split-K
# ------------------------------------------------------------------------------------------------------------------------------
def test_backward_n32_split_k_against_autograd_and_deterministic(hk):
    """s = 2, n = 32 crops (R = 18432 rows >= the split-K threshold), H = 1024: every parameter gradient against autograd over the
    fp32 torch port (TF32 off), with the gate of test_fullsize_gpu.py::test_gradients_h4096_n8 (1.5 % rel-RMS + a floor for the
    analytically zero k-branch bias gradients); a second forward + backward gives the same bits."""
    from oracle import torch_port
    from tokenpacker_b200 import TokenPackerB200
    from tokenpacker_b200 import synthetic as syn
    n, s, H = 32, 2, 1024
    assert n * 576 >= hk.split_min_rows
    sd = {k: torch.from_numpy(v).to(BF) for k, v in syn.synthetic_state_dict(H, seed=12).items()}
    m = TokenPackerB200(hidden_size=H, scale_factor=s)
    m.load_state_dict(sd)
    m = m.to("cuda", BF).train()
    x0, xm = _bf((n, 576, 1024), 13), _bf((n, 576, 4096), 14)
    gw = _bf((n, 144, H), 15)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        (m((x0, xm)).float() * gw.float()).sum().backward()
        grads.append({k: p.grad.clone() for k, p in m.named_parameters()})
    for k in grads[0]:
        assert torch.equal(grads[0][k].view(torch.int16), grads[1][k].view(torch.int16)), k
    ref_p = {k: v.float().cuda().requires_grad_(True) for k, v in sd.items()}
    ref_out = torch_port.forward(ref_p, x0.float(), xm.float(), s)
    (ref_out * gw.float()).sum().backward()
    worst = {}
    for name, g in grads[0].items():
        gq, r = g.float(), ref_p[name].grad
        assert gq.shape == r.shape and torch.isfinite(gq).all(), name
        worst[name] = (float((gq - r).pow(2).mean().sqrt()), float(r.pow(2).mean().sqrt()))
    floor = 1e-2 * worst["k_proj_1.0.bias"][1]
    bad = {k: (e, r) for k, (e, r) in worst.items() if e > 1.5e-2 * r + floor}
    assert not bad, (bad, worst)
