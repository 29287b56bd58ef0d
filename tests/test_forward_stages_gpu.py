"""The single-launch forward's stages one by one, each against a plain float64 reference of that stage alone.

The weights are packed through the module (``_packed_weights``); the product library's ``tp_forward`` then runs on a workspace this
file owns, and every stage's output is read where the forward stored it (region offsets from ``tpt_work_layout`` /
``tpt_packed_layout`` in the test-hook library, tests/csrc/tp_test_hooks.cu).  Each reference starts from the bf16 values the kernel
itself stored for the stage before, so a stage is checked in isolation: h_kv, y_k / y_v / y_q and their per-128-column (mean, M2)
slots, q', k' / v' (separate plan only: the fused plan keeps them in registers), the window attention, h_m and the output.

Tolerances are derived from the arithmetic, never fitted, as in test_train_kernels_gpu.py: a stored bf16 result is within U = 2^-8
of the value it rounds, and an fp32 chain of n dependent additions is within n E sum|terms| of the exact sum (E = 2^-24).  Each check
asserts |got - ref| <= U |ref| + (1 + U) floor elementwise (fp32 results: |got - ref| <= floor), the floor being that fp32 bound
propagated through the stage's operation order.  The worst ratio error / bound of each check is recorded as a test property
(``pytest -o junit_family=legacy --junitxml``) and quoted in the docstrings, as measured on an H100 (80 GB HBM3, 700 W power limit).
The file runs in about 45 s on that H100.

Every call runs on a workspace filled with 0xFF bytes (NaN in bf16 and fp32) and writes into an output framed by sentinel rows:
afterwards every region the plan writes must be finite, and the alignment padding between regions, the bytes past the end, the
regions the plan does not use and the sentinel rows must be untouched.  A stage that read a buffer before its producer wrote it
would read NaN, which the caching allocator's reuse of the previous call's block would otherwise hide.
"""
import ctypes as C
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_testhooks.so")
E = 2.0 ** -24            # fp32 unit roundoff
U = 2.0 ** -8             # bf16 unit roundoff
F64 = torch.float64
BF = torch.bfloat16
GELU_LIP = 1.13           # max |GELU'(z)| = 1.1289 (at z = sqrt 2)
EXP_REL = 2.0 ** -21      # __expf: ex2.approx relative error (plus |x| E from rounding its argument, added where used)
REGIONS = ["h_kv", "y_k", "y_v", "k_p", "v_p", "stats", "q", "y_q", "q_p", "ctx", "h_m", "flags"]
PACKED = ["w_kv0", "b_kv0", "w_k2", "b_k2", "w_v2", "b_v2", "w_ik", "wsum_k", "c_k", "w_iv", "wsum_v", "c_v", "w_q", "w_iq", "wsum_q",
          "c_q", "w_ot", "w_om", "b_om", "w_m2", "b_m2", "w_o", "b_o", "w_m0", "b_m0"]
TAIL = 4096               # poisoned bytes past the workspace's end
GUARD = 3                 # sentinel rows on each side of the output
SENTINEL = 0x5A5A


class Hooks:
    def __init__(self):
        from tokenpacker_b200._lib import lib
        assert os.path.exists(HOOKS), f"{HOOKS} missing: build with `make -C tokenpacker_b200/csrc`"
        self.lib = C.CDLL(HOOKS)
        self.lib.tpt_work_layout.restype = C.c_int
        self.lib.tpt_work_layout.argtypes = [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int64)]
        self.lib.tpt_packed_layout.restype = C.c_int
        self.lib.tpt_packed_layout.argtypes = [C.c_int, C.POINTER(C.c_int64)]
        self.tp = lib

    def work_layout(self, n, s, H):
        o = (C.c_int64 * 25)()
        assert self.lib.tpt_work_layout(n, s, H, o) == 0
        return {name: (int(o[2 * i]), int(o[2 * i + 1])) for i, name in enumerate(REGIONS)}, int(o[24])

    def packed_layout(self, H):
        o = (C.c_int64 * 26)()
        assert self.lib.tpt_packed_layout(H, o) == 0
        return {name: int(o[i]) for i, name in enumerate(PACKED)}, int(o[25])


@pytest.fixture(scope="module")
def hk():
    return Hooks()


@pytest.fixture(autouse=True)
def _fp64_exact():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old
    torch.cuda.empty_cache()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


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
    got = got.to(F64)
    assert torch.isfinite(got).all(), name
    ratio = float(((got - ref).abs() / floor.clamp_min(1e-300)).max())
    record(name, f"{ratio:.3g}")
    assert ratio <= 1.0, (name, ratio)
    return ratio


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


# ------------------------------------------------------------------------------------------------------------------------------
# module, inputs, one forward on an owned workspace
# ------------------------------------------------------------------------------------------------------------------------------
def _state_dict(H, seed, kind="plain"):
    """synthetic weights (bf16); ``kind`` selects an adversarial variant of the K/V branch"""
    from tokenpacker_b200 import synthetic as syn
    sd = {k: torch.from_numpy(v) for k, v in syn.synthetic_state_dict(H, seed=seed).items()}
    g = torch.Generator().manual_seed(seed)
    if kind == "bias30":            # y_k / y_v rows with |mean| >> std (mean +-30, std ~0.5): the LayerNorm fold cancels
        for b, sign in (("k_proj_1.2.bias", 1.0), ("v_proj_1.2.bias", -1.0)):
            sd[b] = sign * 30.0 + 0.1 * torch.randn(1024, generator=g)
    elif kind == "gamma0":          # every key of a window gives the same score: p = 1 / W, ctx = the mean of v'
        sd["ln_k_1.weight"] = torch.zeros(1024)
    elif kind == "gamma64":         # logits of several hundred: the softmax saturates to one-hot
        sd["ln_k_1.weight"] = sd["ln_k_1.weight"] * 64
    elif kind == "tinyvar":         # y_k = 2^-10 + O(1e-4): row variance below eps = 1e-6, rstd close to 1000 and set by eps
        sd["k_proj_1.2.weight"] = sd["k_proj_1.2.weight"] * 2.0 ** -12
        sd["k_proj_1.2.bias"] = torch.full((1024,), 2.0 ** -10)
    return {k: v.to(BF) for k, v in sd.items()}


def _module(H, s, sd):
    from tokenpacker_b200 import TokenPackerB200
    m = TokenPackerB200(hidden_size=H, scale_factor=s)
    m.load_state_dict(sd)
    return m.to("cuda", BF).eval()


def _inputs(n, seed):
    x0 = torch.randn((n, 576, 1024), device="cuda", generator=_gen(seed)).to(BF)
    xm = torch.randn((n, 576, 4096), device="cuda", generator=_gen(seed + 1)).to(BF)
    return x0, xm


class Run:
    pass


def _forward(hk, m, x0, xm, packed_rows=0):
    """tp_forward (or tp_forward_packed with packed_rows rows per crop) on a poisoned, test-owned workspace; returns the stage views"""
    lib = hk.tp
    n, s, H = x0.shape[0], m.scale_factor, m.hidden_size
    Mq = (24 // s) ** 2
    R, Q = n * 576, n * Mq
    packed = m._packed_weights(x0.device)
    L, total = hk.work_layout(n, s, H)
    assert total == lib.tp_workspace_bytes(n, s, H)
    ws = torch.full((total + TAIL,), 0xFF, dtype=torch.uint8, device="cuda")
    rows = n * packed_rows if packed_rows else Q
    buf = torch.full((rows + 2 * GUARD, H), SENTINEL, dtype=torch.int16, device="cuda").view(BF)
    out = buf[GUARD:GUARD + rows]
    stream = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    c0 = lib.tp_launch_count()
    if packed_rows:
        st = lib.tp_forward_packed(packed.data_ptr(), x0.data_ptr(), xm.data_ptr(), n, 576 * 1024, 576 * 4096, s, H, out.data_ptr(),
                                   packed_rows, ws.data_ptr(), total, stream)
    else:
        st = lib.tp_forward(packed.data_ptr(), x0.data_ptr(), xm.data_ptr(), n, 576 * 1024, 576 * 4096, s, H, out.data_ptr(), None,
                            ws.data_ptr(), total, stream)
    torch.cuda.synchronize()
    assert st == 0, lib.tp_strerror(st)
    r = Run()
    r.launches = int(lib.tp_launch_count() - c0)
    r.n, r.s, r.H, r.R, r.Q, r.Mq, r.W = n, s, H, R, Q, Mq, s * s
    r.ws, r.L, r.total, r.buf, r.out, r.packed = ws, L, total, buf, out, packed

    def view(name, dtype, shape):
        off, nb = L[name]
        return ws[off:off + nb].view(dtype).view(shape)
    r.h_kv = view("h_kv", BF, (R, 2048))
    for k in ("y_k", "y_v", "k_p", "v_p"):
        setattr(r, k, view(k, BF, (R, 1024)))
    r.stats = view("stats", torch.float32, (2 * R + Q, 8, 2))
    for k in ("q", "y_q", "q_p", "ctx"):
        setattr(r, k, view(k, BF, (Q, 1024)))
    r.h_m = view("h_m", BF, (Q, H))
    r.flags = view("flags", torch.int32, (-1,))
    return r


def _packed_views(hk, r):
    P, total = hk.packed_layout(r.H)
    H = r.H
    shapes = {"w_kv0": (2048, 4096), "b_kv0": (2048,), "w_k2": (1024, 1024), "b_k2": (1024,), "w_v2": (1024, 1024), "b_v2": (1024,),
              "w_ik": (1024, 1024), "wsum_k": (1024,), "c_k": (1024,), "w_iv": (1024, 1024), "wsum_v": (1024,), "c_v": (1024,),
              "w_q": (1024, 1024), "w_iq": (1024, 1024), "wsum_q": (1024,), "c_q": (1024,), "w_om": (H, 1024), "b_om": (H,),
              "w_m2": (H, H), "b_m2": (H,), "w_o": (1024, 1024), "b_o": (1024,), "w_m0": (H, 1024), "b_m0": (H,)}
    assert r.packed.numel() >= total
    w = {}
    for name, shape in shapes.items():
        dt = BF if len(shape) == 2 else torch.float32
        nb = math.prod(shape) * (2 if dt == BF else 4)
        w[name] = r.packed[P[name]:P[name] + nb].view(dt).view(shape)
    return w


def _check_poison(r, fused):
    """every region the plan writes is finite; padding, the tail, unused regions and the output's sentinel rows are untouched"""
    written = [k for k in REGIONS if not (fused and k in ("k_p", "v_p"))]
    for k in written:
        t = getattr(r, k)
        if k == "flags":
            assert bool((t >= 0).all()), k
        else:
            assert bool(torch.isfinite(t.float()).all()), (k, int((~torch.isfinite(t.float())).sum()))
    spans = sorted(r.L.values())
    for (o0, n0), (o1, _) in zip(spans, spans[1:] + [(r.total + TAIL, 0)]):
        assert o0 + n0 <= o1
        assert bool((r.ws[o0 + n0:o1] == 0xFF).all()), ("padding after offset", o0)
    for k in REGIONS:
        if k not in written:
            off, nb = r.L[k]
            assert bool((r.ws[off:off + nb] == 0xFF).all()), k
    g = r.buf.view(torch.int16)
    assert bool((g[:GUARD] == SENTINEL).all()) and bool((g[-GUARD:] == SENTINEL).all())
    assert bool(torch.isfinite(r.out.float()).all())


# ------------------------------------------------------------------------------------------------------------------------------
# float64 references of the stages, with their fp32 error floors
# ------------------------------------------------------------------------------------------------------------------------------
def _sample(total, per, seed, blocks=(256,)):
    """all rows of a small problem; else the first and last row of every block and of every crop plus 256 seeded ones"""
    if total <= 8192:
        return torch.arange(total, device="cuda")
    parts = [torch.randint(0, total, (256,), device="cuda", generator=_gen(seed))]
    for b in tuple(blocks) + (per,):
        st = torch.arange(0, total, b, device="cuda")
        parts += [st, (st + b - 1).clamp_max(total - 1)]
    return torch.unique(torch.cat(parts))


def _gelu(z):
    return z * 0.5 * torch.special.erfc(-z / math.sqrt(2))


def _gemm_floor(a, w, b=None):
    """fp32 accumulation over K (+ the bias add): (K + 1) E sum |a w| (+ |b|)"""
    K = a.shape[1]
    f = (K + 1) * E * (a.abs() @ w.abs().t())
    return f if b is None else f + (K + 1) * E * b.abs()


def _gelu_floor(z, f_z):
    """error of GELU(z) in fp32 from an error f_z in z: GELU' <= 1.13, erf approximation 1.5e-7 |z| + a few roundings, subnormals"""
    return GELU_LIP * (f_z + E * z.abs()) + z.abs() * (1.5e-7 + 4 * E) + 2.0 ** -133


def _stats_ref(y):
    """fp64 per-128-column (mean, M2) of stored bf16 rows y [rows, 1024], the floors of the kernel's fp32 sequence (shift = the
    block's first value; s1 = 64 pair sums, s2 = 128 fmas; mean = shift + s1 / 128, M2 = max(s2 - s1 dm, 0)), and the row LayerNorm
    statistics with the error bounds of ln_row_stats (8-slot Chan combine in fp32, rsqrtf: 2 ulp) built on those floors."""
    yd = y.to(F64).view(-1, 8, 128)
    mean = yd.mean(-1)
    m2 = ((yd - mean[..., None]) ** 2).sum(-1)
    d = yd - yd[..., :1]
    S1, S2, A1 = d.sum(-1), (d * d).sum(-1), d.abs().sum(-1)
    f_s1 = 66 * E * A1                               # y - shift may round (E), 1 pair add + 64 sequential adds
    f_s2 = 131 * E * S2                              # 128 sequential fmas, (y - shift)^2 of a rounded difference
    dm = S1 / 128
    f_dm = f_s1 / 128 + E * dm.abs()
    f_mean = f_dm + E * mean.abs()
    f_m2 = f_s2 + f_s1 * dm.abs() + S1.abs() * f_dm + E * (S2 + f_s2)
    st = {"mean": mean, "m2": m2, "f_mean": f_mean, "f_m2": f_m2}
    # ln_row_stats: t1 = sum of the 8 means (8 adds), mu = t1 / 8; between = sum fma(d, d), d = mean_i - mu; m2 = sum M2_i;
    # var = fma(between, 128, m2) / 1024; rstd = rsqrtf(var + eps)
    mu = mean.mean(-1)
    dmu = (f_mean.sum(-1) + 8 * E * mean.abs().sum(-1)) / 8
    dd = mean - mu[:, None]
    f_d = f_mean + dmu[:, None] + E * dd.abs()
    between = (dd * dd).sum(-1)
    f_between = (2 * dd.abs() * f_d + f_d * f_d).sum(-1) + 8 * E * between
    m2t = m2.sum(-1)
    var = (128 * between + m2t) / 1024
    f_var = (128 * f_between + f_m2.sum(-1) + 8 * E * m2t) / 1024 + 2 * E * var
    st["mu"], st["dmu"] = mu, dmu
    st["rstd"] = 1 / torch.sqrt(var + 1e-6)
    st["rho"] = 0.5 * (f_var + E * (var + 1e-6)) / (var + 1e-6) + 4 * E
    return st


def _check_stats(record, name, got, st):
    _check_f32(record, name + "_mean", got[..., 0], st["mean"], st["f_mean"])
    _check_f32(record, name + "_m2", got[..., 1], st["m2"], st["f_m2"])


def _ln_fold_ref(y, st, w, c, alpha=1.0):
    """alpha (rstd (y . w^T - mu rowsum(w)) + c) in fp64 from the stored y, exact row statistics and the packed folded weights w
    (bf16) and constant c; floor: the accumulation, the kernel's mu / rstd errors, its fp32 wsum (37 E sum|w|: 32 lane adds + 5
    shuffles) times |mu| (the fold's cancellation term), and the two fmas of the epilogue.  Returns (ref, floor) before any bf16
    rounding of the result."""
    yd, wd, cd = y.to(F64), w.to(F64), c.to(F64)
    wsum = wd.sum(1)
    acc = yd @ wd.t()
    pre = acc - st["mu"][:, None] * wsum
    rstd = st["rstd"][:, None]
    val = rstd * pre + cd
    f_inner = 1024 * E * (yd.abs() @ wd.abs().t()) + st["dmu"][:, None] * wsum.abs() + st["mu"].abs()[:, None] * (37 * E * wd.abs().sum(1)) \
        + E * pre.abs()
    f_val = rstd * f_inner + st["rho"][:, None] * rstd * pre.abs() + E * val.abs()
    ref = alpha * val
    return ref, alpha * f_val + (E * ref.abs() if alpha != 1.0 else 0.0)


def _window_rows(s, n):
    """[Q, W] raster token rows of each query's window, key j = (hi, wi) = (j / s, j % s)"""
    G = 24 // s
    q = torch.arange(n * G * G, device="cuda")
    c, m = q // (G * G), q % (G * G)
    hb, wb = m // G, m % G
    j = torch.arange(s * s, device="cuda")
    return c[:, None] * 576 + (hb[:, None] * s + j[None] // s) * 24 + wb[:, None] * s + j[None] % s


def _window_major(s, R):
    """stored row of each raster row in the window-major layout: (crop, hb, wb, hi, wi)"""
    r = torch.arange(R, device="cuda")
    n, t = r // 576, r % 576
    tr, tc = t // 24, t % 24
    G = 24 // s
    return n * 576 + (((tr // s) * G + tc // s) * s + tr % s) * s + tc % s


def _attn_ref(qp, k, v, f_k, f_v, score_chain, exp_terms, sum_terms, acc_terms):
    """8-head single-query attention over W keys in fp64: qp [Q, 1024], k / v [Q, W, 1024] (f_k / f_v: their errors, or 0 for
    stored bf16 values).  Floor: score error d_s = sum|q| f_k + score_chain E sum|q k| (the longest fp32 chain of the dot product);
    |dp_j| <= p_j rho with rho = 2 max d_s + exp_terms (__expf of the arguments) + sum_terms E (denominator, reciprocal, product);
    ctx = sum p v with acc_terms E of fp32 accumulation."""
    Q, W = k.shape[:2]
    q = qp.to(F64).view(Q, 8, 128)
    kd, vd = k.to(F64).view(Q, W, 8, 128), v.to(F64).view(Q, W, 8, 128)
    logit = torch.einsum("qhc,qwhc->qhw", q, kd)
    p = torch.softmax(logit, -1)
    ctx = torch.einsum("qhw,qwhc->qhc", p, vd)
    d_s = score_chain * E * torch.einsum("qhc,qwhc->qhw", q.abs(), kd.abs())
    if not isinstance(f_k, float):
        d_s = d_s + torch.einsum("qhc,qwhc->qhw", q.abs(), f_k.view(Q, W, 8, 128))
    xr = (logit.amax(-1, keepdim=True) - logit.amin(-1, keepdim=True))
    rho = 2 * d_s.amax(-1, keepdim=True) + exp_terms * (EXP_REL + 2 * xr * E) + sum_terms * E
    d_p = p * rho + 2.0 ** -120
    floor = torch.einsum("qhw,qwhc->qhc", d_p, vd.abs()) + acc_terms * E * torch.einsum("qhw,qwhc->qhc", p, vd.abs())
    if not isinstance(f_v, float):
        floor = floor + torch.einsum("qhw,qwhc->qhc", p, f_v.view(Q, W, 8, 128))
    return ctx.reshape(Q, 1024), floor.reshape(Q, 1024), p


def _q_ref(x0, s):
    """point queries: the centre token (odd s) or the mean of the centre 2x2 (even s) in fp64, the device's fp32 sequence
    (0.25a + 0.25b) + (0.25c + 0.25d) rounded to bf16, and 0.25 sum|taps| (None for odd s)"""
    n = x0.shape[0]
    G = 24 // s
    img = x0.view(n, 24, 24, 1024)
    if s % 2:
        c = torch.arange(G, device="cuda") * s + (s - 1) // 2
        v = img[:, c][:, :, c].reshape(-1, 1024)
        return v.to(F64), v, None
    c = torch.arange(G, device="cuda") * s + s // 2 - 1
    a, b, cc, d = (img[:, c + i][:, :, c + j].reshape(-1, 1024) for i in (0, 1) for j in (0, 1))
    exact = (a.to(F64) + b.to(F64) + cc.to(F64) + d.to(F64)) / 4
    emu = ((0.25 * a.float() + 0.25 * b.float()) + (0.25 * cc.float() + 0.25 * d.float())).to(BF)
    return exact, emu, (a.to(F64).abs() + b.to(F64).abs() + cc.to(F64).abs() + d.to(F64).abs()) / 4


def _check_q(record, name, q, x0, s):
    """q bit for bit against the device sequence emulated in fp32, and within 2 fp32 roundings of the exact mean (+ bf16's
    subnormal spacing) after the bf16 rounding"""
    exact, emu, mag = _q_ref(x0, s)
    assert _bits_equal(q, emu), name
    if mag is not None:
        assert torch.isfinite(exact).all()
        _check(record, name, q, exact, 3 * E * mag + 2.0 ** -134)
    return exact


# ------------------------------------------------------------------------------------------------------------------------------
# the stage checks of one forward
# ------------------------------------------------------------------------------------------------------------------------------
def _check_stages(record, hk, r, x0, xm, fused):
    s, R, Q, W, H = r.s, r.R, r.Q, r.W, r.H
    w = _packed_views(hk, r)
    _check_poison(r, fused)
    # [S] point queries
    _check_q(record, "q", r.q, x0, s)
    # [1] h_kv = GELU(xm [W_k0; W_v0]^T + b)
    rows = _sample(R, 576, 11)
    xr = xm.view(R, 4096)[rows].to(F64)
    wkv, bkv = w["w_kv0"].to(F64), w["b_kv0"].to(F64)
    z = xr @ wkv.t() + bkv
    _check(record, "h_kv", r.h_kv[rows], _gelu(z), _gelu_floor(z, _gemm_floor(xr, wkv, bkv)))
    # [2] y_k / y_v (window-major rows in the fused plan, raster rows otherwise), y_q; statistics of every stored row
    perm = _window_major(s, R) if fused else torch.arange(R, device="cuda")
    if fused:
        assert torch.equal(torch.sort(perm).values, torch.arange(R, device="cuda"))
    for k, half, wn, bn in (("y_k", 0, "w_k2", "b_k2"), ("y_v", 1, "w_v2", "b_v2")):
        h = r.h_kv[rows, half * 1024:(half + 1) * 1024].to(F64)
        wd, bd = w[wn].to(F64), w[bn].to(F64)
        _check(record, k, getattr(r, k)[perm[rows]], h @ wd.t() + bd, _gemm_floor(h, wd, bd))
    qd, wq = r.q.to(F64), w["w_q"].to(F64)
    qs = _sample(Q, r.Mq, 12, blocks=(256, max(1, 256 // W)))   # (a KV-attention tile holds the keys of 256 / W queries)
    _check(record, "y_q", r.y_q[qs], qd[qs] @ wq.t(), _gemm_floor(qd[qs], wq))
    st_k, st_v, st_q = _stats_ref(r.y_k), _stats_ref(r.y_v), _stats_ref(r.y_q)
    _check_stats(record, "stats_k", r.stats[:R], st_k)
    _check_stats(record, "stats_v", r.stats[R:2 * R], st_v)
    _check_stats(record, "stats_q", r.stats[2 * R:], st_q)
    # [3]q q' = (LN(y_q) W_iq^T + b) / sqrt 128 with the folded packed weights
    sub = {k: v[qs] for k, v in st_q.items()}
    ref, floor = _ln_fold_ref(r.y_q[qs], sub, w["w_iq"], w["c_q"], alpha=0.08838834764831845)
    _check(record, "q_p", r.q_p[qs], ref, floor)
    # window attention -> ctx
    if fused:
        # the KV-attention tiles: folded LayerNorm of the stored y_k / y_v rows (window-major: query i's keys are rows i W .. i W + W - 1),
        # k' / v' unrounded fp32 in registers, scores against the stored q', softmax over W lanes, p v' summed by a halving exchange
        kv_rows = (qs[:, None] * W + torch.arange(W, device="cuda")[None]).reshape(-1)
        kp, fk = _ln_fold_ref(r.y_k[kv_rows], {k: v[kv_rows] for k, v in st_k.items()}, w["w_ik"], w["c_k"])
        vp, fv = _ln_fold_ref(r.y_v[kv_rows], {k: v[kv_rows] for k, v in st_v.items()}, w["w_iv"], w["c_v"])
        lg = int(math.log2(W))
        ref, floor, p = _attn_ref(r.q_p[qs], kp.view(-1, W, 1024), vp.view(-1, W, 1024), fk, fv, 130, 2, lg + 3, lg + 2)
    else:
        # [3]k/v k', v' (raster rows, stored bf16), then the attention kernel from the stored q', k', v'
        rr = _window_rows(s, r.n)[qs].reshape(-1)
        for k, y, st, wn, cn in (("k_p", r.y_k, st_k, "w_ik", "c_k"), ("v_p", r.y_v, st_v, "w_iv", "c_v")):
            ref_kv, f_kv = _ln_fold_ref(y[rr], {a: b[rr] for a, b in st.items()}, w[wn], w[cn])
            _check(record, k, getattr(r, k)[rr], ref_kv, f_kv)
        kk, vv = r.k_p[rr].view(-1, W, 1024), r.v_p[rr].view(-1, W, 1024)
        if s in (2, 3, 4):   # window_attn_kernel<S>: scores over 8 fmas + 4 shuffles, W exps summed in order, one division
            ref, floor, p = _attn_ref(r.q_p[qs], kk, vv, 0.0, 0.0, 20, 2, W + 4, W + 1)
        else:                # window_attn_stream_kernel: every key may rescale the running sums (corr): one more exp and rounding per key
            ref, floor, p = _attn_ref(r.q_p[qs], kk, vv, 0.0, 0.0, 20, 2 * W, 3 * W + 4, 2 * W + 1)
    _check(record, "ctx", r.ctx[qs], ref, floor)
    # [4] h_m = GELU(ctx (W_m0 W_o)^T + (W_m0 b_o + b_m0))
    cd, wom, bom = r.ctx[qs].to(F64), w["w_om"].to(F64), w["b_om"].to(F64)
    z = cd @ wom.t() + bom
    _check(record, "h_m", r.h_m[qs], _gelu(z), _gelu_floor(z, _gemm_floor(cd, wom, bom)))
    # [5] out = h_m W_m2^T + b_m2
    hd, wm2, bm2 = r.h_m[qs].to(F64), w["w_m2"].to(F64), w["b_m2"].to(F64)
    _check(record, "out", r.out[qs], hd @ wm2.t() + bm2, _gemm_floor(hd, wm2, bm2))
    return p


# ------------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------------
def test_pack(hk, record_property):
    """tp_pack_weights at H = 512: the LayerNorm-folded in-projections equal bf16(W * gamma) bit for bit (a product of two bf16
    values is exact in fp32, so there is one rounding); their row sums (of the rounded values: 32 lane adds + 5 shuffles) and the
    folded constants W beta + b (32 fmas + 5 shuffles + the bias) within their fp32 bounds; the out_proj fold W_m0 W_o (one GEMM,
    K = 1024) and W_m0 b_o + b_m0 (32 fmas + 5 shuffles + the bias); every copied matrix and fp32 bias exact.
    Measured on an H100: worst error / bound: wsum 0.004, c 0.010, w_om 0.88 (its bf16 rounding), b_om 0.007."""
    H = 512
    sd = _state_dict(H, 3)
    m = _module(H, 2, sd)
    sd = {k: v.cuda() for k, v in sd.items()}
    packed = m._packed_weights(torch.device("cuda"))
    torch.cuda.synchronize()
    r = Run()
    r.H, r.packed = H, packed
    w = _packed_views(hk, r)
    win, bin_ = sd["clip_attn.in_proj_weight"], sd["clip_attn.in_proj_bias"]
    for i, x in enumerate("qkv"):
        W, b = win[i * 1024:(i + 1) * 1024], bin_[i * 1024:(i + 1) * 1024]
        gam, bet = sd[f"ln_{x}_1.weight"], sd[f"ln_{x}_1.bias"]
        wi = w[f"w_i{x}"]
        assert _bits_equal(wi, (W.float() * gam.float()).to(BF)), x
        wd = wi.to(F64)
        _check_f32(record_property, f"wsum_{x}", w[f"wsum_{x}"], wd.sum(1), 37 * E * wd.abs().sum(1))
        Wd, bd = W.to(F64), b.to(F64)
        _check_f32(record_property, f"c_{x}", w[f"c_{x}"], Wd @ bet.to(F64) + bd, 38 * E * (Wd.abs() @ bet.to(F64).abs() + bd.abs()))
    wm0, wo = sd["mlp.0.weight"].to(F64), sd["clip_attn.out_proj.weight"].to(F64)
    _check(record_property, "w_om", w["w_om"], wm0 @ wo, 1024 * E * (wm0.abs() @ wo.abs()))
    bo, bm0 = sd["clip_attn.out_proj.bias"].to(F64), sd["mlp.0.bias"].to(F64)
    _check_f32(record_property, "b_om", w["b_om"], wm0 @ bo + bm0, 38 * E * (wm0.abs() @ bo.abs() + bm0.abs()))
    assert _bits_equal(w["w_kv0"], torch.cat([sd["k_proj_1.0.weight"], sd["v_proj_1.0.weight"]]))
    assert torch.equal(w["b_kv0"], torch.cat([sd["k_proj_1.0.bias"], sd["v_proj_1.0.bias"]]).float())
    for mat, src in (("w_k2", "k_proj_1.2.weight"), ("w_v2", "v_proj_1.2.weight"), ("w_q", "q_proj_1.weight"),
                     ("w_o", "clip_attn.out_proj.weight"), ("w_m0", "mlp.0.weight"), ("w_m2", "mlp.2.weight")):
        assert _bits_equal(w[mat], sd[src]), mat
    for vec, src in (("b_k2", "k_proj_1.2.bias"), ("b_v2", "v_proj_1.2.bias"), ("b_o", "clip_attn.out_proj.bias"),
                     ("b_m0", "mlp.0.bias"), ("b_m2", "mlp.2.bias")):
        assert torch.equal(w[vec], sd[src].float()), vec


_FUSED = [(2, 1, 256), (4, 1, 256), (2, 3, 512), (4, 3, 512), (4, 7, 5120), (2, 64, 4096)]


@pytest.mark.parametrize("s,n,H", _FUSED)
def test_fused_forward_stages(hk, record_property, monkeypatch, s, n, H):
    """The fused plan (s = 2, 4): ONE launch (tp_launch_count + 1) computes the point queries as front work, [1] - [5] ordered by
    tile counters, y_k / y_v stored window-major, and the window attention as the epilogue of the K/V in-projections.  n = 1 has
    R = 576 and Q < 256 rows: every stage ends in a partial tile.  At n = 64 the GEMM stages are checked on a seeded row sample that
    holds the first and last row of every 256-row block and of every crop; point queries, statistics and the poison / canary checks
    cover every row.  n = 3 also runs tp_forward_packed: the same bits with one sentinel row left between crops.
    Measured on an H100: worst error / bound over the six configurations: q 0.996, h_kv 0.53, y_k 0.94, y_v 0.93, y_q 0.90,
    statistics 0.05 (means) / 0.24 (M2), q' 0.87, ctx 0.31 (k' and v' are unrounded fp32 here), h_m 0.87, out 0.98."""
    monkeypatch.delenv("TP_FUSE_ATTN", raising=False)
    sd = _state_dict(H, 20 + s)
    m = _module(H, s, sd)
    x0, xm = _inputs(n, 30 + n * s)
    r = _forward(hk, m, x0, xm)
    assert r.launches == 1
    _check_stages(record_property, hk, r, x0, xm, fused=True)
    if n == 3:
        rp = _forward(hk, m, x0, xm, packed_rows=r.Mq + 1)
        assert rp.launches == 1
        _check_poison(rp, fused=True)
        o = rp.out.view(n, r.Mq + 1, H)
        assert _bits_equal(o[:, :r.Mq], r.out.view(n, r.Mq, H))
        assert bool((o[:, r.Mq].contiguous().view(torch.int16) == SENTINEL).all())


@pytest.mark.parametrize("s,n", [(2, 3), (4, 3), (3, 2), (1, 1), (6, 2), (24, 3)])
def test_separate_plan_stages(hk, record_property, monkeypatch, s, n):
    """TP_FUSE_ATTN=0 and the scale factors without a fused plan: chain [1] [2] [3] with k' and v' in memory (checked too), then
    window_attn_kernel<2|3|4> or window_attn_stream_kernel (s = 1, 6, 24: 1 to 576 keys, online softmax), then [4] [5].
    Measured on an H100: worst error / bound: k' 0.90, v' 0.90, ctx 0.994 (register kernels), 0.96 (stream kernel; 0 at s = 1,
    where p = 1); the other stages as in the fused test."""
    monkeypatch.setenv("TP_FUSE_ATTN", "0")
    H = 256
    m = _module(H, s, _state_dict(H, 40 + s))
    x0, xm = _inputs(n, 50 + s)
    r = _forward(hk, m, x0, xm)
    assert r.launches >= 3
    _check_stages(record_property, hk, r, x0, xm, fused=False)


@pytest.mark.parametrize("kind", ["bias30", "gamma0", "gamma64", "tinyvar"])
@pytest.mark.parametrize("s,fuse", [(2, True), (4, True), (2, False)])
def test_adversarial_weights(hk, record_property, monkeypatch, kind, s, fuse):
    """K/V-branch weights where the folded LayerNorm and the softmax are stressed, through both fused plans and the separate one:
    biases +-30 (|mean| >> std: the floor carries the fold's cancellation term rstd |mu| sum|gamma W|); ln_k weight 0 (all scores of
    a window equal: p = 1 / W exactly, ctx = the mean of v'); ln_k weight x 64 (logits of several hundred: p one-hot); k_proj_1.2
    weight x 2^-12 over a constant bias (row variance at or near eps, rstd up to 1000).  Everything stays finite.
    Measured on an H100: worst error / bound: y_k 0.97, k' 0.97, ctx 0.995 (separate plan), 0.82 (fused, all-equal logits), 0.26
    (fused, variance below eps); for |mean| >> std and saturated logits the fused ctx bound is loose (0.006, 0.008): it carries the
    error of the unrounded k', which holds the fold's cancellation or a 64x gamma, times |q'| into every logit."""
    if fuse:
        monkeypatch.delenv("TP_FUSE_ATTN", raising=False)
    else:
        monkeypatch.setenv("TP_FUSE_ATTN", "0")
    H, n = 256, 2
    m = _module(H, s, _state_dict(H, 60, kind))
    x0, xm = _inputs(n, 70 + s)
    r = _forward(hk, m, x0, xm)
    assert (r.launches == 1) == fuse
    p = _check_stages(record_property, hk, r, x0, xm, fused=fuse)
    if kind == "gamma0":
        assert torch.equal(p, torch.full_like(p, 1.0 / r.W))
    if kind == "gamma64":
        assert float(p.amax(-1).median()) > 0.99
    if kind == "tinyvar":
        assert float(_stats_ref(r.y_k)["rstd"].min()) > 500
    if kind == "bias30":
        for y in (r.y_k, r.y_v):
            st = _stats_ref(y)
            assert float((st["mu"].abs() * st["rstd"]).min()) > 10


def _wide_x0(n, seed):
    """x0 of random finite bf16 values over every binade (subnormals and zeros included, both signs); the centre 2x2 taps of the
    first 8 windows of crop 0 in bf16's top binade (|x| >= 2^127) with equal and mixed signs"""
    bits = torch.randint(0, 1 << 16, (n, 576, 1024), device="cuda", generator=_gen(seed), dtype=torch.int32)
    bits = torch.where((bits & 0x7F80) == 0x7F80, bits & 0x807F, bits)
    x0 = bits.to(torch.int16).view(BF)
    top = torch.randint(0x7F00, 0x7F80, (8, 4, 1024), device="cuda", generator=_gen(seed + 1), dtype=torch.int32)
    sign = torch.tensor([[0, 0, 0, 0], [1, 1, 1, 1], [0, 1, 0, 1], [0, 0, 1, 0], [1, 0, 0, 1], [0, 0, 0, 1], [1, 1, 0, 0], [0, 1, 1, 1]],
                        device="cuda", dtype=torch.int32)
    top = (top | (sign[..., None] << 15)).to(torch.int16).view(BF)
    return x0, top


@pytest.mark.parametrize("impl", ["chained", "point_query_kernel"])
@pytest.mark.parametrize("s", [1, 2, 3, 4, 6, 8, 12, 24])
def test_point_queries(hk, record_property, monkeypatch, s, impl):
    """Both implementations of the point-query stencil: the front work of a chained launch (the fused plan for s = 2, 4; the
    separate plan's chain otherwise: TP_GEMM_MODE=2 puts every GEMM on pair tiles) and point_query_kernel (TP_CHAIN=0: every stage
    launched on its own); the launch count tells which ran.  Odd s: a bit-exact copy of the centre token.  Even s: on randn taps the
    round-to-nearest-even of the exact mean, bit for bit; on taps from every bf16 binade, subnormals and top-binade windows with mixed
    signs, finite and within 2 fp32 roundings of 0.25 sum|taps| plus bf16's subnormal spacing.  Only q is checked here: such inputs
    overflow the stages after it.  Measured on an H100: worst error / bound 0.996 (randn and wide-range taps alike: the bf16
    rounding)."""
    monkeypatch.delenv("TP_FUSE_ATTN", raising=False)
    if impl == "chained":
        monkeypatch.setenv("TP_GEMM_MODE", "2")
    else:
        monkeypatch.setenv("TP_CHAIN", "0")
    H, n = 256, 1
    m = _module(H, s, _state_dict(H, 80))
    x0, xm = _inputs(n, 90 + s)
    r = _forward(hk, m, x0, xm)
    if impl == "chained":
        assert r.launches == (1 if s in (2, 4) else 3)
    else:
        assert r.launches >= 7
    _check_q(record_property, "q_randn", r.q, x0, s)
    x0w, top = _wide_x0(n, 100 + s)
    if s % 2 == 0:
        G = 24 // s
        img = x0w.view(n, 24, 24, 1024)
        for k in range(min(8, G * G)):
            hb, wb = k // G, k % G
            r0, c0 = hb * s + s // 2 - 1, wb * s + s // 2 - 1
            img[0, r0, c0], img[0, r0, c0 + 1], img[0, r0 + 1, c0], img[0, r0 + 1, c0 + 1] = top[k]
    r = _forward(hk, m, x0w, xm)
    _check_q(record_property, "q_wide", r.q, x0w, s)
