"""The training step's stages one by one, each against a plain float64 reference of that stage alone.

tp_pack_weights_train, tp_forward_train and tp_backward run through the C ABI on buffers this file owns, and every activation the
forward saves and every intermediate the backward forms is read where it was put (region offsets from ``tpt_train_layout`` in the
test-hook library, tests/csrc/tp_test_hooks.cu).  Each reference starts from the bf16 values the kernels stored for the stage
before, so a stage is checked in isolation:

- forward: q, z_kv and h_kv (the dual epilogue: h_kv = GELU of the fp32 pre-activation), y_k / y_v / y_q and their (mean, M2)
  slots, k' / v' / q' (the folded LayerNorm), ctx, o, z_m and h_m (dual epilogue when H % 256 == 0, else the GELU pass, which must
  equal gelu_fwd_kernel over the stored z_m bit for bit), the output;
- backward: every parameter gradient and every workspace region: the bias gradients as column sums of the stored dY, the weight
  gradients as dY^T X of the stored operands (the split-K ones also bit for bit against the fixed-order reduce of their fp32
  slices), the dgrads, the GELU backward (dz = bf16(bf16(dh) GELU'(z)): its floor carries the rounding of the dh the dgrad
  epilogue stored first), the window-attention backward, the recomputed LayerNorm outputs and the LayerNorm backward.

The references and their floors are those of test_forward_stages_gpu.py and test_train_kernels_gpu.py, imported from there.
Tolerances are derived from the arithmetic, never fitted: |got - ref| <= U |ref| + (1 + U) floor elementwise (U = 2^-8), the floor
being the fp32 error bound (E = 2^-24 per addition of the longest chain) propagated through the stage's operation order.  The
worst ratio error / bound of each check is recorded as a test property (``pytest -o junit_family=legacy --junitxml``) and quoted in
the docstrings, as measured on an H100 (80 GB HBM3, 700 W power limit).  The file runs in about 15 s on that H100.

``saved`` and the backward workspace start as 0xFF bytes (NaN in bf16 and fp32) with a poisoned tail, every gradient as NaN, and
the output is framed by sentinel rows.  After the forward every saved region is finite and the padding, the tail and the sentinel
rows are untouched; after the backward every gradient and every region the backward writes is finite, the padding and the tail are
untouched and ``saved`` is bit-identical to what the forward left; a second backward gives the same bits everywhere.  A stage
that read a buffer before its producer wrote it, or a gradient that was never written, would show up as NaN.  The inference
forward's separate plan (TP_FUSE_ATTN=0) must produce the same bits as the training forward in every region both store.
"""
import ctypes as C
import os

import pytest
import torch

from test_forward_stages_gpu import BF, E, F64, U
from test_forward_stages_gpu import Hooks as ForwardHooks
from test_forward_stages_gpu import _attn_ref as _fwd_attn_ref
from test_forward_stages_gpu import (_bits_equal, _check, _check_q, _check_stats, _forward, _gelu, _gelu_floor, _gemm_floor, _inputs,
                                     _ln_fold_ref, _module, _packed_views, _sample, _state_dict, _stats_ref, _window_rows)
from test_train_kernels_gpu import Hooks as KernelHooks
from test_train_kernels_gpu import _attn_ref as _bwd_attn_ref
from test_train_kernels_gpu import _colsum_chain, _gelu_grad_ref, _ln_apply_ref, _ln_bwd_ref, _reduce_emulated, _splitk

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_testhooks.so")
ALPHA = 0.08838834764831845   # 1 / sqrt(head_dim = 128)
SAVED = ["z_kv", "h_kv", "y_k", "y_v", "stats", "k_p", "v_p", "q", "y_q", "q_p", "ctx", "o", "z_m", "h_m"]
BWD = ["w_m2t", "g_t", "hm_t", "dzm", "d_o", "dctx", "dqp", "dkp", "dvp", "lnq_t", "lnk_t", "lnv_t", "dqh", "dkh", "dvh", "dyq", "dyk",
       "dyv", "dzkv", "ln_part", "col_part", "splitk"]
PARTIALS = ("ln_part", "col_part")   # fp32 partial sums: written in part, and only ever read by the reduce that follows
TAIL = 4096                   # poisoned bytes past the end of saved and of the workspace
GUARD = 3                     # sentinel rows on each side of the output
SENTINEL = 0x5A5A


def _train_layout(n, s, H):
    """tpt_train_layout: ({saved region: (byte offset, byte size)}, {workspace region: (offset, size)}, saved total, workspace total)"""
    import tokenpacker_b200  # noqa: F401  (the product library is loaded next to this one, as in a real process)
    assert os.path.exists(HOOKS), f"{HOOKS} missing: build with `make -C tokenpacker_b200/csrc`"
    fn = C.CDLL(HOOKS).tpt_train_layout
    fn.restype, fn.argtypes = C.c_int, [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int64)]
    o = (C.c_int64 * 74)()
    assert fn(n, s, H, o) == 0
    regions = [(int(o[2 * i]), int(o[2 * i + 1])) for i in range(36)]
    return dict(zip(SAVED, regions[:14])), dict(zip(BWD, regions[14:])), int(o[72]), int(o[73])


@pytest.fixture(scope="module")
def hk():
    return KernelHooks()


@pytest.fixture(scope="module")
def fh():
    return ForwardHooks()


@pytest.fixture(autouse=True)
def _fp64_exact():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    torch.cuda.empty_cache()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Step:
    pass


def _views(buf, layout, shapes):
    """{name: typed view of the region} (None for a region of size 0); shapes: name -> (dtype, shape)"""
    out = {}
    for name, (dt, shape) in shapes.items():
        off, nb = layout[name]
        out[name] = buf[off:off + nb].view(dt).view(shape) if nb else None
    return out


def _untouched_gaps(buf, layout, total):
    """the alignment padding between regions and the poisoned tail still hold 0xFF"""
    spans = sorted(layout.values())
    for (o0, n0), (o1, _) in zip(spans, spans[1:] + [(total + TAIL, 0)]):
        assert o0 + n0 <= o1, ("regions overlap", o0)
        assert bool((buf[o0 + n0:o1] == 0xFF).all()), ("padding after offset", o0)


# ------------------------------------------------------------------------------------------------------------------------------
# one training step on owned buffers
# ------------------------------------------------------------------------------------------------------------------------------
def _train_forward(m, x0, xm):
    """tp_pack_weights_train + tp_forward_train on a poisoned saved buffer; x0 / xm may be crop-strided views"""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    n, s, H = x0.shape[0], m.scale_factor, m.hidden_size
    st = Step()
    st.n, st.s, st.H, st.Mq, st.W = n, s, H, (24 // s) ** 2, s * s
    st.R, st.Q = n * 576, n * st.Mq
    R, Q = st.R, st.Q
    st.params = [p.detach().contiguous() for p in m._raw_params()]
    st.p = {f: t for (f, _), t in zip(_lib.WEIGHT_FIELDS, st.params)}
    st.w = _lib.TpWeights(*[t.data_ptr() for t in st.params])
    pbytes = lib.tp_packed_bytes(H)
    st.packed = torch.empty(pbytes, dtype=torch.uint8, device="cuda")
    _lib.check(lib.tp_pack_weights_train(C.byref(st.w), H, st.packed.data_ptr(), pbytes, _stream()), "tp_pack_weights_train")
    st.SL, st.BL, st.saved_total, st.ws_total = _train_layout(n, s, H)
    assert st.saved_total == lib.tp_train_saved_bytes(n, s, H) and st.ws_total == lib.tp_backward_workspace_bytes(n, s, H)
    st.saved = torch.full((st.saved_total + TAIL,), 0xFF, dtype=torch.uint8, device="cuda")
    st.buf = torch.full((Q + 2 * GUARD, H), SENTINEL, dtype=torch.int16, device="cuda").view(BF)
    st.out = st.buf[GUARD:GUARD + Q]
    assert x0.stride(1) == 1024 and xm.stride(1) == 4096
    torch.cuda.synchronize()
    _lib.check(lib.tp_forward_train(C.byref(st.w), st.packed.data_ptr(), x0.data_ptr(), xm.data_ptr(), n, x0.stride(0), xm.stride(0), s, H,
                                    st.out.data_ptr(), st.saved.data_ptr(), st.saved_total, _stream()), "tp_forward_train")
    torch.cuda.synchronize()
    act, qry = (BF, (R, 1024)), (BF, (Q, 1024))
    st.sv = _views(st.saved, st.SL, {"z_kv": (BF, (R, 2048)), "h_kv": (BF, (R, 2048)), "y_k": act, "y_v": act,
                                     "stats": (torch.float32, (2 * R + Q, 8, 2)), "k_p": act, "v_p": act, "q": qry, "y_q": qry,
                                     "q_p": qry, "ctx": qry, "o": qry, "z_m": (BF, (Q, H)), "h_m": (BF, (Q, H))})
    return st


def _backward(st, gout, xm):
    """tp_backward from st.saved on a poisoned workspace into NaN gradients; returns ({field: gradient}, workspace, region views)"""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    R, Q, H = st.R, st.Q, st.H
    grads = [torch.full_like(t, float("nan")) for t in st.params]
    gs = _lib.TpWeights(*[t.data_ptr() for t in grads])
    ws = torch.full((st.ws_total + TAIL,), 0xFF, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    _lib.check(lib.tp_backward(C.byref(st.w), xm.data_ptr(), 576 * 4096, st.n, st.s, H, gout.data_ptr(), st.saved.data_ptr(), C.byref(gs),
                               ws.data_ptr(), st.ws_total, _stream()), "tp_backward")
    torch.cuda.synchronize()
    Qp = (Q + 7) // 8 * 8
    act, qry = (BF, (R, 1024)), (BF, (Q, 1024))
    b = _views(ws, st.BL, {"w_m2t": (BF, (H, H)), "g_t": (BF, (H, Qp)), "hm_t": (BF, (H, Qp)), "dzm": (BF, (Q, H)), "d_o": qry, "dctx": qry,
                           "dqp": qry, "dkp": act, "dvp": act, "lnq_t": qry, "lnk_t": act, "lnv_t": act, "dqh": qry, "dkh": act, "dvh": act,
                           "dyq": qry, "dyk": act, "dyv": act, "dzkv": (BF, (R, 2048)), "ln_part": (torch.float32, (-1,)),
                           "col_part": (torch.float32, (-1,)), "splitk": (torch.float32, (2, -1, 1024, 1024))})
    return {f: t for (f, _), t in zip(_lib.WEIGHT_FIELDS, grads)}, ws, b


# ------------------------------------------------------------------------------------------------------------------------------
# the forward's stages
# ------------------------------------------------------------------------------------------------------------------------------
def _check_saved_poison(st):
    for k, t in st.sv.items():
        assert bool(torch.isfinite(t.float()).all()), (k, int((~torch.isfinite(t.float())).sum()))
    _untouched_gaps(st.saved, st.SL, st.saved_total)
    g = st.buf.view(torch.int16)
    assert bool((g[:GUARD] == SENTINEL).all()) and bool((g[-GUARD:] == SENTINEL).all())
    assert bool(torch.isfinite(st.out.float()).all())


def _check_forward(record, hk, fh, st, x0, xm):
    s, n, R, Q, W, H = st.s, st.n, st.R, st.Q, st.W, st.H
    v, p = st.sv, {k: t.to(F64) for k, t in st.p.items()}
    _check_saved_poison(st)
    _check_q(record, "q", v["q"], x0, s)
    # z_kv = xm [W_k0; W_v0]^T + b (stored rounded) and h_kv = GELU of the same fp32 value (the dual epilogue)
    rows = _sample(R, 576, 11)
    xr = xm.reshape(R, 4096)[rows].to(F64)
    wkv, bkv = torch.cat([p["k_proj_0_w"], p["v_proj_0_w"]]), torch.cat([p["k_proj_0_b"], p["v_proj_0_b"]])
    z = xr @ wkv.t() + bkv
    fz = _gemm_floor(xr, wkv, bkv)
    _check(record, "z_kv", v["z_kv"][rows], z, fz)
    _check(record, "h_kv", v["h_kv"][rows], _gelu(z), _gelu_floor(z, fz))
    # y_k / y_v from the stored h_kv, y_q from the stored q; statistics of every stored row
    for k, half, wn, bn in (("y_k", 0, "k_proj_2_w", "k_proj_2_b"), ("y_v", 1, "v_proj_2_w", "v_proj_2_b")):
        h = v["h_kv"][rows, half * 1024:(half + 1) * 1024].to(F64)
        _check(record, k, v[k][rows], h @ p[wn].t() + p[bn], _gemm_floor(h, p[wn], p[bn]))
    qs = _sample(Q, st.Mq, 12)
    qd = v["q"][qs].to(F64)
    _check(record, "y_q", v["y_q"][qs], qd @ p["q_proj_w"].t(), _gemm_floor(qd, p["q_proj_w"]))
    st_k, st_v, st_q = _stats_ref(v["y_k"]), _stats_ref(v["y_v"]), _stats_ref(v["y_q"])
    _check_stats(record, "stats_k", v["stats"][:R], st_k)
    _check_stats(record, "stats_v", v["stats"][R:2 * R], st_v)
    _check_stats(record, "stats_q", v["stats"][2 * R:], st_q)
    # k', v', q': the LayerNorm folded into the in-projections (the packed folded weights), q' scaled by 1 / sqrt 128
    w = _packed_views(fh, st)
    ref, floor = _ln_fold_ref(v["y_q"][qs], {a: b[qs] for a, b in st_q.items()}, w["w_iq"], w["c_q"], alpha=ALPHA)
    _check(record, "q_p", v["q_p"][qs], ref, floor)
    rr = _window_rows(s, n)[qs].reshape(-1)
    for k, y, sts, wn, cn in (("k_p", v["y_k"], st_k, "w_ik", "c_k"), ("v_p", v["y_v"], st_v, "w_iv", "c_v")):
        ref, floor = _ln_fold_ref(y[rr], {a: b[rr] for a, b in sts.items()}, w[wn], w[cn])
        _check(record, k, v[k][rr], ref, floor)
    # window attention from the stored q', k', v'
    kk, vv = v["k_p"][rr].view(-1, W, 1024), v["v_p"][rr].view(-1, W, 1024)
    if s in (2, 3, 4):   # window_attn_kernel<S>
        ref, floor, _ = _fwd_attn_ref(v["q_p"][qs], kk, vv, 0.0, 0.0, 20, 2, W + 4, W + 1)
    else:                # window_attn_stream_kernel
        ref, floor, _ = _fwd_attn_ref(v["q_p"][qs], kk, vv, 0.0, 0.0, 20, 2 * W, 3 * W + 4, 2 * W + 1)
    _check(record, "ctx", v["ctx"][qs], ref, floor)
    # o = ctx W_o^T + b_o (no out_proj fold in training), z_m = o W_m0^T + b_m0, h_m = GELU(z_m), out = h_m W_m2^T + b_m2
    cd = v["ctx"][qs].to(F64)
    _check(record, "o", v["o"][qs], cd @ p["out_proj_w"].t() + p["out_proj_b"], _gemm_floor(cd, p["out_proj_w"], p["out_proj_b"]))
    od = v["o"][qs].to(F64)
    zm = od @ p["mlp_0_w"].t() + p["mlp_0_b"]
    fzm = _gemm_floor(od, p["mlp_0_w"], p["mlp_0_b"])
    _check(record, "z_m", v["z_m"][qs], zm, fzm)
    if H % 256 == 0:     # dual epilogue: GELU of the unrounded fp32 pre-activation
        _check(record, "h_m", v["h_m"][qs], _gelu(zm), _gelu_floor(zm, fzm))
    else:                # a GEMM that stores z_m, then gelu_fwd_kernel over the stored z_m
        h = torch.empty_like(v["h_m"])
        assert hk.tpt_gelu_fwd(v["z_m"].data_ptr(), h.data_ptr(), h.numel()) == 0
        torch.cuda.synchronize()
        assert _bits_equal(v["h_m"], h)
    hd = v["h_m"][qs].to(F64)
    _check(record, "out", st.out[qs], hd @ p["mlp_2_w"].t() + p["mlp_2_b"], _gemm_floor(hd, p["mlp_2_w"], p["mlp_2_b"]))


# ------------------------------------------------------------------------------------------------------------------------------
# the backward's stages
# ------------------------------------------------------------------------------------------------------------------------------
def _gelu_bwd_ref(dh, f_dh, z):
    """dz = bf16(dh_s GELU'(z)), dh_s = the bf16 dh the dgrad epilogue stored (within U |dh| + (1 + U) f_dh of the exact dh) and
    re-read by gelu_bwd_colsum_kernel: the floor carries that rounding times |GELU'(z)|, the fp32 error of gelu_grad and the product's
    rounding"""
    gp, f_gp = _gelu_grad_ref(z.to(F64))
    e_dh = U * dh.abs() + (1 + U) * f_dh
    mag = dh.abs() + e_dh
    return dh * gp, e_dh * gp.abs() + mag * f_gp + E * mag * (gp.abs() + f_gp)


def _wgrad_floor(dy, x, alpha=1.0):
    """dW = alpha dY^T X, fp32 over the rows (alpha applied to the sum, then one more rounding)"""
    f = alpha * _gemm_floor(dy.t(), x.t())
    return f + E * alpha * (dy.t().abs() @ x.abs()) if alpha != 1.0 else f


def _check_colsum(record, name, got, x, chain, scale=1.0):
    """bias gradient = bf16(scale * column sums of the stored x)"""
    ref = scale * x.sum(0)
    _check(record, name, got, ref, scale * chain * E * x.abs().sum(0) + (E * ref.abs() if scale != 1.0 else 0.0))


def _check_backward(record, hk, st, g, b, gout, xm):
    s, n, R, Q, H = st.s, st.n, st.R, st.Q, st.H
    v, p = st.sv, {k: t.to(F64) for k, t in st.p.items()}
    cq, cr = _colsum_chain(Q, hk.col_chunks), _colsum_chain(R, hk.col_chunks)
    split = R >= hk.split_min_rows
    rows = _sample(R, 576, 13)
    # mlp.2: out = h_m W_m2^T + b
    G = gout.to(F64)
    _check_colsum(record, "mlp_2_b", g["mlp_2_b"], G, cq)
    hm = v["h_m"].to(F64)
    _check(record, "mlp_2_w", g["mlp_2_w"], G.t() @ hm, _wgrad_floor(G, hm))
    if b["w_m2t"] is not None:   # the transposing fallback of the mlp.2 dgrad (H % 256 != 0): an exact copy of W_m2^T
        assert _bits_equal(b["w_m2t"], st.p["mlp_2_w"].t())
    dh = G @ p["mlp_2_w"]
    _check(record, "dzm", b["dzm"], *_gelu_bwd_ref(dh, _gemm_floor(G, p["mlp_2_w"].t()), v["z_m"]))
    # mlp.0: z_m = o W_m0^T + b
    dz = b["dzm"].to(F64)
    _check_colsum(record, "mlp_0_b", g["mlp_0_b"], dz, cq)
    od = v["o"].to(F64)
    _check(record, "mlp_0_w", g["mlp_0_w"], dz.t() @ od, _wgrad_floor(dz, od))
    _check(record, "d_o", b["d_o"], dz @ p["mlp_0_w"], _gemm_floor(dz, p["mlp_0_w"].t()))
    # out_proj: o = ctx W_o^T + b
    do = b["d_o"].to(F64)
    _check_colsum(record, "out_proj_b", g["out_proj_b"], do, cq)
    cd = v["ctx"].to(F64)
    _check(record, "out_proj_w", g["out_proj_w"], do.t() @ cd, _wgrad_floor(do, cd))
    _check(record, "dctx", b["dctx"], do @ p["out_proj_w"], _gemm_floor(do, p["out_proj_w"].t()))
    # window attention from the stored q', k', v' and dctx
    win = _window_rows(s, n)
    dq, dk, dv, fq, fk, fv = _bwd_attn_ref(v["q_p"], v["k_p"], v["v_p"], b["dctx"], win)
    flat = win.reshape(-1)
    _check(record, "dqp", b["dqp"], dq, fq)
    _check(record, "dkp", b["dkp"][flat], dk, fk)
    _check(record, "dvp", b["dvp"][flat], dv, fv)
    del dq, dk, dv, fq, fk, fv
    # LayerNorm outputs recomputed from the saved statistics
    stats = {"q": v["stats"][2 * R:], "k": v["stats"][:R], "v": v["stats"][R:2 * R]}
    for x in "qkv":
        _check(record, f"ln{x}_t", b[f"ln{x}_t"], *_ln_apply_ref(v[f"y_{x}"], stats[x], st.p[f"ln_{x}_w"], st.p[f"ln_{x}_b"]))
    # MHA in-projections: q' = alpha (LN(y_q) W_iq^T + b_q), k' = LN(y_k) W_ik^T + b_k, v' likewise.  The k slice of the bias
    # gradient is zero analytically (softmax is invariant to a per-query shift of the keys): it is checked as the column sums of
    # the stored dk', so an unwritten slice fails (NaN) and a written one must be the sum of what the attention backward stored.
    dqp, dkp, dvp = (b[k].to(F64) for k in ("dqp", "dkp", "dvp"))
    _check_colsum(record, "in_proj_b_q", g["in_proj_b"][:1024], dqp, cq, ALPHA)
    _check_colsum(record, "in_proj_b_k", g["in_proj_b"][1024:2048], dkp, cr)
    _check_colsum(record, "in_proj_b_v", g["in_proj_b"][2048:], dvp, cr)
    lnq = b["lnq_t"].to(F64)
    _check(record, "in_proj_w_q", g["in_proj_w"][:1024], ALPHA * (dqp.t() @ lnq), _wgrad_floor(dqp, lnq, ALPHA))
    for i, x in ((1, "k"), (2, "v")):
        dyx, lnx = b[f"d{x}p"], b[f"ln{x}_t"]
        got = g["in_proj_w"][i * 1024:(i + 1) * 1024]
        _check(record, f"in_proj_w_{x}", got, dyx.to(F64).t() @ lnx.to(F64), _wgrad_floor(dyx.to(F64), lnx.to(F64)))
        if split:   # the slot was reused by the next stage: recompute the fp32 slices from the same stored operands
            rc, part = _splitk(hk, dyx, lnx, hk.splits)
            assert rc == 0
            assert _bits_equal(got, _reduce_emulated(part, 1.0)), x
    wi = {x: p["in_proj_w"][i * 1024:(i + 1) * 1024] for i, x in enumerate("qkv")}
    ref = ALPHA * (dqp @ wi["q"])
    _check(record, "dqh", b["dqh"], ref, ALPHA * _gemm_floor(dqp, wi["q"].t()) + E * ref.abs())
    for x, d in (("k", dkp), ("v", dvp)):
        _check(record, f"d{x}h", b[f"d{x}h"][rows], d[rows] @ wi[x], _gemm_floor(d[rows], wi[x].t()))
    del dqp, dkp, dvp
    # LayerNorm backward (+ the bias gradients of k_proj_1.2 / v_proj_1.2: the column sums of the stored dy)
    for x, bias in (("q", None), ("k", "k_proj_2_b"), ("v", "v_proj_2_b")):
        refs, chain = _ln_bwd_ref(b[f"d{x}h"], v[f"y_{x}"], stats[x], st.p[f"ln_{x}_w"], hk.ln_blocks)
        _check(record, f"dy{x}", b[f"dy{x}"], *refs["dy"])
        _check(record, f"ln_{x}_w", g[f"ln_{x}_w"], *refs["dgamma"])
        _check(record, f"ln_{x}_b", g[f"ln_{x}_b"], *refs["dbeta"])
        if bias is not None:
            _check_colsum(record, bias, g[bias], b[f"dy{x}"].to(F64), chain)
    # q_proj_1, k_proj_1.2, v_proj_1.2 (against the two column halves of h_kv)
    dyq = b["dyq"].to(F64)
    qd = v["q"].to(F64)
    _check(record, "q_proj_w", g["q_proj_w"], dyq.t() @ qd, _wgrad_floor(dyq, qd))
    for half, x in enumerate("kv"):
        dy, h = b[f"dy{x}"].to(F64), v["h_kv"][:, half * 1024:(half + 1) * 1024].to(F64)
        _check(record, f"{x}_proj_2_w", g[f"{x}_proj_2_w"], dy.t() @ h, _wgrad_floor(dy, h))
        if split:   # the last split-K stage: its fp32 slices are still in the workspace
            assert _bits_equal(g[f"{x}_proj_2_w"], _reduce_emulated(b["splitk"][half], 1.0)), x
        dh = dy[rows] @ p[f"{x}_proj_2_w"]
        ref, floor = _gelu_bwd_ref(dh, _gemm_floor(dy[rows], p[f"{x}_proj_2_w"].t()), v["z_kv"][rows, half * 1024:(half + 1) * 1024])
        _check(record, f"dzkv_{x}", b["dzkv"][rows, half * 1024:(half + 1) * 1024], ref, floor)
    # k_proj_1.0, v_proj_1.0: z = xm W0^T + b
    dzkv = b["dzkv"].to(F64)
    xmd = xm.reshape(R, 4096).to(F64)
    cols = torch.arange(1024, device="cuda")    # output rows: all, or 256 seeded ones when the contraction is long
    if R > 8192:
        cols = torch.randperm(1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(14))[:256]
    for half, x in enumerate("kv"):
        dz = dzkv[:, half * 1024:(half + 1) * 1024]
        _check_colsum(record, f"{x}_proj_0_b", g[f"{x}_proj_0_b"], dz, cr)
        dzc = dz[:, cols]
        _check(record, f"{x}_proj_0_w", g[f"{x}_proj_0_w"][cols], dzc.t() @ xmd, _wgrad_floor(dzc, xmd))


def _check_workspace(st, g, ws, b, split):
    """every gradient finite; every region the backward writes finite, the rest (padding, tail, unused split-K slots, the
    transposes' row padding) still 0xFF"""
    for k, t in g.items():
        assert bool(torch.isfinite(t.float()).all()), (k, int((~torch.isfinite(t.float())).sum()))
    for k, t in b.items():
        if t is None or k in PARTIALS:
            continue
        if k == "splitk" and not split:
            off, nb = st.BL[k]
            assert bool((ws[off:off + nb] == 0xFF).all()), k
            continue
        if k in ("g_t", "hm_t"):      # [H, Qp] transposes of [Q, H] operands: columns Q .. Qp are row padding
            assert bool((t[:, st.Q:].contiguous().view(torch.int16) == -1).all()), k
            t = t[:, :st.Q]
        assert bool(torch.isfinite(t.float()).all()), (k, int((~torch.isfinite(t.float())).sum()))
    _untouched_gaps(ws, st.BL, st.ws_total)


# ------------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------------
_CONFIGS = [
    (2, 4096, 2),     # the released 144-token model at the 7B width
    (4, 5120, 3),     # the 36-token model at the 13B width
    (3, 896, 3),      # H % 256 == 128: GELU pass, mlp.2 transposes + NT dgrad / wgrad, one-CTA kernels, Q = 192
    (24, 160, 3),     # H not a multiple of 64: K / N tails in both mlp GEMMs; Q = 3; stream attention backward over 576 keys
    (1, 256, 1),      # one key per window
    (6, 256, 2),      # stream kernels, 36 keys
    (2, 1024, 29),    # R = 16704 >= the split-K threshold, last slice shorter
    (2, 4096, 64),    # the benchmarked training step: R = 36864, Q = 9216
]


@pytest.mark.parametrize("s,H,n", _CONFIGS)
def test_train_step_stages(hk, fh, record_property, monkeypatch, s, H, n):
    """Forward, backward, confinement and determinism of one training step, and the inference forward's separate plan on the
    same module and inputs: q, h_kv, y_k, y_v, y_q, the statistics, k', v', q' and ctx bit for bit equal to what training saved.
    At n = 29 and 64 the row-wise forward and dgrad checks run on a seeded row sample that holds the first and last row of every 256-row
    block and of every crop, and k/v_proj_1.0's weight gradients on 256 seeded output rows; statistics, poison, the other gradients
    and the column sums cover everything.  At s = 1 (one key per window, p = 1) the gradients of the q and k branches are exactly
    zero, and so is what the kernels produce (ratio 0).
    Measured on an H100, the benchmarked step (s = 2, H = 4096, N = 64): forward: q 0.996, z_kv 0.55, h_kv 0.52, y_k 0.91, y_v 0.93,
    y_q 0.90, statistics 0.05 / 0.23, q' 0.87, k' 0.90, v' 0.90, ctx 0.993, o 0.88, z_m 0.89, h_m 0.86, out 0.58; backward: mlp_2_b
    0.92, mlp_2_w 0.31, dz_m 0.69, mlp_0_b 0.96, mlp_0_w 0.31, d_o 0.64, out_proj_b 0.91, out_proj_w 0.30, dctx 0.91, dq' / dk' / dv'
    0.99 / 0.99 / 0.994, LayerNorm outputs 0.996, in_proj_b q / k / v 0.87 / 0.02 / 0.85, in_proj_w q / k / v 0.34 / 0.07 / 0.07,
    dqh / dkh / dvh 0.91 / 0.90 / 0.89, dy_q / dy_k / dy_v 0.994, ln_q 0.85 / 0.92, ln_k 0.85 / 0.04, ln_v 0.83 / 0.89, k_proj_2_b
    0.43, v_proj_2_b 0.89, q_proj_w 0.31, k_proj_2_w 0.06, v_proj_2_w 0.09, dz_kv 0.87 / 0.87, k_proj_0_b 0.82, v_proj_0_b 0.91,
    k_proj_0_w 0.07, v_proj_0_w 0.07.  Worst error / bound over the other seven configurations: forward: q 0.996, z_kv 0.55, h_kv 0.52, y_k 0.93,
    y_v 0.93, y_q 0.91, statistics 0.05 (means) / 0.23 (M2), q' 0.89, k' 0.91, v' 0.90, ctx 0.994, o 0.91, z_m 0.90, h_m 0.87,
    out 0.985; backward: mlp_2_b 0.98, mlp_2_w 0.994, dz_m 0.97, mlp_0_b 0.99, mlp_0_w 0.996, d_o 0.99, out_proj_b 0.996,
    out_proj_w 0.996, dctx 0.91, dq' 0.99, dk' 0.99, dv' 0.994, LayerNorm outputs 0.996, in_proj_b q / k / v 0.98 / 0.24 / 0.99,
    in_proj_w q / k / v 0.996 / 0.91 / 0.96, dqh / dkh / dvh 0.90 / 0.93 / 0.91, dy_q / dy_k / dy_v 0.994, ln_q weight / bias
    0.99 / 0.995, ln_k 0.94 / 0.27 (the bias gradient is zero analytically), ln_v 0.96 / 0.99, k_proj_2_b 0.86, v_proj_2_b 0.99,
    q_proj_w 0.996, k_proj_2_w 0.90, v_proj_2_w 0.96, dz_kv k / v halves 0.90 / 0.88, k_proj_0_b 0.94, v_proj_0_b 0.98,
    k_proj_0_w 0.91, v_proj_0_w 0.95."""
    m = _module(H, s, _state_dict(H, 200 + s))
    x0, xm = _inputs(n, 210 + s)
    st = _train_forward(m, x0, xm)
    _check_forward(record_property, hk, fh, st, x0, xm)
    split = st.R >= hk.split_min_rows
    assert split == (n in (29, 64))

    gout = torch.randn((st.Q, H), device="cuda", generator=torch.Generator(device="cuda").manual_seed(220 + s)).to(BF)
    saved0 = st.saved.clone()
    g, ws, b = _backward(st, gout, xm)
    assert torch.equal(st.saved, saved0)
    _check_workspace(st, g, ws, b, split)
    _check_backward(record_property, hk, st, g, b, gout, xm)
    g2, ws2, _ = _backward(st, gout, xm)
    assert torch.equal(ws, ws2)
    for k in g:
        assert _bits_equal(g[k], g2[k]), k
    del ws2, g2

    monkeypatch.setenv("TP_FUSE_ATTN", "0")
    r = _forward(fh, m, x0, xm)
    for k in ("q", "h_kv", "y_k", "y_v", "y_q", "k_p", "v_p", "q_p", "ctx"):
        assert _bits_equal(getattr(r, k), st.sv[k]), k
    assert torch.equal(r.stats.view(torch.int32), st.sv["stats"].view(torch.int32))


def test_train_forward_on_clip_views(hk, fh, record_property):
    """[:, 1:] views of CLIP outputs with the class token in row 0 (crop strides 577 x 1024 and 577 x 4096: the 3-D A map feeds
    z_kv): every stage checked, and every saved region and the output equal, bit for bit, those of the same features contiguous.
    Measured on an H100: worst error / bound: q 0.996, z_kv 0.55, h_kv 0.52, y_k 0.92, y_v 0.92, y_q 0.90, statistics 0.03 / 0.22,
    q' 0.87, k' 0.90, v' 0.89, ctx 0.993, o 0.90, z_m 0.89, h_m 0.87, out 0.92."""
    s, H, n = 2, 1024, 3
    m = _module(H, s, _state_dict(H, 230))
    x0, xm = _inputs(n, 240)
    gen = torch.Generator(device="cuda").manual_seed(250)
    f0 = torch.randn((n, 577, 1024), device="cuda", generator=gen).to(BF)
    fm = torch.randn((n, 577, 4096), device="cuda", generator=gen).to(BF)
    f0[:, 1:], fm[:, 1:] = x0, xm
    sv = _train_forward(m, f0[:, 1:], fm[:, 1:])
    assert sv.sv["q"].shape[0] == n * 144
    _check_forward(record_property, hk, fh, sv, x0, xm)
    st = _train_forward(m, x0, xm)
    for k in SAVED:
        assert torch.equal(sv.sv[k].contiguous().view(torch.uint8), st.sv[k].contiguous().view(torch.uint8)), k
    assert _bits_equal(sv.out, st.out)
