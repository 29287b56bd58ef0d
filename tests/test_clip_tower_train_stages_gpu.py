"""The CLIP tower's layer backward (tp_clip_tower_train.inl, ``run_clip_layer_backward``) step by step, each step against a plain
float64 reference of that step alone.

``tptt_layer_backward`` (tests/csrc/tp_clip_tower_train_hooks.cu) runs one layer's backward up to step s (1 fc2, 2 quick_gelu
backward, 3 fc1, 4 layer_norm2, 5 out_proj, 6 attention, 7 q/k/v, 8 layer_norm1: the numbering of the .inl's header) on a workspace
this file owns, from a saved set of ``tp_clip_tower_forward_train``.  The workspace aliases its intermediates (dh -> dz -> dqkv; g =
d LN2 -> dctx -> d LN1; the carry updated in place), so every step s is run afresh from the top, and its reference starts from the
bf16 / fp32 values the run to s - 1 left (the runs are deterministic: checked), so a step is checked in isolation.  Every byte a step
does not own (other regions, alignment padding, the poisoned tail, gradients of later steps, the sentinel gaps between gradients)
must keep the bits the run to s - 1 left.

Tolerances are derived from the arithmetic, as in test_train_stages_gpu.py: |got - ref| <= U |ref| + (1 + U) floor elementwise
(U = 2^-8; fp32 results: |got - ref| <= floor), the floor being the fp32 bound (E = 2^-24 per addition of the longest chain)
propagated through the step's operation order.  NN dgrads are checked on the row samples of test_forward_stages_gpu.py (every row
up to 14 crops), weight gradients over their full contractions, the attention backward on three crops.  The worst ratio error /
bound of each check is recorded as a test property (``pytest -o junit_family=legacy --junitxml``) and quoted in the docstrings, as
measured on an H100 (80 GB HBM3, 700 W power limit).

Batches: N = 1 (577 rows: fewer rows than the 592 column-sum chunks, most of the 296 LayerNorm blocks idle), N = 28 (16156 rows, the
last batch without split-K), N = 29 (16733 rows = 261 * 64 + 29: the first with split-K, whose last slice ends in a 29-row k-block),
the latter also on weights with outlier residual channels; and N = 3 with a caller gradient of the layer's input and an fp32 carry
that bf16 cannot represent.  The file runs in about 6 s on that H100 (plus the torch import), at a peak of 8.2 GB allocated.

Measured on an H100, worst error / bound over the five configurations: fc2_b 0.94, fc2_w 0.96, dh 0.91, dz 0.996, fc1_b 0.97,
fc1_w 0.96, d LN2 0.59, carry after layer_norm2 0.49, ln2_w 0.91, ln2_b 0.96, o_b 0.98, dctx 0.91, o_w 0.93 (its split-K slices
0.0035), delta 0.10, dqkv 0.29 (rel-RMS per head 0.70 U, 1.6 U on the outlier weights), q_b 0.94, q_w 0.95, k_b 0.68, k_w 0.96,
v_b 0.98, v_w 0.99 (q / k / v slices 0.0026 / 0.0042 / 0.12), d LN1 0.70, carry after layer_norm1 0.95, ln1_w 0.97, ln1_b 0.98.
A ratio close to 1 is the bf16 rounding of the result taking up the whole U |ref| term; the slices are fp32 against a worst-case
chain bound.
"""
import ctypes as C
import math
import os

import pytest
import torch

from oracle import clip_tower_oracle as cto
from test_forward_stages_gpu import BF, E, EXP_REL, F64, U, _check, _check_f32, _gemm_floor, _sample
from test_train_kernels_gpu import _colsum_chain, _reduce_emulated, _slices
from test_train_stages_gpu import _check_colsum, _wgrad_floor

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_clip_tower_train_hooks.so")
REGIONS = ("carry32", "carry16", "dh", "g", "delta", "ln_part", "col_part", "splitk", "unused_grad")
SAVED = ("pack", "x", "y1", "qkv", "lse", "ctx", "xp", "y2", "z", "h")
LN_BLOCKS, COL_CHUNKS, SPLITS = 296, 592, 4     # tp_train.inl: kLnBlocks, kColChunks, kWgradSplits
SPLIT_MIN_ROWS = 64 * 64 * SPLITS               # wgrad_split_pays: 577 N >= 16384, N >= 29
TAIL = 4096                                     # poisoned bytes past the end of saved and of the workspace
GAP = 8                                         # sentinel bf16 elements before, between and after the gradient views (16 bytes)
SENTINEL = 0x5A5A
NAN16 = 0x7FC0                                  # bf16 quiet NaN
LOG2E = 1.0 / math.log(2.0)
GRAD_SHAPES = {"ln1_w": (1024,), "ln1_b": (1024,), "q_w": (1024, 1024), "q_b": (1024,), "k_w": (1024, 1024), "k_b": (1024,),
               "v_w": (1024, 1024), "v_b": (1024,), "o_w": (1024, 1024), "o_b": (1024,), "ln2_w": (1024,), "ln2_b": (1024,),
               "fc1_w": (4096, 1024), "fc1_b": (4096,), "fc2_w": (1024, 4096), "fc2_b": (1024,)}
# what each step writes: gradients, and workspace regions (splitk only on the split-K path)
STEP_GRADS = {1: ("fc2_b", "fc2_w"), 2: ("fc1_b",), 3: ("fc1_w",), 4: ("ln2_w", "ln2_b", "o_b"), 5: ("o_w",), 6: (),
              7: ("q_b", "k_b", "v_b", "q_w", "k_w", "v_w"), 8: ("ln1_w", "ln1_b")}
STEP_REGIONS = {1: ("dh", "col_part"), 2: ("dh", "col_part"), 3: ("g",), 4: ("carry32", "carry16", "ln_part"), 5: ("g", "splitk"),
                6: ("delta", "dh"), 7: ("col_part", "g", "splitk"), 8: ("carry32", "carry16", "ln_part")}


@pytest.fixture(scope="module")
def hooks():
    import tokenpacker_b200  # noqa: F401  (the product library is loaded next to this one, as in a real process)
    from tokenpacker_b200 import _lib
    assert os.path.exists(HOOKS), f"{HOOKS} missing: build with `make -C tokenpacker_b200/csrc`"
    lib = C.CDLL(HOOKS)
    p, i64 = C.c_void_p, C.c_int64
    for name, args in {"tptt_saved_offsets": [i64, C.POINTER(i64)], "tptt_bwd_offsets": [i64, C.POINTER(i64)],
                       "tptt_layer_backward": [C.POINTER(_lib.TpClipTowerWeights), C.c_int, p, i64, p,
                                               C.POINTER(_lib.TpClipTowerLayerGrads), p, C.c_size_t, C.c_int, p]}.items():
        getattr(lib, name).restype = C.c_int
        getattr(lib, name).argtypes = args
    return lib


@pytest.fixture(autouse=True)
def _fp64_exact():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old
    torch.cuda.empty_cache()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(torch.uint8)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------------------
# one forward, and the backward of one layer up to a step, on owned buffers
# ------------------------------------------------------------------------------------------------------------------------------
class Case:
    pass


def _model(seed, outlier):
    w = cto.make_weights(23, seed=seed, outlier=outlier, device=DEV)
    return cto.FakeCLIPVisionModel({k: v.to(BF) for k, v in w.items()})


def _forward(hooks, model, images, k=2):
    """tp_clip_tower_forward_train of the last k layers on a poisoned saved buffer; views of every saved set"""
    from tokenpacker_b200 import CLIPVisionTowerB200, _lib
    lib = _lib.lib
    c = Case()
    c.n = n = images.shape[0]
    c.M = M = n * 577
    c.k = k
    c.tower = CLIPVisionTowerB200(model)
    c.packed, (c.w, _) = c.tower._packed_weights(torch.device(DEV))
    c.outs = [torch.empty(n, 577, 1024, dtype=BF, device=DEV) for _ in range(4)]
    c.saved_bytes = lib.tp_clip_tower_train_saved_bytes(n, k)
    fwd_bytes = lib.tp_clip_tower_train_workspace_bytes(n, k)
    c.saved = torch.full((c.saved_bytes + TAIL,), 0xFF, dtype=torch.uint8, device=DEV)
    fws = torch.full((fwd_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
    ptrs = (C.c_void_p * 4)(*[o.data_ptr() for o in c.outs])
    _lib.check(lib.tp_clip_tower_forward_train(c.packed.data_ptr(), C.byref(c.w), images.data_ptr(), n, images.stride(0), k, ptrs,
                                               c.saved.data_ptr(), c.saved_bytes, fws.data_ptr(), fwd_bytes, _stream()),
               "tp_clip_tower_forward_train")
    torch.cuda.synchronize()
    del fws
    so = (C.c_int64 * 12)()
    assert hooks.tptt_saved_offsets(n, so) == 0
    c.so = dict(zip(SAVED + ("bytes", "w_qkv"), (int(v) for v in so)))
    assert c.saved_bytes == k * c.so["bytes"]
    bo = (C.c_int64 * 10)()
    assert hooks.tptt_bwd_offsets(n, bo) == 0
    c.bo = dict(zip(REGIONS + ("total",), (int(v) for v in bo)))
    assert c.bo["total"] == lib.tp_clip_tower_backward_workspace_bytes(n, k)
    c.sizes = {"carry32": M * 4096, "carry16": M * 2048, "dh": M * 8192, "g": M * 2048, "delta": n * 16 * 640 * 4,
               "ln_part": LN_BLOCKS * 3 * 1024 * 4, "col_part": COL_CHUNKS * 4096 * 4, "splitk": 3 * SPLITS * 1024 * 1024 * 4,
               "unused_grad": 3 * 1024 * 2}
    spans = sorted((c.bo[r], c.sizes[r]) for r in REGIONS)
    assert all(o0 + n0 <= o1 for (o0, n0), (o1, _) in zip(spans, spans[1:] + [(c.bo["total"], 0)]))
    c.sets = [_saved_views(c, t) for t in range(k)]
    return c


def _saved_views(c, t):
    base, o, M = t * c.so["bytes"], c.so, c.M

    def v(name, shape, dtype=BF, extra=0):
        nb = math.prod(shape) * torch.empty(0, dtype=dtype).element_size()
        return c.saved[base + o[name] + extra: base + o[name] + extra + nb].view(dtype).view(shape)
    s = {"ptr": c.saved.data_ptr() + base, "x": v("x", (M, 1024)), "y1": v("y1", (M, 1024)), "qkv": v("qkv", (M, 3072)),
         "lse": v("lse", (c.n, 16, 640), torch.float32), "ctx": v("ctx", (M, 1024)), "xp": v("xp", (M, 1024), torch.float32),
         "y2": v("y2", (M, 1024)), "z": v("z", (M, 4096)), "h": v("h", (M, 4096)), "w_qkv": v("pack", (3072, 1024), extra=o["w_qkv"])}
    return s


def _layer_params(model, layer):
    named = dict(model.named_parameters())
    return {f: named[f"vision_model.encoder.layers.{layer}.{key}"].detach() for f, key in _field_keys()}


def _field_keys():
    from tokenpacker_b200 import _lib
    return _lib.CLIP_TOWER_LAYER_FIELDS


def _grad_buffer(skip=()):
    """one NaN-filled bf16 buffer holding the 16 gradient views, framed by sentinel gaps; the struct (NULL for ``skip``)"""
    from tokenpacker_b200 import _lib
    total = sum(math.prod(s) for s in GRAD_SHAPES.values()) + GAP * (len(GRAD_SHAPES) + 1)
    buf = torch.full((total,), SENTINEL, dtype=torch.int16, device=DEV)
    views, gaps, off = {}, [(0, GAP)], GAP
    for f, shape in GRAD_SHAPES.items():
        nel = math.prod(shape)
        buf[off:off + nel] = NAN16
        views[f] = buf[off:off + nel].view(BF).view(shape)
        off += nel
        gaps.append((off, off + GAP))
        off += GAP
    struct = _lib.TpClipTowerLayerGrads(*[None if f in skip else views[f].data_ptr() for f, _ in _field_keys()])
    return buf, views, gaps, struct


class Run:
    pass


def _ws_views(c, ws):
    M, n, bo = c.M, c.n, c.bo
    r = {}
    r["carry32"] = ws[bo["carry32"]: bo["carry32"] + M * 4096].view(torch.float32).view(M, 1024)
    r["carry16"] = ws[bo["carry16"]: bo["carry16"] + M * 2048].view(BF).view(M, 1024)
    r["dh"] = ws[bo["dh"]: bo["dh"] + M * 8192].view(BF).view(M, 4096)
    r["dqkv"] = ws[bo["dh"]: bo["dh"] + M * 6144].view(BF).view(M, 3072)
    r["g"] = ws[bo["g"]: bo["g"] + M * 2048].view(BF).view(M, 1024)
    r["delta"] = ws[bo["delta"]: bo["delta"] + n * 16 * 640 * 4].view(torch.float32).view(n, 16, 640)
    r["splitk"] = ws[bo["splitk"]: bo["splitk"] + c.sizes["splitk"]].view(torch.float32).view(3, SPLITS, 1024, 1024)
    return r


def _backward(hooks, c, layer, t, carry32, d_x, last_step, skip=(), ws=None):
    """tptt_layer_backward of ``layer`` from saved set t up to last_step, on a fresh poisoned workspace whose carry is carry32 (and
    carry16 = bf16(carry32)); ws: continue on this workspace and its carry instead"""
    r = Run()
    if ws is None:
        ws = torch.full((c.bo["total"] + TAIL,), 0xFF, dtype=torch.uint8, device=DEV)
        v = _ws_views(c, ws)
        v["carry32"].copy_(carry32)
        v["carry16"].copy_(carry32.to(BF))
    r.ws = ws
    r.gbuf, r.g, r.gaps, struct = _grad_buffer(skip)
    torch.cuda.synchronize()
    rc = hooks.tptt_layer_backward(C.byref(c.w), layer, c.sets[t]["ptr"], c.n, None if d_x is None else d_x.data_ptr(), C.byref(struct),
                                   ws.data_ptr(), c.bo["total"], last_step, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    r.v = _ws_views(c, ws)
    return r


def _product_backward(c, k, d_outs, saved_ptr):
    """tp_clip_tower_backward over the last k layers on a fresh poisoned workspace: (workspace, [(grad buffer, views)] per layer)"""
    from tokenpacker_b200 import _lib
    ws = torch.full((c.bo["total"] + TAIL,), 0xFF, dtype=torch.uint8, device=DEV)
    gb = [_grad_buffer() for _ in range(k)]
    structs = (_lib.TpClipTowerLayerGrads * k)(*[b[3] for b in gb])
    d_ptrs = (C.c_void_p * 4)(*[None if d is None else d.data_ptr() for d in d_outs])
    torch.cuda.synchronize()
    _lib.check(_lib.lib.tp_clip_tower_backward(C.byref(c.w), saved_ptr, c.n, k, d_ptrs, structs, ws.data_ptr(), c.bo["total"], _stream()),
               "tp_clip_tower_backward")
    torch.cuda.synchronize()
    return ws, [(b[0], b[1]) for b in gb]


# ------------------------------------------------------------------------------------------------------------------------------
# float64 references of the steps, with their fp32 error floors
# ------------------------------------------------------------------------------------------------------------------------------
def _quick_gelu_grad_ref(z):
    """quick_gelu'(z) = s (1 + 1.702 z (1 - s)), s = sigmoid(1.702 z), and a bound of quick_gelu_grad's fp32 error: the argument of
    __expf off by |1.702 z| 3 E (1.702f, the product, the log2 e scaling), EXP_REL for ex2.approx; s = 1 / (1 + e) then has relative
    error (1 - s) rho + 2 E, which carries into 1 - s and the product; each further operation rounds once (E)"""
    zd = z.to(F64)
    s = torch.sigmoid(1.702 * zd)
    t = 1.702 * zd * (1 - s)
    gp = s * (1 + t)
    rho = EXP_REL + 3 * E * 1.702 * zd.abs()
    ds = s * ((1 - s) * rho + 2 * E)
    d1s = ds + E * (1 - s)
    f_gp = ds * (1 + t).abs() + s * 1.702 * zd.abs() * d1s + 4 * E * s * (1 + t.abs()) + 2.0 ** -126
    return gp, f_gp


def _ln_bwd_ref(gy, x, gamma, rows_total):
    """clip_ln_bwd_kernel's dLN = rstd (gg - mean(gg) - xhat mean(gg xhat)), gg = gamma g, from the bf16 g and the LayerNorm input x
    (fp32 x' or bf16 x) whose statistics the kernel recomputes, with its fp32 floor; and dgamma / dbeta with theirs.  Row sums: 32
    sequential lane adds + 5 shuffle levels (48 E as in test_train_kernels_gpu.py's LayerNorm); the variance from the rounded
    deviations; rsqrtf 2 ulp.  Column sums: rows-per-warp + 8 warps + 19 + 16 lane partials (ln_param_reduce_kernel)."""
    xd, g, gm = x.to(F64), gy.to(F64), gamma.to(F64)
    mu = xd.mean(-1, keepdim=True)
    e = xd - mu
    var = (e * e).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + 1e-5)
    xh = e * rstd
    dmu = 48 * E * xd.abs().mean(-1, keepdim=True)
    de = E * e.abs() + dmu                                                  # error of each fp32 deviation x - mean
    dvar = 48 * E * var + (2 * e.abs() * de + de * de).mean(-1, keepdim=True) + E * (var + 1e-5)
    rho = 0.5 * dvar / (var + 1e-5) + 4 * E                                 # relative error of rstd
    dyh = rstd * de + xh.abs() * (rho + 2 * E)                              # error of each xhat
    gg = gm * g
    c1, c2 = gg.mean(-1, keepdim=True), (gg * xh).mean(-1, keepdim=True)
    ref = rstd * (gg - c1 - xh * c2)
    dc1 = 48 * E * gg.abs().mean(-1, keepdim=True)
    dc2 = 48 * E * (gg * xh).abs().mean(-1, keepdim=True) + (gg.abs() * dyh).mean(-1, keepdim=True)
    floor = rstd * (dc1 + xh.abs() * dc2 + c2.abs() * dyh) + (rho + 4 * E) * rstd * (gg.abs() + c1.abs() + (xh * c2).abs())
    warps = LN_BLOCKS * 8
    chain = (rows_total + warps - 1) // warps + 8 + (LN_BLOCKS + 15) // 16 + 16 + 2
    return ref, floor, {"dgamma": ((g * xh).sum(0), chain * E * (g * xh).abs().sum(0) + (g.abs() * dyh).sum(0)),
                        "dbeta": (g.sum(0), chain * E * g.abs().sum(0))}, chain


def _attn_bwd_ref(qkv, lse, ctx, dctx, crop):
    """dq | dk | dv [577, 3072] of one crop in fp64 from the stored qkv (q pre-scaled), LSE (log2), ctx and dctx, with
    P = exp2(S log2 e - LSE) and D = rowsum(dctx o ctx), and the floor of clip_attn_bwd_kernel's arithmetic:
      S, dP: fp32 wgmma over 64 channels (65 E sum|.|); D: clip_attn_delta_kernel's 8 fmas + 3 shuffles (12 E);
      P relative error eps_p = ln 2 (log2 e (f_S + E |S|) + E |arg|) + EXP_REL (the fma forming the argument, ex2.approx);
      dS = P (dP - D) rounded once in fp32, then to bf16 (U) before dQ = dS K and dK = dS^T Q; P rounded to bf16 before dV = P^T dO;
      the products accumulate in fp32 over 640 columns (641 E sum|.|); the final bf16 rounding is the check's U |ref|."""
    rows = slice(crop * 577, (crop + 1) * 577)
    x = qkv[rows].to(F64).view(577, 3, 16, 64).permute(1, 2, 0, 3)
    q, k, v = x[0], x[1], x[2]
    do = dctx[rows].to(F64).view(577, 16, 64).transpose(0, 1)
    o = ctx[rows].to(F64).view(577, 16, 64).transpose(0, 1)
    L = lse[crop, :, :577].to(F64)[..., None]
    s = q @ k.transpose(-1, -2)
    arg = s * LOG2E - L
    p = torch.exp2(arg)
    dp = do @ v.transpose(-1, -2)
    D = (do * o).sum(-1, keepdim=True)
    ds = p * (dp - D)
    f_s = 65 * E * (q.abs() @ k.abs().transpose(-1, -2))
    eps_p = math.log(2.0) * (LOG2E * (f_s + E * s.abs()) + E * arg.abs()) + EXP_REL
    del f_s, arg
    f_dp = 65 * E * (do.abs() @ v.abs().transpose(-1, -2)) + 12 * E * (do * o).abs().sum(-1, keepdim=True)
    e_ds = p * (eps_p * (dp - D).abs() + f_dp) * (1 + eps_p) + 2.0 ** -126
    e_ds = e_ds + (U + E) * (ds.abs() + e_ds)
    e_p = p * eps_p + U * p * (1 + eps_p) + 2.0 ** -126
    del dp, f_dp, eps_p
    a_ds, a_p = ds.abs() + e_ds, p + e_p
    ref = torch.stack([ds @ k, ds.transpose(-1, -2) @ q, p.transpose(-1, -2) @ do])                     # [3, 16, 577, 64]
    floor = torch.stack([e_ds @ k.abs() + 641 * E * (a_ds @ k.abs()), e_ds.transpose(-1, -2) @ q.abs() + 641 * E * (a_ds.transpose(-1, -2) @ q.abs()),
                         e_p.transpose(-1, -2) @ do.abs() + 641 * E * (a_p.transpose(-1, -2) @ do.abs())])
    back = lambda t: t.permute(2, 0, 1, 3).reshape(577, 3072)                                          # -> [577, (dq | dk | dv)]
    return back(ref), back(floor)


# ------------------------------------------------------------------------------------------------------------------------------
# the steps
# ------------------------------------------------------------------------------------------------------------------------------
def _check_step(record, c, s, st, prev, run, p, d_x):
    """step s of run ``run`` against fp64 from what the run to s - 1 (``prev``) stored"""
    S, v, pv, g, M, n = c.sets[st], run.v, prev.v, run.g, c.M, c.n
    split = M >= SPLIT_MIN_ROWS
    chain = _colsum_chain(M, COL_CHUNKS)
    rows = _sample(M, 577, 300 + s)
    W = {f: t.to(F64) for f, t in p.items() if t.dim() == 2}
    if s == 1:        # fc2: x_out = h W_fc2^T + b + x'
        c16 = pv["carry16"].to(F64)
        _check_colsum(record, "fc2_b", g["fc2_b"], c16, chain)
        h = S["h"].to(F64)
        _check(record, "fc2_w", g["fc2_w"], c16.t() @ h, _wgrad_floor(c16, h))
        del h
        _check(record, "dh", v["dh"][rows], c16[rows] @ W["fc2_w"], _gemm_floor(c16[rows], W["fc2_w"].t()))
    elif s == 2:      # quick_gelu backward in place (elementwise: every row, a few thousand at a time), fc1's bias from the stored dz
        for r0 in range(0, M, 4096):
            dh = pv["dh"][r0:r0 + 4096].to(F64)
            gp, f_gp = _quick_gelu_grad_ref(S["z"][r0:r0 + 4096])
            ref = dh * gp
            _check(record, "dz", v["dh"][r0:r0 + 4096], ref, dh.abs() * f_gp + E * ref.abs())
            del dh, gp, f_gp, ref
        _check_colsum(record, "fc1_b", g["fc1_b"], v["dh"].to(F64), chain)
    elif s == 3:      # fc1: z = LN2(x') W_fc1^T + b
        dz, y2 = pv["dh"].to(F64), S["y2"].to(F64)
        _check(record, "fc1_w", g["fc1_w"], dz.t() @ y2, _wgrad_floor(dz, y2))
        del y2
        _check(record, "d_ln2", v["g"][rows], dz[rows] @ W["fc1_w"], _gemm_floor(dz[rows], W["fc1_w"].t()))
    elif s == 4:      # layer_norm2 backward into the carry; out_proj's bias from the new carry16
        ref, floor, pr, lchain = _ln_bwd_ref(pv["g"], S["xp"], p["ln2_w"], M)
        c0 = pv["carry32"].to(F64)
        ref = c0 + ref
        _check_f32(record, "carry_ln2", v["carry32"], ref, floor + E * ref.abs())
        del ref, floor, c0
        assert torch.equal(_bits(v["carry16"]), _bits(v["carry32"].to(BF)))
        _check(record, "ln2_w", g["ln2_w"], *pr["dgamma"])
        _check(record, "ln2_b", g["ln2_b"], *pr["dbeta"])
        c16 = v["carry16"].to(F64)
        _check(record, "o_b", g["o_b"], c16.sum(0), lchain * E * c16.abs().sum(0))
    elif s == 5:      # out_proj: x' = ctx W_o^T + b + x
        c16, cx = pv["carry16"].to(F64), S["ctx"].to(F64)
        _check(record, "dctx", v["g"][rows], c16[rows] @ W["o_w"], _gemm_floor(c16[rows], W["o_w"].t()))
        _check(record, "o_w", g["o_w"], c16.t() @ cx, _wgrad_floor(c16, cx))
        if split:     # the fp32 slices over their own rows, and the reduce in its fixed order (q's slices take slot 0 at step 7)
            for i, (r0, r1) in enumerate(_slices(M, SPLITS)):
                _check_f32(record, "o_w_slice", v["splitk"][0, i], c16[r0:r1].t() @ cx[r0:r1],
                           (r1 - r0) * E * (c16[r0:r1].abs().t() @ cx[r0:r1].abs()))
            assert torch.equal(_bits(g["o_w"]), _bits(_reduce_emulated(v["splitk"][0], 1.0)))
    elif s == 6:      # attention: delta, then dq | dk | dv
        dc, cx = pv["g"].to(F64).view(n, 577, 16, 64), S["ctx"].to(F64).view(n, 577, 16, 64)
        _check_f32(record, "delta", v["delta"][:, :, :577], (dc * cx).sum(-1).transpose(1, 2), 12 * E * (dc * cx).abs().sum(-1).transpose(1, 2))
        del dc, cx
        assert bool((_bits(v["delta"][:, :, 577:]) == 0xFF).all())                  # tokens 577 .. 639 are never written
        crops = sorted({0, n // 2, n - 1})
        refs, floors = zip(*[_attn_bwd_ref(S["qkv"], S["lse"], S["ctx"], pv["g"], cr) for cr in crops])
        got = torch.cat([v["dqkv"][cr * 577:(cr + 1) * 577] for cr in crops])
        ref, floor = torch.cat(refs), torch.cat(floors)
        _check(record, "dqkv", got, ref, floor)
        # rel-RMS per (crop, head, dq | dk | dv): P and dS are rounded to bf16 once each and the result once more, three independent
        # roundings of RMS U / sqrt 3 relative; the sums over 577 keys average them rather than add them, so an error of 1 - 2 U is
        # what a right kernel gives, and 4 U leaves room for the near-cancellation in dS = P (dP - D) while any systematic slip in
        # one head (a wrong LSE, D or column mask) is far above it
        eb = (got.to(F64) - ref).view(len(crops), 577, 3, 16, 64).pow(2).mean(dim=(1, 4)).sqrt()
        rb = ref.view(len(crops), 577, 3, 16, 64).pow(2).mean(dim=(1, 4)).sqrt()
        rel = float((eb / rb).max())
        record("dqkv_head_rel_rms_over_U", f"{rel / U:.3g}")
        assert rel <= 4 * U, rel
    elif s == 7:      # q | k | v: bias thirds x 1/8, 1, 1; weight gradients (split-K or direct) with alpha = 1/8 on q; g = dqkv W_qkv
        dqkv, y1 = pv["dqkv"].to(F64), S["y1"].to(F64)
        for t, (name, alpha) in enumerate((("q", 0.125), ("k", 1.0), ("v", 1.0))):
            d = dqkv[:, t * 1024:(t + 1) * 1024]
            _check_colsum(record, f"{name}_b", g[f"{name}_b"], d, chain, alpha)
            _check(record, f"{name}_w", g[f"{name}_w"], alpha * (d.t() @ y1), _wgrad_floor(d, y1, alpha))
            if split:
                for i, (r0, r1) in enumerate(_slices(M, SPLITS)):
                    _check_f32(record, f"{name}_w_slice", v["splitk"][t, i], d[r0:r1].t() @ y1[r0:r1],
                               (r1 - r0) * E * (d[r0:r1].abs().t() @ y1[r0:r1].abs()))
                assert torch.equal(_bits(g[f"{name}_w"]), _bits(_reduce_emulated(v["splitk"][t], alpha))), name
        del y1
        wq = S["w_qkv"].to(F64)                                                      # the forward's pack: q rows scaled by 1/8
        assert torch.equal(wq[:1024], W["q_w"] / 8) and torch.equal(wq[1024:], torch.cat([W["k_w"], W["v_w"]]))
        _check(record, "d_ln1", v["g"][rows], dqkv[rows] @ wq, _gemm_floor(dqkv[rows], wq.t()))
    elif s == 8:      # layer_norm1 backward into the carry, plus the caller's gradient of the layer's input
        ref, floor, pr, _ = _ln_bwd_ref(pv["g"], S["x"], p["ln1_w"], M)
        c0 = pv["carry32"].to(F64)
        if d_x is not None:
            c0 = c0 + d_x.view(M, 1024).to(F64)
            floor = floor + E * c0.abs()
        ref = c0 + ref
        _check_f32(record, "carry_ln1", v["carry32"], ref, floor + E * ref.abs())
        del ref, floor, c0
        assert torch.equal(_bits(v["carry16"]), _bits(v["carry32"].to(BF)))
        _check(record, "ln1_w", g["ln1_w"], *pr["dgamma"])
        _check(record, "ln1_b", g["ln1_b"], *pr["dbeta"])


def _check_confined(c, s, prev, run, split):
    """everything step s does not own keeps the bits the run to s - 1 left: workspace regions, padding and tail; gradients of other
    steps (NaN until written) and the sentinel gaps"""
    owned = [r for r in STEP_REGIONS[s] if r != "splitk" or split]
    mask = torch.ones(prev.ws.numel(), dtype=torch.bool, device=DEV)
    for r in owned:
        mask[c.bo[r]: c.bo[r] + c.sizes[r]] = False
    assert torch.equal(run.ws[mask], prev.ws[mask]), s
    gmask = torch.ones(prev.gbuf.numel(), dtype=torch.bool, device=DEV)
    for f in STEP_GRADS[s]:
        o = run.g[f].data_ptr() - run.gbuf.data_ptr()
        gmask[o // 2: o // 2 + run.g[f].numel()] = False
    assert torch.equal(run.gbuf[gmask], prev.gbuf[gmask]), s
    for f in STEP_GRADS[s]:
        assert bool(torch.isfinite(run.g[f].float()).all()), f


def _check_final(c, run, split):
    """after the whole layer: every gradient and every region the backward keeps finite, the scratch it does not need 0xFF"""
    for f, t in run.g.items():
        assert bool(torch.isfinite(t.float()).all()), f
    for a, b in run.gaps:
        assert bool((run.gbuf[a:b] == SENTINEL).all())
    v = run.v
    for k in ("carry32", "carry16", "dh", "g"):
        assert bool(torch.isfinite(v[k].float()).all()), k
    assert bool(torch.isfinite(v["delta"][:, :, :577]).all())
    if split:
        assert bool(torch.isfinite(v["splitk"]).all())
    else:
        assert bool((run.ws[c.bo["splitk"]: c.bo["splitk"] + c.sizes["splitk"]] == 0xFF).all())       # the direct path only
    assert bool((run.ws[c.bo["unused_grad"]: c.bo["unused_grad"] + c.sizes["unused_grad"]] == 0xFF).all())


def _initial(c, carry32):
    r = Run()
    r.ws = torch.full((c.bo["total"] + TAIL,), 0xFF, dtype=torch.uint8, device=DEV)
    r.v = _ws_views(c, r.ws)
    r.v["carry32"].copy_(carry32)
    r.v["carry16"].copy_(carry32.to(BF))
    r.gbuf, r.g, r.gaps, _ = _grad_buffer()
    return r


def _all_steps(hooks, record, c, layer, st, carry32, d_x):
    """runs to steps 1 .. 8, each checked against the run before; returns the run to step 8"""
    p = _layer_params(c.model, layer)
    split = c.M >= SPLIT_MIN_ROWS
    prev = _initial(c, carry32)
    for s in range(1, 9):
        run = _backward(hooks, c, layer, st, carry32, d_x, s)
        _check_confined(c, s, prev, run, split)
        _check_step(record, c, s, st, prev, run, p, d_x)
        del prev
        prev = run
    _check_final(c, prev, split)
    return prev


def _d_outs(n, seed):
    g = _gen(seed)
    return [(torch.randn(n, 577, 1024, generator=g, device=DEV) * 0.1).to(BF) for _ in range(4)]


@pytest.fixture(scope="module")
def plain_model():
    return _model(31, False)


@pytest.fixture(scope="module")
def outlier_model():
    return _model(37, True)


# ------------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------------
def _stages_case(hooks, record, model, n, seed):
    """forward of the last two layers, then layer 22's backward step by step from the carry of d_out[23] (the path of
    tp_clip_tower_backward with K = 1), its step-8 state against tp_clip_tower_backward(K = 1) bit for bit, saved unchanged, a
    second run bit-identical"""
    images = cto.make_images(n, seed=seed, device=DEV).to(BF)
    c = _forward(hooks, model, images)
    c.model = model
    saved0 = c.saved.clone()
    d_outs = _d_outs(n, seed + 1)
    carry = d_outs[3].view(c.M, 1024).float()
    final = _all_steps(hooks, record, c, 22, 1, carry, None)
    ws, [(gbuf, _)] = _product_backward(c, 1, d_outs, c.sets[1]["ptr"])
    assert torch.equal(final.ws, ws) and torch.equal(final.gbuf, gbuf)
    again = _backward(hooks, c, 22, 1, carry, None, 8)
    assert torch.equal(again.ws, final.ws) and torch.equal(again.gbuf, final.gbuf)
    assert torch.equal(c.saved, saved0)
    return c, images, d_outs, final


@pytest.mark.parametrize("n", [1, 28])
def test_layer_backward_stages(hooks, plain_model, record_property, n):
    """N = 1 (577 rows: bias_grad sums 577 < 592 chunks of one row, most LayerNorm blocks idle) and N = 28 (16156 rows, the last
    batch whose 1024 x 1024 weight gradients are direct TN items): every step against fp64, the splitk slots never touched.
    Measured on an H100: worst error / bound 0.996 (dz), dqkv 0.29, per-head rel-RMS 0.66 U."""
    _stages_case(hooks, record_property, plain_model, n, 400 + n)


@pytest.mark.parametrize("outlier", [False, True], ids=["plain", "outlier"])
def test_layer_backward_stages_split_k(hooks, plain_model, outlier_model, record_property, outlier):
    """N = 29: 16733 rows, the first batch on the split-K path (4 fp32 slices of 66 / 66 / 66 / 64 k-blocks, the last ending in a
    29-row block; the A operands of q / k / v are column thirds of dqkv at ld 3072 read in TN form).  Every step against fp64, each
    slice against fp64 over its own rows and every reduce bit for bit against its fixed-order emulation (o_w at step 5, before q's
    slices take slot 0).  Plain weights, and weights whose residual stream carries four channels at +-50..90.  On the plain
    weights also: the per-row intermediates of crops 0 - 2 (dh, dz, g, both carries, dqkv, delta) bit-identical to a run at N = 3;
    two layers through the hook equal tp_clip_tower_backward(K = 2); q_w, o_w and fc1_w passed as NULL leave every other gradient's
    bits and slot 0 of the split-K partials untouched.
    Measured on an H100: worst error / bound 0.996 (dz); o_w / q_w / k_w / v_w 0.12 / 0.14 / 0.22 / 0.72 and their slices 0.0035 /
    0.0026 / 0.0042 / 0.12; dqkv 0.28, per-head rel-RMS 0.70 U (plain) and 1.6 U (outlier); carry after layer_norm2 0.49 (outlier)."""
    model = outlier_model if outlier else plain_model
    n = 29
    c, images, d_outs, final = _stages_case(hooks, record_property, model, n, 500 + outlier)
    if outlier:
        return
    carry = d_outs[3].view(c.M, 1024).float()
    # batch invariance of every per-row intermediate: crops 0 - 2 at N = 3
    c3 = _forward(hooks, model, images[:3].contiguous())
    c3.model = model
    for name in ("x", "qkv", "xp", "z", "h"):
        assert torch.equal(_bits(c.sets[1][name][:c3.M]), _bits(c3.sets[1][name])), name
    assert torch.equal(_bits(c.sets[1]["lse"][:3, :, :577]), _bits(c3.sets[1]["lse"][:, :, :577]))
    for s in range(1, 9):
        run = _backward(hooks, c, 22, 1, carry, None, s)
        r3 = _backward(hooks, c3, 22, 1, carry[:c3.M], None, s)
        for k in {1: ("dh",), 2: ("dh",), 3: ("g",), 4: ("carry32", "carry16"), 5: ("g",), 6: ("dqkv",), 7: ("g",), 8: ("carry32", "carry16")}[s]:
            assert torch.equal(_bits(run.v[k][:c3.M]), _bits(r3.v[k])), (s, k)
        if s == 6:
            assert torch.equal(_bits(run.v["delta"][:3, :, :577]), _bits(r3.v["delta"][:, :, :577]))
        del run, r3
    del c3
    # NULL gradients: the others keep their bits, out_proj's and q's split-K slot stays poisoned
    skip = ("q_w", "o_w", "fc1_w")
    part = _backward(hooks, c, 22, 1, carry, None, 8, skip=skip)
    for f in GRAD_SHAPES:
        if f in skip:
            assert bool((part.g[f].view(torch.int16) == NAN16).all()), f
        else:
            assert torch.equal(_bits(part.g[f]), _bits(final.g[f])), f
    assert bool((_bits(part.v["splitk"][0]) == 0xFF).all())
    assert torch.equal(_bits(part.v["splitk"][1:]), _bits(final.v["splitk"][1:]))
    for k in ("carry32", "carry16", "g", "dh"):
        assert torch.equal(_bits(part.v[k]), _bits(final.v[k])), k
    del part, final
    # two layers: layer 22 with the caller's gradient of hidden_states[22], then layer 21 from the carry layer 22 left
    r22 = _backward(hooks, c, 22, 1, carry, d_outs[2], 8)
    r21 = _backward(hooks, c, 21, 0, None, None, 8, ws=r22.ws)
    ws, [(g21, _), (g22, _)] = _product_backward(c, 2, d_outs, c.sets[0]["ptr"])
    assert torch.equal(g22, r22.gbuf) and torch.equal(g21, r21.gbuf)
    assert torch.equal(ws, r21.ws)


def test_layer_backward_stages_fp32_carry_and_input_gradient(hooks, plain_model, record_property):
    """N = 3 with an fp32 carry that bf16 cannot represent (d_out[23] plus N(0, 1e-3) noise: every element has bits below bf16's) and
    a caller gradient of the layer's input: steps 1 - 7 read only carry16 = bf16(carry32), layer_norm2 and layer_norm1 add to the fp32
    carry as stored, layer_norm1 adds d_x first.  Every step against fp64.
    Measured on an H100: worst error / bound 0.996 (dz), carry after layer_norm2 0.23 and after layer_norm1 0.91."""
    n = 3
    images = cto.make_images(n, seed=601, device=DEV).to(BF)
    c = _forward(hooks, plain_model, images)
    c.model = plain_model
    d_outs = _d_outs(n, 602)
    carry = d_outs[3].view(c.M, 1024).float() + 1e-3 * torch.randn(c.M, 1024, generator=_gen(603), device=DEV)
    assert not torch.equal(carry.to(BF).float(), carry)
    d_x = d_outs[2]
    _all_steps(hooks, record_property, c, 22, 1, carry, d_x)
