"""Argument validation of every projector entry point, host side (no CUDA): the status each returns for a table of bad arguments,
including which of two bad arguments is reported first.  Every case is refused before any CUDA call, so the pointers are fakes that
are never dereferenced, and every expected status is INVALID_ARGUMENT or BAD_SCALE_FACTOR: no case can reach a launch."""
import ctypes as C

import pytest

P = 4096                                   # a fake, 16-byte aligned device pointer
X0S, XMS, LAYS = 576 * 1024, 576 * 4096, 577 * 1024   # crop strides: feat, the concatenated stack, one hidden state ([:, 1:] view)
MAX_ROWS = 0x7FFF0000 // 576 + 1           # crops whose 576 N rows overflow the GEMMs' row count


def _lib():
    from tokenpacker_b200 import _lib
    return _lib


def _weights(null_last=False):
    n = len(_lib().WEIGHT_FIELDS)
    return _lib().TpWeights(*([P] * (n - 1) + [None if null_last else P]))


def _ptrs(*vals):
    return (C.c_void_p * len(vals))(*vals)


LAYERS = (P, P + 4096, P + 8192, P + 12288)


def _layers(v):
    return None if v is None else _ptrs(*v)


def _call(name, a):
    lib = _lib().lib
    if name in ("tp_forward", "tp_forward_packed"):
        last = a["seg"] if name == "tp_forward" else a["rows"]
        return getattr(lib, name)(a["packed"], a["x0"], a["xm"], a["n"], a["x0s"], a["xms"], a["s"], a["h"], a["out"], last, a["ws"], 1, None)
    if name in ("tp_forward_layers", "tp_forward_layers_packed"):
        last = a["seg"] if name == "tp_forward_layers" else a["rows"]
        return getattr(lib, name)(a["packed"], _layers(a["layers"]), a["n"], a["cs"], a["s"], a["h"], a["out"], last, a["ws"], 1, None)
    if name == "tp_forward_allgather":
        return lib.tp_forward_allgather(a["packed"], a["x0"], a["xm"], a["n"], a["x0s"], a["xms"], a["s"], a["h"], _layers(a["peers"]),
                                        a["n_peers"], a["offset"], a["rows"], a["ws"], 1, None)
    if name == "tp_forward_train":
        return lib.tp_forward_train(a["w"], a["packed"], a["x0"], a["xm"], a["n"], a["x0s"], a["xms"], a["s"], a["h"], a["out"], a["saved"], 1,
                                    None)
    if name == "tp_forward_train_layers":
        return lib.tp_forward_train_layers(a["w"], a["packed"], _layers(a["layers"]), a["n"], a["cs"], a["s"], a["h"], a["out"], a["saved"], 1,
                                           None)
    if name == "tp_backward":
        return lib.tp_backward(a["w"], a["xm"], a["xms"], a["n"], a["s"], a["h"], a["go"], a["saved"], a["g"], a["ws"], 1, None)
    if name == "tp_backward_inputs":
        return lib.tp_backward_inputs(a["w"], a["packed"], a["xm"], a["xms"], a["n"], a["s"], a["h"], a["go"], a["saved"], a["g"], a["dx0"],
                                      a["dxm"], a["ws"], 1, None)
    if name == "tp_backward_layers":
        return lib.tp_backward_layers(a["w"], a["packed"], _layers(a["layers"]), a["cs"], a["n"], a["s"], a["h"], a["go"], a["saved"], a["g"],
                                      _layers(a["d"]), a["dcs"], a["ws"], 1, None)
    if name in ("tp_pack_weights", "tp_pack_weights_train"):
        return getattr(lib, name)(a["w"], a["h"], a["packed"], 1 << 40, None)
    raise KeyError(name)


def _base():
    return dict(packed=P, x0=P, xm=P, n=1, x0s=X0S, xms=XMS, s=2, h=4096, out=P, seg=None, rows=0, ws=P, layers=LAYERS, cs=LAYS,
                peers=(P,) * 8, n_peers=2, offset=0, w=C.byref(_weights()), saved=P, go=P, g=C.byref(_weights()), dx0=P, dxm=P,
                d=(None, None, None, P), dcs=LAYS)


NULL_W = "null weight field"
NULL_G = "null gradient field"

# (entry point, overrides, expected); an override value NULL_W / NULL_G stands for a tp_weights with its last field NULL
FORWARD_CAT = ("tp_forward", "tp_forward_packed", "tp_forward_allgather", "tp_forward_train")
LAYERED = ("tp_forward_layers", "tp_forward_layers_packed", "tp_forward_train_layers", "tp_backward_layers")
BAD, BAD_S = "INVALID_ARGUMENT", "BAD_SCALE_FACTOR"

CASES = []
for fn in FORWARD_CAT:
    CASES += [
        (fn, dict(s=0), BAD_S), (fn, dict(s=5), BAD_S), (fn, dict(s=48), BAD_S), (fn, dict(s=-2), BAD_S),
        (fn, dict(s=5, packed=None), BAD_S), (fn, dict(s=5, x0=None), BAD_S), (fn, dict(s=5, xms=XMS - 8), BAD_S),
        (fn, dict(s=5, n=0), BAD_S),
        (fn, dict(packed=None), BAD), (fn, dict(x0=None), BAD), (fn, dict(xm=None), BAD),
        (fn, dict(n=0), BAD), (fn, dict(n=-1), BAD), (fn, dict(n=MAX_ROWS), BAD),
        (fn, dict(x0s=X0S - 1024), BAD), (fn, dict(x0s=X0S + 4), BAD),
        (fn, dict(xms=XMS - 4096), BAD), (fn, dict(xms=XMS + 4), BAD), (fn, dict(xms=576 * 1024), BAD),
        (fn, dict(h=100), BAD), (fn, dict(h=16), BAD), (fn, dict(h=65536 + 256), BAD),
    ]
    if fn != "tp_forward_allgather":
        CASES += [(fn, dict(out=None), BAD)]
    if fn != "tp_forward_train":
        CASES += [(fn, dict(ws=None), BAD)]
CASES += [("tp_forward_train", dict(saved=None), BAD), ("tp_forward_train", dict(s=5, saved=None), BAD_S)]
CASES += [
    # the all-gather's own arguments come before the scale factor
    ("tp_forward_allgather", dict(peers=None), BAD), ("tp_forward_allgather", dict(peers=None, s=5), BAD),
    ("tp_forward_allgather", dict(n_peers=0), BAD), ("tp_forward_allgather", dict(n_peers=9), BAD),
    ("tp_forward_allgather", dict(offset=-1), BAD), ("tp_forward_allgather", dict(offset=-1, s=5), BAD),
    ("tp_forward_allgather", dict(h=4096 + 32), BAD), ("tp_forward_allgather", dict(h=4096 + 32, s=5), BAD),
    ("tp_forward_allgather", dict(rows=100), BAD),                          # fewer rows per crop than queries (144 at s = 2)
    ("tp_forward_allgather", dict(s=8, rows=10), BAD),                      # packed rows the pair kernel's stores cannot serve
    ("tp_forward_allgather", dict(s=5, rows=100), BAD_S),
    ("tp_forward_allgather", dict(peers=(P, None) + (P,) * 6), BAD),
]
for fn in LAYERED:
    CASES += [
        (fn, dict(s=0), BAD_S), (fn, dict(s=5), BAD_S), (fn, dict(s=48), BAD_S),
        (fn, dict(s=5, cs=LAYS - 2048), BAD_S), (fn, dict(s=5, layers=(P, P, P + 2, P)), BAD_S),
        (fn, dict(layers=None), BAD), (fn, dict(layers=(P, None, P, P)), BAD), (fn, dict(layers=(P, P, P, None)), BAD),
        (fn, dict(cs=576 * 1024 - 1024), BAD), (fn, dict(cs=LAYS + 4), BAD),
        (fn, dict(packed=None), BAD),
        (fn, dict(n=0), BAD), (fn, dict(h=100), BAD), (fn, dict(layers=(P, P, P + 2, P)), BAD),
    ]
    if fn == "tp_forward_layers":           # a missing layer is reported before a bad scale factor
        CASES += [(fn, dict(layers=None, s=5), BAD), (fn, dict(layers=(P, None, P, P), s=5), BAD)]
    else:                                   # the scale factor is checked first
        CASES += [(fn, dict(layers=None, s=5), BAD_S), (fn, dict(layers=(P, None, P, P), s=5), BAD_S)]
    if fn in ("tp_forward_layers", "tp_forward_layers_packed"):
        CASES += [(fn, dict(out=None), BAD), (fn, dict(ws=None), BAD), (fn, dict(n=MAX_ROWS), BAD)]
CASES += [
    ("tp_forward_layers_packed", dict(out=P + 2), BAD), ("tp_forward_layers_packed", dict(rows=100), BAD),
    ("tp_forward_layers_packed", dict(rows=0x7FFFFFFF // 4096 + 1), BAD), ("tp_forward_layers_packed", dict(rows=100, s=5), BAD_S),
    ("tp_forward_train_layers", dict(out=None), BAD), ("tp_forward_train_layers", dict(saved=None), BAD),
    ("tp_forward_train_layers", dict(n=MAX_ROWS), BAD),
    ("tp_backward_layers", dict(w=None), BAD), ("tp_backward_layers", dict(g=None), BAD), ("tp_backward_layers", dict(go=None), BAD),
    ("tp_backward_layers", dict(saved=None), BAD), ("tp_backward_layers", dict(ws=None), BAD),
    ("tp_backward_layers", dict(w=NULL_W), BAD), ("tp_backward_layers", dict(g=NULL_G), BAD),
    ("tp_backward_layers", dict(w=None, s=5), BAD_S),
    ("tp_backward_layers", dict(d=(None, P + 8, None, None)), BAD),         # a misaligned gradient destination
    ("tp_backward_layers", dict(dcs=LAYS + 8), BAD),                        # not a whole number of 1024-channel rows
    ("tp_backward_layers", dict(dcs=575 * 1024), BAD),
    ("tp_backward_layers", dict(dcs=LAYS + 8, s=5), BAD_S),
]
for fn in ("tp_backward", "tp_backward_inputs"):
    CASES += [
        (fn, dict(s=0), BAD_S), (fn, dict(s=5), BAD_S), (fn, dict(s=48), BAD_S), (fn, dict(s=5, xms=XMS + 8), BAD_S),
        # missing operands and bad sizes are reported before a bad scale factor
        (fn, dict(w=None), BAD), (fn, dict(w=None, s=5), BAD), (fn, dict(g=None), BAD), (fn, dict(g=None, s=5), BAD),
        (fn, dict(xm=None), BAD), (fn, dict(xm=None, s=5), BAD), (fn, dict(go=None), BAD), (fn, dict(saved=None), BAD),
        (fn, dict(ws=None), BAD), (fn, dict(n=0), BAD), (fn, dict(n=0, s=5), BAD), (fn, dict(h=100), BAD), (fn, dict(h=100, s=5), BAD),
        (fn, dict(xms=XMS + 8), BAD), (fn, dict(xms=XMS - 4096), BAD),      # the backward takes a contiguous stack
        (fn, dict(w=NULL_W), BAD), (fn, dict(g=NULL_G), BAD),
        (fn, dict(n=MAX_ROWS), BAD), (fn, dict(n=MAX_ROWS, s=5), BAD),      # the forwards' row limit holds for the backward too
    ]
CASES += [("tp_backward_layers", dict(n=MAX_ROWS), BAD)]
CASES += [
    ("tp_backward_inputs", dict(packed=None), BAD),                          # d_xm reads [W_k0; W_v0] from the packed weights
    ("tp_backward_inputs", dict(dx0=P + 2), BAD), ("tp_backward_inputs", dict(dxm=P + 8), BAD),
    ("tp_backward_inputs", dict(dx0=P + 2, s=5), BAD_S),
]
for fn in ("tp_pack_weights", "tp_pack_weights_train"):
    CASES += [(fn, dict(w=None), BAD), (fn, dict(packed=None), BAD), (fn, dict(h=100), BAD), (fn, dict(h=0), BAD),
              (fn, dict(h=65536 + 32), BAD), (fn, dict(w=NULL_W), BAD)]


def _id(case):
    fn, over, want = case
    return f"{fn}-" + ",".join(f"{k}={v}" for k, v in over.items()) + f"-{want}"


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_entry_point_status(case):
    fn, over, want = case
    assert want in ("INVALID_ARGUMENT", "BAD_SCALE_FACTOR")       # nothing that a status check lets through to the GPU
    a = _base()
    for k, v in over.items():
        a[k] = C.byref(_weights(null_last=True)) if v in (NULL_W, NULL_G) else v
    assert _call(fn, a) == getattr(_lib(), "TP_ERR_" + want)


@pytest.mark.parametrize("query", ["tp_workspace_bytes", "tp_train_saved_bytes", "tp_backward_workspace_bytes"])
def test_size_queries_stop_at_the_row_limit(query):
    """Every size query gives a size up to the largest batch the entry points take (MAX_ROWS - 1 crops) and 0 past it, like the
    entry points' own refusal: no caller allocates a workspace for a batch nothing will run."""
    fn = getattr(_lib().lib, query)
    for s, h in ((1, 4096), (2, 4096), (3, 896), (24, 160)):
        assert fn(MAX_ROWS - 1, s, h) > 0, (s, h)
        assert fn(MAX_ROWS, s, h) == 0 and fn(1 << 40, s, h) == 0, (s, h)
