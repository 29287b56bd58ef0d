"""Training straight from the four CLIP hidden states (TokenPackerB200.forward_hidden_states, include/tokenpacker_b200_layers.h) on
the GPU.  The reference arm is today's LLaVA path: x0 = hs[3][:,1:], xm = torch.cat(hs, -1)[:,1:], forward() under autograd.
Every comparison is bit for bit: the layers path reads the same values in the same k-block order as the concatenation.

1. tp_forward_train_layers against tp_forward_train on the concatenation: the output and the whole ``saved`` buffer.
2. Through autograd: the output, all 23 parameter gradients and, with input_grad, each layer's gradient (layer 23's is the sum of its
   feat and feat_multi paths; CLS rows exactly +0.0); subsets of layers, frozen parameters, tower-shaped and [N,576,1024] inputs.
3. tp_backward_layers into sentinel-filled, guard-padded destinations: every token row written, everything else untouched.
4. forward_hidden_states_packed against forward_packed on the concatenation, in inference and in training.
5. An in-place edit of a layer between forward and backward raises; run-to-run identity; no concatenation or copy of the layers.
"""
import ctypes as C

import pytest
import torch

from oracle import hd_oracle as hdo
from oracle import tokenpacker_oracle as tpo

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(torch.int16)


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _module(s, hidden, seed):
    from tokenpacker_b200 import TokenPackerB200
    params = {k: tpo.round_bf16(v) for k, v in tpo.make_params(hidden, seed=seed).items()}
    m = TokenPackerB200(hidden_size=hidden, scale_factor=s)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    return m.to("cuda", BF).train()


def _layers(n, seed, rows=577):
    """four bf16 hidden states [n, rows, 1024] of CLIP-like scale"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(n, rows, 1024, device="cuda", generator=g).to(BF) for _ in range(4)]


def _grad_out(n, s, hidden, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, (24 // s) ** 2, hidden, device="cuda", generator=g).to(BF)


def _tokens(t):
    return t[:, 1:] if t.shape[1] == 577 else t


def _run(m, hs, gout, want, arm):
    """One training step; returns (out, parameter grads, layer grads).  arm 'cat': the concatenation through forward(); 'layers':
    forward_hidden_states."""
    leaves = [t.clone().requires_grad_(w) for t, w in zip(hs, want)]
    for p in m.parameters():
        p.grad = None
    if arm == "cat":
        out = m((_tokens(leaves[3]), torch.cat(leaves, -1)[:, 1:] if leaves[0].shape[1] == 577 else torch.cat(leaves, -1)))
    else:
        out = m.forward_hidden_states(leaves)
    out.backward(gout)
    torch.cuda.synchronize()
    pg = [None if p.grad is None else p.grad.clone() for p in m._raw_params()]
    return out.detach(), pg, [t.grad for t in leaves]


def _assert_same_step(a, b):
    out_a, pg_a, lg_a = a
    out_b, pg_b, lg_b = b
    assert _same(out_a, out_b)
    for i, (x, y) in enumerate(zip(pg_a, pg_b)):
        assert (x is None) == (y is None), i
        assert x is None or _same(x, y), i
    for i, (x, y) in enumerate(zip(lg_a, lg_b)):
        assert (x is None) == (y is None), i
        assert x is None or _same(x, y), i


# ------------------------------------------------------------------------------------------------------------------------------
# 1. the training forward: output and saved activations
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s,n,hidden", [(s, n, 256) for s in (2, 3, 4, 6) for n in (1, 5)] + [(2, 8, 4096)])
@pytest.mark.parametrize("rows", [577, 576])
def test_training_forward_and_saved_match_concatenation(s, n, hidden, rows):
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    m = _module(s, hidden, seed=s + n)
    hs = _layers(n, seed=100 + s * 10 + n, rows=rows)
    bf = [p.detach().contiguous() for p in m._raw_params()]
    w = _lib.TpWeights(*[t.data_ptr() for t in bf])
    pbytes = lib.tp_packed_bytes(hidden)
    packed = torch.empty(pbytes, dtype=torch.uint8, device="cuda")
    _lib.check(lib.tp_pack_weights_train(C.byref(w), hidden, packed.data_ptr(), pbytes, _stream()), "pack")
    sbytes = lib.tp_train_saved_bytes(n, s, hidden)
    x0 = _tokens(hs[3]).contiguous()
    xm = torch.cat([_tokens(t) for t in hs], -1).contiguous()
    res = []
    for arm in ("cat", "layers"):
        out = torch.zeros(n, (24 // s) ** 2, hidden, dtype=BF, device="cuda")
        saved = torch.zeros(sbytes, dtype=torch.uint8, device="cuda")
        if arm == "cat":
            st = lib.tp_forward_train(C.byref(w), packed.data_ptr(), x0.data_ptr(), xm.data_ptr(), n, 576 * 1024, 576 * 4096, s, hidden,
                                      out.data_ptr(), saved.data_ptr(), sbytes, _stream())
        else:
            ptrs = (C.c_void_p * 4)(*[_tokens(t).data_ptr() for t in hs])
            st = lib.tp_forward_train_layers(C.byref(w), packed.data_ptr(), ptrs, n, rows * 1024, s, hidden, out.data_ptr(),
                                             saved.data_ptr(), sbytes, _stream())
        _lib.check(st, arm)
        res.append((out, saved))
    torch.cuda.synchronize()
    assert _same(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])


# ------------------------------------------------------------------------------------------------------------------------------
# 2. through autograd, against the concatenation
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s,n,hidden", [(2, 2, 256), (3, 3, 256), (4, 2, 256), (6, 5, 256), (2, 8, 4096)])
@pytest.mark.parametrize("rows", [577, 576])
def test_gradients_match_concatenation(s, n, hidden, rows):
    m = _module(s, hidden, seed=7 * s + n)
    m.input_grad = True
    hs = _layers(n, seed=200 + s * 10 + n, rows=rows)
    gout = _grad_out(n, s, hidden, seed=300 + s)
    want = (True, True, True, True)
    ref = _run(m, hs, gout, want, "cat")
    got = _run(m, hs, gout, want, "layers")
    _assert_same_step(ref, got)
    assert all(g is not None for g in got[1])                      # all 23 parameter gradients
    for g in got[2]:
        assert g.shape == (n, rows, 1024) and g.dtype == BF
        if rows == 577:
            assert torch.equal(_bits(g[:, 0]), torch.zeros_like(_bits(g[:, 0])))    # +0.0, not -0.0


@pytest.mark.parametrize("want,frozen", [((True, False, False, False), False), ((False, False, False, True), False),
                                         ((False, False, False, True), True), ((False, False, False, False), False)])
def test_subsets_and_frozen_parameters(want, frozen):
    s, n, hidden = 2, 3, 256
    m = _module(s, hidden, seed=31)
    m.input_grad = True
    if frozen:
        for p in m.parameters():
            p.requires_grad_(False)
    hs = _layers(n, seed=32)
    gout = _grad_out(n, s, hidden, seed=33)
    _assert_same_step(_run(m, hs, gout, want, "cat"), _run(m, hs, gout, want, "layers"))


def test_dtype_and_mixed_shapes_fall_back_to_copies():
    """fp16 layers, and a mix of [N,577,1024] and [N,576,1024] layers, go through bf16 [:,1:] copies; gradients come back in each
    layer's shape and dtype.  For fp16 the reference casts the layers to bf16 before the concatenation, so that layer 23's two
    gradient paths are summed in bf16 on both sides."""
    s, n, hidden = 3, 2, 256
    m = _module(s, hidden, seed=41)
    m.input_grad = True
    gout = _grad_out(n, s, hidden, seed=42)
    hs = [t.to(torch.float16) for t in _layers(n, seed=43)]
    got = _run(m, hs, gout, (True,) * 4, "layers")
    leaves = [t.clone().requires_grad_(True) for t in hs]
    for p in m.parameters():
        p.grad = None
    hb = [t.to(BF) for t in leaves]
    ref_out = m((hb[3][:, 1:], torch.cat(hb, -1)[:, 1:]))
    ref_out.backward(gout)
    ref = (ref_out.detach().to(torch.float16), [p.grad.clone() for p in m._raw_params()], [t.grad for t in leaves])
    assert got[0].dtype == torch.float16 and all(g.dtype == torch.float16 and g.shape == (n, 577, 1024) for g in got[2])
    _assert_same_step(ref, got)
    mixed = _layers(n, seed=44)
    mixed[1] = mixed[1][:, 1:].contiguous()
    leaves = [t.clone().requires_grad_(True) for t in mixed]
    out = m.forward_hidden_states(leaves)
    out.backward(gout)
    cat_leaves = [t.clone().requires_grad_(True) for t in mixed]
    ref_out = m((cat_leaves[3][:, 1:], torch.cat([_tokens(t) for t in cat_leaves], -1)))
    ref_out.backward(gout)
    assert _same(out.detach(), ref_out.detach())
    for a, b in zip(leaves, cat_leaves):
        assert _same(a.grad, b.grad)


# ------------------------------------------------------------------------------------------------------------------------------
# 3. the C entry point into guard-padded destinations
# ------------------------------------------------------------------------------------------------------------------------------
def test_backward_layers_writes_exactly_the_token_rows():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    s, n, hidden = 2, 3, 256
    m = _module(s, hidden, seed=51)
    m.input_grad = True
    hs = _layers(n, seed=52)
    gout = _grad_out(n, s, hidden, seed=53)
    _, ref_pg, ref_lg = _run(m, hs, gout, (True,) * 4, "cat")
    bf = [p.detach().contiguous() for p in m._raw_params()]
    w = _lib.TpWeights(*[t.data_ptr() for t in bf])
    pbytes = lib.tp_packed_bytes(hidden)
    packed = torch.empty(pbytes, dtype=torch.uint8, device="cuda")
    _lib.check(lib.tp_pack_weights_train(C.byref(w), hidden, packed.data_ptr(), pbytes, _stream()), "pack")
    sbytes = lib.tp_train_saved_bytes(n, s, hidden)
    saved = torch.empty(sbytes, dtype=torch.uint8, device="cuda")
    out = torch.empty(n, 144, hidden, dtype=BF, device="cuda")
    ptrs = (C.c_void_p * 4)(*[t[:, 1:].data_ptr() for t in hs])
    _lib.check(lib.tp_forward_train_layers(C.byref(w), packed.data_ptr(), ptrs, n, 577 * 1024, s, hidden, out.data_ptr(), saved.data_ptr(),
                                           sbytes, _stream()), "forward")
    # destinations: 8 guard rows, then crops of 579 rows (2 leading rows, 576 token rows, 1 trailing row), then 8 guard rows
    guard, crop_rows, lead = 8, 579, 2
    dest = [torch.full((2 * guard + n * crop_rows, 1024), 0x7FC5, dtype=torch.int16, device="cuda") for _ in range(4)]   # a NaN
    grads = [torch.full_like(t, float("nan")) for t in bf]
    gs = _lib.TpWeights(*[t.data_ptr() for t in grads])
    dptr = (C.c_void_p * 4)(*[d[guard + lead:].data_ptr() for d in dest])
    wbytes = lib.tp_backward_workspace_bytes(n, s, hidden)
    ws = torch.full((wbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    _lib.check(lib.tp_backward_layers(C.byref(w), packed.data_ptr(), ptrs, 577 * 1024, n, s, hidden, gout.data_ptr(), saved.data_ptr(),
                                      C.byref(gs), dptr, crop_rows * 1024, ws.data_ptr(), wbytes, _stream()), "backward")
    torch.cuda.synchronize()
    for a, b in zip(grads, ref_pg):
        assert _same(a, b)
    for d, ref in zip(dest, ref_lg):
        bits = d
        body = bits[guard:guard + n * crop_rows].view(n, crop_rows, 1024)
        assert torch.equal(body[:, lead:lead + 576], _bits(ref[:, 1:]))
        untouched = torch.cat([bits[:guard], bits[guard + n * crop_rows:], body[:, :lead].reshape(-1, 1024),
                               body[:, lead + 576:].reshape(-1, 1024)])
        assert bool((untouched == 0x7FC5).all())


# ------------------------------------------------------------------------------------------------------------------------------
# 4. packed HD rows
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [2, 4])
def test_packed_matches_forward_packed(s):
    hidden = 256
    grids = [(1, 1), (2, 3)]
    n = sum(hdo.n_crops(a, b) for a, b in grids)
    hb, wb = [a for a, _ in grids], [b for _, b in grids]
    m = _module(s, hidden, seed=61)
    hs = _layers(n, seed=62)
    g = torch.Generator(device="cuda").manual_seed(63)
    sep = torch.randn(hidden, device="cuda", generator=g).to(BF)
    ret = torch.randn(hidden, device="cuda", generator=g).to(BF)
    with torch.no_grad():
        ref, cu_ref = m.forward_packed((hs[3][:, 1:], torch.cat(hs, -1)[:, 1:]), hb, wb, sep, ret)
        got, cu = m.forward_hidden_states_packed(hs, hb, wb, sep, ret)
    assert _same(ref, got) and list(cu) == list(cu_ref)
    # training: parameter, layer and separator-row gradients
    m.input_grad = True
    gp = torch.randn(ref.shape, device="cuda", generator=g).to(BF)
    results = []
    for arm in ("cat", "layers"):
        leaves = [t.clone().requires_grad_(True) for t in hs]
        sp, rt = sep.clone().requires_grad_(True), ret.clone().requires_grad_(True)
        for p in m.parameters():
            p.grad = None
        if arm == "cat":
            out, _ = m.forward_packed((leaves[3][:, 1:], torch.cat(leaves, -1)[:, 1:]), hb, wb, sp, rt)
        else:
            out, _ = m.forward_hidden_states_packed(leaves, hb, wb, sp, rt)
        out.backward(gp)
        results.append((out.detach(), [p.grad.clone() for p in m._raw_params()], [t.grad for t in leaves] + [sp.grad, rt.grad]))
    _assert_same_step(*results)


# ------------------------------------------------------------------------------------------------------------------------------
# 5. autograd plumbing, determinism, no copies
# ------------------------------------------------------------------------------------------------------------------------------
def test_in_place_edit_before_backward_raises():
    m = _module(2, 256, seed=71)
    hs = _layers(2, seed=72)
    out = m.forward_hidden_states(hs)
    hs[1].add_(1)
    with pytest.raises(RuntimeError, match="inplace"):
        out.backward(_grad_out(2, 2, 256, seed=73))


def test_run_to_run_identity():
    s, n, hidden = 2, 4, 4096
    m = _module(s, hidden, seed=81)
    m.input_grad = True
    hs = _layers(n, seed=82)
    gout = _grad_out(n, s, hidden, seed=83)
    a = _run(m, hs, gout, (True,) * 4, "layers")
    b = _run(m, hs, gout, (True,) * 4, "layers")
    _assert_same_step(a, b)


def test_no_concatenation_or_copy_of_the_layers():
    """forward + backward from bf16 tower-shaped layers: no aten::cat anywhere, and no copy of a layer-sized ([., 576 | 577, 1024 |
    4096]) tensor."""
    from torch.profiler import ProfilerActivity, profile
    s, n, hidden = 2, 2, 256
    m = _module(s, hidden, seed=91)
    hs = _layers(n, seed=92)
    gout = _grad_out(n, s, hidden, seed=93)
    out = m.forward_hidden_states(hs)           # warm-up (plan caches, module loads)
    out.backward(gout)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        out = m.forward_hidden_states(hs)
        out.backward(gout)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert not any(nm == "aten::cat" for nm in names)
    for e in prof.events():
        if e.name in ("aten::copy_", "aten::clone", "aten::contiguous", "aten::_to_copy"):
            for shp in e.input_shapes:
                assert not (len(shp) >= 2 and shp[-1] in (1024, 4096) and shp[-2] in (576, 577)), (e.name, e.input_shapes)
    assert not any("CatArrayBatchedCopy" in nm for nm in names)
