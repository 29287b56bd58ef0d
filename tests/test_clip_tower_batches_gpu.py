"""The CLIP tower at every kernel plan its batch size selects, at the benchmarked batches and at batches past 32-bit offsets.

The tile engine picks each of the tower's GEMMs a kernel (CTA-pair 256 x 256 tiles, or one-CTA 128 x 256 / 128 x 128 tiles) by an
estimated cost that depends on M = 577 N, so the batch size changes what runs.  Every kernel must give the same bits:
- every crop of a batch of N in NS (the small batches where the choices change, 64 crops as benchmarked, 231 for an HD batch) has the
  bits of that crop run alone, in the bf16 and the fp16 tower; each such N runs on a plan whose layer is checked stage by stage against
  fp64 here (N = 1, 3) or in test_clip_tower_gpu.py / test_clip_tower_f16_gpu.py (N = 2), or on the kernels those plans use;
- the forced plans (TP_GEMM_MODE = 1 / 2, TP_CHAIN = 0) give the default plan's bits, and under mode 2 fc1 -> fc2 runs as one launch;
- batches of 930 and 1818 crops, whose fc1 output holds more than 2^31 and 2^32 elements, and the refusal of a batch past the tower's
  row limit (930452 crops) before anything launches;
- the training step at the benchmarked shapes: 64 crops with the last 12 layers trainable, and 231 crops training the whole tower with
  gradient checkpointing, against the fp64 autograd oracles.
The launch count of each default forward is recorded as the test property ``launches``."""
import ctypes as C
import os
import time

import pytest
import torch

from oracle import clip_tower_embed_oracle as cte
from oracle import clip_tower_oracle as cto
from oracle import clip_tower_train_oracle as ctt
from test_clip_tower_embed_gpu import EMBED_NAMES, _backward, _clear, _d_outs, _grads, _rel
from test_clip_tower_f16_gpu import _one_layer_stages as _one_layer_stages_f16
from test_clip_tower_gpu import _one_layer_stages
from test_clip_tower_train_gpu import _gate, _grad_error

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16 = torch.float16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GiB = 1 << 30
LAYERS = 23
CROP = 3 * 336 * 336
NS = (1, 2, 3, 4, 5, 8, 11, 29, 64, 231)
POOL = max(NS)                                    # distinct seeded crops; the batch of N takes N consecutive ones
STRIDED = (5, 64)                                 # batches passed as views with a crop stride past 3 x 336 x 336


def _hooks(name, suffix):
    lib = C.CDLL(os.path.join(ROOT, "tokenpacker_b200", name))
    offsets, layer = getattr(lib, "tpc_workspace_offsets" + suffix), getattr(lib, "tpc_layer" + suffix)
    offsets.restype, offsets.argtypes = C.c_int, [C.c_int64, C.POINTER(C.c_int64)]
    layer.restype = C.c_int
    layer.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]
    return lib


def _tower(f16, outlier=False):
    """(weights, model, tower) over the seeded weights the tower tests use: rounded to the tower's storage type"""
    from tokenpacker_b200 import CLIPVisionTowerB200
    w = cto.make_weights(LAYERS, seed=11, outlier=outlier, device=DEV)
    if f16:
        w = {k: v.half().float() for k, v in w.items()}
        model = cto.FakeCLIPVisionModel({k: v.half() for k, v in w.items()}).to(DEV)
        return w, model, CLIPVisionTowerB200(model, dtype=F16)
    w = cto.round_bf16(w)
    model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    return w, model, CLIPVisionTowerB200(model)


def _counted(t, x):
    """t.hidden_states(x) and the number of kernels it launched"""
    from tokenpacker_b200 import _lib
    torch.cuda.synchronize()
    c0 = _lib.lib.tp_launch_count()
    with torch.no_grad():
        outs = t.hidden_states(x)
    torch.cuda.synchronize()
    return outs, _lib.lib.tp_launch_count() - c0


def _assert_crops_equal(got, want, what, crops=None):
    """got, want: the four hidden states of the same crops (crops: their numbers in the batch, when not 0, 1, ..); names the crops
    whose bits differ"""
    for g, r, j in zip(got, want, cto.OUT_LAYERS):
        assert g.shape == r.shape and g.dtype == r.dtype, (what, j)
        assert torch.isfinite(g).all(), (what, j)
        differ = (g != r).flatten(1).any(1).nonzero().flatten().tolist()
        assert not differ, (what, f"hidden_states[{j}]", "crops", [i if crops is None else crops[i] for i in differ][:16])


# ------------------------------------------------------------------------------------------------------------------------------
# batch invariance at every plan
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pool():
    return cto.make_images(POOL, seed=101, device=DEV).bfloat16()


@pytest.fixture(scope="module", params=["bf16", "f16"])
def plan_tower(request):
    return _tower(request.param == "f16")[2]


@pytest.fixture(scope="module")
def singles(plan_tower, pool):
    """the four hidden states of every crop of the pool, each run alone"""
    outs = [torch.empty((POOL, 577, 1024), dtype=plan_tower.dtype, device=DEV) for _ in cto.OUT_LAYERS]
    with torch.no_grad():
        for i in range(POOL):
            for o, h in zip(outs, plan_tower.hidden_states(pool[i:i + 1])):
                o[i] = h[0]
    torch.cuda.synchronize()
    return outs


def _offset(n):
    return (37 * n) % (POOL - n + 1)


def _batch(pool, n):
    off = _offset(n)
    if n not in STRIDED:
        return pool[off:off + n]
    big = torch.full((n, CROP + 4096), float("nan"), device=DEV, dtype=pool.dtype)
    view = big[:, :CROP].view(n, 3, 336, 336)
    view.copy_(pool[off:off + n])
    return view


@pytest.mark.parametrize("n", NS)
def test_every_crop_has_the_bits_of_that_crop_alone(plan_tower, pool, singles, n, record_property):
    x = _batch(pool, n)
    outs, launches = _counted(plan_tower, x)
    record_property("launches", launches)
    print(f"\nN={n} {plan_tower.dtype}: {launches} launches")
    off = _offset(n)
    _assert_crops_equal(outs, [s[off:off + n] for s in singles], f"N={n}")


# ------------------------------------------------------------------------------------------------------------------------------
# one layer, stage by stage, at the plans N = 2 does not cover
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("outlier", [False, True], ids=["standard", "outlier"])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("precision", ["bf16", "f16"])
def test_one_layer_stage_by_stage(precision, n, outlier):
    w, model, t = _tower(precision == "f16", outlier)
    if precision == "f16":
        _one_layer_stages_f16(_hooks("libtokenpacker_b200_clip_tower_f16_hooks.so", "_f16"), (w, model, t), n)
    else:
        _one_layer_stages(_hooks("libtokenpacker_b200_clip_tower_hooks.so", ""), (w, t), n)


# ------------------------------------------------------------------------------------------------------------------------------
# forced plans
# ------------------------------------------------------------------------------------------------------------------------------
FORCED = {"one-CTA": {"TP_GEMM_MODE": "1"}, "pair-chained": {"TP_GEMM_MODE": "2"}, "pair-unchained": {"TP_GEMM_MODE": "2", "TP_CHAIN": "0"}}


@pytest.mark.parametrize("n", [5, 64])
def test_forced_plans_give_the_default_bits(plan_tower, pool, n, monkeypatch, record_property):
    """Every GEMM on the one-CTA kernels, every GEMM on the pair kernel with fc1 -> fc2 chained, and unchained: the default plan's
    bits.  The chain is one launch per layer where the unchained plan makes two."""
    x = pool[POOL - n:]
    for var in ("TP_GEMM_MODE", "TP_CHAIN"):
        monkeypatch.delenv(var, raising=False)
    default, launches = _counted(plan_tower, x)
    counts = {"default": launches}
    for name, env in FORCED.items():
        for var in ("TP_GEMM_MODE", "TP_CHAIN"):
            monkeypatch.delenv(var, raising=False)
        for var, value in env.items():
            monkeypatch.setenv(var, value)
        outs, counts[name] = _counted(plan_tower, x)
        _assert_crops_equal(outs, default, f"N={n} {name}")
    record_property("launches", counts)
    print(f"\nN={n} {plan_tower.dtype}: launches {counts}")
    assert counts["pair-unchained"] - counts["pair-chained"] == LAYERS, counts


# ------------------------------------------------------------------------------------------------------------------------------
# batches past the 32-bit offsets, and the largest batch the tower accepts
# ------------------------------------------------------------------------------------------------------------------------------
# crops whose rows straddle or follow a 32-bit boundary (M = 577 N token rows): h [M, 4096] passes element 2^31 inside crop 908 and
# element 2^32 inside crop 1817, qkv [M, 3072] passes element 2^31 inside crop 1211, the fp32 x' [M, 1024] passes byte 2^31 inside crop
# 908 and byte 2^32 inside crop 1817
BIG = {930: [0, 465, 907] + list(range(908, 930)),
       1818: [0, 907, 908, 909, 1210, 1211, 1212, 1816, 1817]}


@pytest.mark.parametrize("n", sorted(BIG))
def test_batches_past_32_bit_offsets(n, record_property):
    """Picked crops of a batch of n have the bits of the crop run alone, and every output is finite."""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    assert 908 * 577 * 4096 < 2 ** 31 <= 909 * 577 * 4096 and 1817 * 577 * 4096 < 2 ** 32 <= 1818 * 577 * 4096
    assert 1211 * 577 * 3072 < 2 ** 31 <= 1212 * 577 * 3072
    need = lib.tp_clip_tower_workspace_bytes(n) + 4 * n * 577 * 1024 * 2 + n * CROP * 2 + 2 * GiB     # + weights, cache, singles
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need + 2 * GiB:
        pytest.skip(f"N={n} needs {need / GiB:.1f} GiB + a 2 GiB margin of device memory, {free / GiB:.1f} GiB free")
    _, _, t = _tower(False)
    x = torch.empty((n, 3, 336, 336), dtype=torch.bfloat16, device=DEV)
    for c0 in range(0, n, 100):
        x[c0:c0 + 100] = cto.make_images(len(x[c0:c0 + 100]), seed=1000 + c0, device=DEV).bfloat16()
    picks = BIG[n]
    with torch.no_grad():
        alone = [t.hidden_states(x[i:i + 1]) for i in picks]                  # (builds the derived weight cache too)
    alone = [torch.cat([a[k] for a in alone]) for k in range(4)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    outs, launches = _counted(t, x)
    peak = torch.cuda.max_memory_allocated() - base
    record_property("launches", launches)
    record_property("peak_bytes_above_inputs", peak)
    print(f"\nN={n}: {launches} launches, peak {peak / GiB:.2f} GiB above the inputs")
    _assert_crops_equal([o[picks] for o in outs], alone, f"N={n}", picks)
    for o, j in zip(outs, cto.OUT_LAYERS):
        assert torch.isfinite(o).all(), j


def test_refuses_a_batch_past_its_row_limit():
    """tp_clip_tower_workspace_bytes accepts n_crops up to 2^31 / (4 x 577) = 930452 (M = 577 N <= 2^29 token rows).  One crop more is
    refused with TP_ERR_INVALID_ARGUMENT before anything launches, by both forwards; at the limit the next check, the workspace size,
    refuses a small workspace, still before anything launches."""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    limit = (1 << 31) // (4 * 577)
    assert lib.tp_clip_tower_workspace_bytes(limit) > 0 and lib.tp_clip_tower_workspace_bytes(limit + 1) == 0
    for f16 in (False, True):
        _, _, t = _tower(f16)
        x = cto.make_images(1, seed=5, device=DEV).bfloat16()
        with torch.no_grad():
            ref = t.hidden_states(x)                                            # builds the derived weight cache
        packed, (w, _) = t._packed_weights(torch.device(DEV))
        outs = [torch.empty_like(r) for r in ref]
        ptrs = (C.c_void_p * 4)(*[o.data_ptr() for o in outs])
        ws = torch.empty(lib.tp_clip_tower_workspace_bytes(1), dtype=torch.uint8, device=DEV)

        def forward(n):
            if f16:
                return lib.tp_clip_tower_forward_f16(packed.data_ptr(), C.byref(w), x.data_ptr(), _lib.TP_CLIP_CROPS_BF16, n, x.stride(0), ptrs,
                                                     ws.data_ptr(), ws.numel(), None)
            return lib.tp_clip_tower_forward(packed.data_ptr(), C.byref(w), x.data_ptr(), n, x.stride(0), ptrs, ws.data_ptr(), ws.numel(), None)

        torch.cuda.synchronize()
        c0 = lib.tp_launch_count()
        assert forward(limit + 1) == _lib.TP_ERR_INVALID_ARGUMENT
        assert forward(limit) == _lib.TP_ERR_WORKSPACE_TOO_SMALL
        assert lib.tp_launch_count() == c0
        assert forward(1) == _lib.TP_OK                                         # the same arguments at one crop run
        torch.cuda.synchronize()
        _assert_crops_equal(outs, ref, f"f16={f16}")

# ------------------------------------------------------------------------------------------------------------------------------
# training at the benchmarked shapes
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def weights():
    return cto.round_bf16(cto.make_weights(LAYERS, seed=11, device=DEV))


def _train_model(w, first, embed=False):
    """the layers from ``first`` up (and with embed, the embedding stage) require grad"""
    model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    for name, p in model.named_parameters():
        layer = int(name.split("encoder.layers.")[1].split(".")[0]) if "encoder.layers." in name else None
        p.requires_grad_(embed if layer is None else layer >= first)
    return model


def _layer_errors(got, ref, first):
    """worst rel-RMS per parameter kind over layers first .. 22 (got: parameter name -> gradient; ref: the oracle's list)"""
    worst = {}
    for i in range(first, LAYERS):
        g = {key: got["vision_model." + cto.layer_keys(i)[key]] for key in ctt.PARAM_KEYS}
        for key in ctt.PARAM_KEYS:
            assert g[key] is not None and torch.isfinite(g[key]).all(), (i, key)
            worst[key] = max(worst.get(key, 0.0), _grad_error(g, ref[i - first], key))
    return worst


def test_training_64_crops_last_12_layers(weights, record_property):
    """The benchmark's largest K at its 64 crops: the outputs have the inference bits, the checkpointed step gives every gradient the
    plain step's bits, and every gradient holds the gates of test_clip_tower_train_gpu.py against the fp64 oracle (4 crops at a time)."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    n, k = 64, 12
    first = LAYERS - k
    model = _train_model(weights, first)
    t = CLIPVisionTowerB200(model, trainable_layers=k)
    images = cto.make_images(n, seed=111, device=DEV).bfloat16()
    with torch.no_grad():
        ref_outs = CLIPVisionTowerB200(model).hidden_states(images)
    d_outs = _d_outs(n, 112)
    steps = {}
    for checkpointing in (False, True):
        _clear(model)
        model.gradient_checkpointing = checkpointing
        outs = t.hidden_states(images)
        for a, b, j in zip(outs, ref_outs, cto.OUT_LAYERS):
            assert torch.equal(a, b), (checkpointing, j)
        assert outs[3].grad_fn.checkpoint == checkpointing
        _backward(outs, d_outs)
        del outs
        steps[checkpointing] = _grads(model)
    plain, ckpt = steps[False], steps[True]
    assert len(plain) == 16 * k and all(g is not None for g in plain.values())
    for name in plain:
        assert torch.equal(ckpt[name], plain[name]), name
    del ref_outs, ckpt
    t0 = time.perf_counter()
    ref = ctt.parameter_gradients_chunked(weights, images.float(), k, d_outs, 4, LAYERS, torch.float64, DEV)
    torch.cuda.synchronize()
    record_property("oracle_seconds", round(time.perf_counter() - t0, 1))
    worst = _layer_errors(plain, ref, first)
    print(f"\nN={n} K={k}: worst rel-RMS per parameter kind: " + ", ".join(f"{a.split('.')[-2]}.{a.split('.')[-1]} {b:.2e}" for a, b in worst.items()))
    assert all(r < _gate(key) for key, r in worst.items()), worst


def test_whole_tower_training_231_crops_checkpointed(weights, record_property):
    """The HD workload of the whole-tower benchmark: 231 crops, every parameter trainable, gradient checkpointing on.  The outputs have
    the inference bits; all 373 gradients hold the gates of the N = 29 case of test_clip_tower_embed_gpu.py against the fp64 oracle
    (4 crops at a time)."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    n = 231
    model = _train_model(weights, 0, embed=True)
    model.gradient_checkpointing = True
    t = CLIPVisionTowerB200(model, trainable_layers=LAYERS, train_embeddings=True)
    images = cto.make_images(n, seed=121, device=DEV).bfloat16()
    with torch.no_grad():
        ref_outs = CLIPVisionTowerB200(model).hidden_states(images)
    d_outs = _d_outs(n, 122)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    outs = t.hidden_states(images)
    assert outs[3].grad_fn.checkpoint
    for a, b, j in zip(outs, ref_outs, cto.OUT_LAYERS):
        assert torch.equal(a, b), j
    _backward(outs, d_outs)
    del outs, ref_outs
    peak = torch.cuda.max_memory_allocated() - base
    record_property("step_peak_bytes", peak)
    got = _grads(model)
    assert len(got) == 373 and all(g is not None for g in got.values())
    assert torch.equal(got[EMBED_NAMES[1]], got[EMBED_NAMES[2]][0])              # d class_embedding = d position_embedding[0], bitwise
    t0 = time.perf_counter()
    eg, lg = cte.parameter_gradients_chunked(weights, images, d_outs, chunk=4, device=DEV)
    torch.cuda.synchronize()
    record_property("oracle_seconds", round(time.perf_counter() - t0, 1))
    errors = {}
    for key, name in zip(cte.EMBED_KEYS, EMBED_NAMES):
        errors[key] = _rel(got[name], eg[key])
    worst = _layer_errors(got, lg, 0)
    print(f"\nN={n}: step peak {peak / GiB:.2f} GiB; embedding stage rel-RMS " + ", ".join(f"{k} {v:.2e}" for k, v in errors.items()) +
          "; worst layer rel-RMS " + ", ".join(f"{a.split('.')[-2]}.{a.split('.')[-1]} {b:.2e}" for a, b in worst.items()))
    assert all(r < _gate(key) for key, r in errors.items()), errors
    assert all(r < _gate(key) for key, r in worst.items()), worst
