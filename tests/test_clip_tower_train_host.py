"""Training the top of the CLIP tower, host side (no CUDA): include/tokenpacker_b200_clip_tower_train.h, its exports and its ctypes
binding agree; a plain-C consumer links it; the size queries and argument checks answer before any CUDA call; CLIPVisionTowerB200
validates ``trainable_layers``; the autograd oracle agrees with the forward oracle and with finite differences."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import clip_tower_oracle as cto
from oracle import clip_tower_train_oracle as ctt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower_train.h")


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_clip_tower_backward", "tp_clip_tower_backward_workspace_bytes", "tp_clip_tower_forward_train",
                           "tp_clip_tower_train_saved_bytes", "tp_clip_tower_train_workspace_bytes"]
    assert sorted(_lib.CLIP_TOWER_TRAIN_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES, _lib.LAYERS_SIGNATURES,
                  _lib.CLIP_TOWER_SIGNATURES, _lib.CLIP_TOWER_F16_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.CLIP_TOWER_TRAIN_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"
    assert C.sizeof(_lib.TpClipTowerLayerGrads) == 16 * C.sizeof(C.c_void_p) == C.sizeof(_lib.TpClipTowerLayer)


def test_plain_c_consumer_of_the_train_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_tower_train")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_tower_train.c")
    text = open(src).read()
    for name in _header_functions():
        assert name in text, f"{name} missing from abi_check_clip_tower_train.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip tower train ok" in r.stdout


def test_size_queries():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    queries = (lib.tp_clip_tower_train_saved_bytes, lib.tp_clip_tower_train_workspace_bytes, lib.tp_clip_tower_backward_workspace_bytes)
    for q in queries:
        assert q(0, 1) == 0 and q(-1, 1) == 0 and q(1, 0) == 0 and q(1, 24) == 0 and q(1, -1) == 0
        for k in (1, 4, 23):
            assert 0 < q(1, k) < q(2, k) < q(64, k)                                   # growing with the crops
        for n in (1, 64):
            assert q(n, 1) <= q(n, 4) <= q(n, 23)                                     # never shrinking with the layers
    # the saved set: 34 KiB per token plus the softmax statistics, per layer; the derived weights once per layer
    per_crop = lib.tp_clip_tower_train_saved_bytes(2, 1) - lib.tp_clip_tower_train_saved_bytes(1, 1)
    assert 577 * 34 * 1024 + 16 * 640 * 4 <= per_crop <= 577 * 34 * 1024 + 16 * 640 * 4 + 10 * 1024
    assert lib.tp_clip_tower_train_saved_bytes(3, 7) == 7 * lib.tp_clip_tower_train_saved_bytes(3, 1)
    assert lib.tp_clip_tower_train_workspace_bytes(3, 2) >= lib.tp_clip_tower_workspace_bytes(3) + 3 * 577 * 4096 * 4


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    bad, small = _lib.TP_ERR_INVALID_ARGUMENT, _lib.TP_ERR_WORKSPACE_TOO_SMALL
    w = _lib.TpClipTowerWeights(*([4096] * 5))
    for i in range(23):
        w.layers[i] = _lib.TpClipTowerLayer(*([4096] * 16))
    outs = (C.c_void_p * 4)(4096, 8192, 12288, 16384)
    cs = 3 * 336 * 336
    sb, wsb, bwsb = (q(1, 2) for q in (lib.tp_clip_tower_train_saved_bytes, lib.tp_clip_tower_train_workspace_bytes,
                                       lib.tp_clip_tower_backward_workspace_bytes))

    def fwd(packed=4096, w=w, crops=4096, n=1, k=2, outs=outs, saved=4096, sb=sb, ws=4096, wsb=wsb):
        return lib.tp_clip_tower_forward_train(packed, C.byref(w) if w is not None else None, crops, n, cs, k, outs, saved, sb, ws, wsb, None)

    for kwargs in ({"packed": None}, {"w": None}, {"crops": None}, {"n": 0}, {"k": 0}, {"k": 24}, {"outs": None}, {"saved": None},
                   {"saved": 4096 + 16}, {"ws": None}, {"outs": (C.c_void_p * 4)(4096, 4096, 12288, 16384)}):
        assert fwd(**kwargs) == bad, kwargs
    assert fwd(sb=sb - 1) == small and fwd(wsb=wsb - 1) == small
    d_outs = (C.c_void_p * 4)(None, None, None, 4096)
    grads = (_lib.TpClipTowerLayerGrads * 2)()

    def bwd(w=w, saved=4096, n=1, k=2, d_outs=d_outs, grads=grads, ws=4096, wsb=bwsb):
        return lib.tp_clip_tower_backward(C.byref(w) if w is not None else None, saved, n, k, d_outs, grads, ws, wsb, None)

    for kwargs in ({"w": None}, {"saved": None}, {"n": 0}, {"k": 0}, {"k": 24}, {"d_outs": None}, {"grads": None}, {"ws": None},
                   {"d_outs": (C.c_void_p * 4)(None, 4096 + 2, None, 4096)}):
        assert bwd(**kwargs) == bad, kwargs
    assert bwd(wsb=bwsb - 1) == small
    odd = (_lib.TpClipTowerLayerGrads * 2)()
    odd[1].ln2_b = 4096 + 2
    assert bwd(grads=odd) == bad
    holey = _lib.TpClipTowerWeights.from_buffer_copy(w)
    holey.layers[22].o_w = None
    assert bwd(w=holey) == bad


def _fake_model():
    w = {k: v.bfloat16() for k, v in cto.make_weights(0, seed=0).items()}
    for i in range(23):                                               # tiny stand-ins: only names and config are looked at here
        for key in cto.layer_keys(i).values():
            w[key] = torch.zeros(1, dtype=torch.bfloat16)
    return cto.FakeCLIPVisionModel(w)


def test_constructor_validates_trainable_layers():
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _fake_model()
    assert CLIPVisionTowerB200(model).trainable_layers == 0
    assert CLIPVisionTowerB200(model, trainable_layers=23).trainable_layers == 23
    for bad in (-1, 24, 2.0, "4", True, None):
        with pytest.raises(ValueError, match="trainable_layers"):
            CLIPVisionTowerB200(model, trainable_layers=bad)
    with pytest.raises(ValueError, match="fp16"):
        CLIPVisionTowerB200(model, dtype=torch.float16, trainable_layers=1)
    assert CLIPVisionTowerB200(model, dtype=torch.float16, trainable_layers=0).trainable_layers == 0


def test_default_tower_still_refuses_gradients_and_trainable_tower_refuses_crop_gradients():
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _fake_model()
    crops = torch.zeros(1, 3, 336, 336)
    next(iter(model.parameters())).requires_grad_(True)
    with pytest.raises(NotImplementedError, match="forward only"):
        CLIPVisionTowerB200(model).hidden_states(crops)                       # K = 0: a parameter that requires grad is refused, as before
    t = CLIPVisionTowerB200(model, trainable_layers=2)
    with pytest.raises(NotImplementedError, match="forward only"):
        t.hidden_states(crops.clone().requires_grad_(True))
    with pytest.raises(RuntimeError, match="no CPU path"):                    # frozen parameters may require grad with K > 0: no refusal for them
        t.hidden_states(crops)
    assert len(t._trainable_params()) == 32 and len(CLIPVisionTowerB200(model)._trainable_params()) == 0


def test_oracle_layer_is_the_forward_oracles_layer():
    w = cto.make_weights(2, seed=3)
    images = cto.make_images(1, seed=4)
    with torch.no_grad():
        ref = cto.forward(w, images, 2, torch.float64)
        params = [ctt.layer_params(w, i, torch.float64) for i in range(2)]
        x = ref[0]
        for i in range(2):
            x = ctt.layer(params[i], x)
            assert float((x - ref[i + 1]).abs().max()) <= 1e-12 * float(ref[i + 1].abs().max())


def test_oracle_gradients_match_finite_differences():
    """2 layers, 1 crop, both trainable: the directional derivative of the loss along a random direction in parameter space, by central
    differences in fp64, against <gradient, direction>."""
    w = cto.make_weights(2, seed=5)
    images = cto.make_images(1, seed=6)
    g = torch.Generator().manual_seed(7)
    d_outs = {1: torch.randn(1, 577, 1024, generator=g, dtype=torch.float64), 2: torch.randn(1, 577, 1024, generator=g, dtype=torch.float64)}
    saved_outs = cto.OUT_LAYERS
    cto.OUT_LAYERS = (1, 2)                                                   # the 2-layer stand-in's "hidden states of interest"
    try:
        grads, _ = ctt.parameter_gradients(w, images, 2, d_outs, n_layers=2)
        direction = {cto.layer_keys(i)[k]: torch.randn(w[cto.layer_keys(i)[k]].shape, generator=g, dtype=torch.float64)
                     for i in range(2) for k in ctt.PARAM_KEYS}
        analytic = sum(float((grads[i][k] * direction[cto.layer_keys(i)[k]]).sum()) for i in range(2) for k in ctt.PARAM_KEYS)

        def loss(eps):
            wd = {k: v.double() + (eps * direction[k] if k in direction else 0) for k, v in w.items()}
            with torch.no_grad():
                hs = cto.forward(wd, images, 2, torch.float64)
            return float(sum((hs[j] * d_outs[j]).sum() for j in (1, 2)))

        eps = 1e-5
        numeric = (loss(eps) - loss(-eps)) / (2 * eps)
    finally:
        cto.OUT_LAYERS = saved_outs
    assert abs(numeric - analytic) <= 1e-6 * abs(analytic), (numeric, analytic)
