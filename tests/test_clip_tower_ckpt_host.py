"""Gradient checkpointing for the CLIP tower's trainable layers, host side (no CUDA): include/tokenpacker_b200_clip_tower_ckpt.h, its
exports and its ctypes binding agree; a plain-C consumer links it; the size queries and argument checks answer before any CUDA call;
the tower checkpoints exactly when the wrapped model asks for it."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import clip_tower_oracle as cto

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower_ckpt.h")
N_PAST_LIMIT = (1 << 31) // (577 * 4) + 1                  # the first crop count tp_clip_tower_workspace_bytes refuses


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_clip_tower_backward_ckpt", "tp_clip_tower_ckpt_backward_workspace_bytes", "tp_clip_tower_ckpt_saved_bytes",
                           "tp_clip_tower_forward_ckpt"]
    assert sorted(_lib.CLIP_TOWER_CKPT_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES, _lib.LAYERS_SIGNATURES,
                  _lib.CLIP_TOWER_SIGNATURES, _lib.CLIP_TOWER_F16_SIGNATURES, _lib.CLIP_TOWER_TRAIN_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.CLIP_TOWER_CKPT_SIGNATURES[name][1]), name
    # the pair takes exactly the arguments of the training pair it stands in for
    assert _lib.CLIP_TOWER_CKPT_SIGNATURES["tp_clip_tower_forward_ckpt"] == _lib.CLIP_TOWER_TRAIN_SIGNATURES["tp_clip_tower_forward_train"]
    assert _lib.CLIP_TOWER_CKPT_SIGNATURES["tp_clip_tower_backward_ckpt"] == _lib.CLIP_TOWER_TRAIN_SIGNATURES["tp_clip_tower_backward"]
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"


def test_plain_c_consumer_of_the_ckpt_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_tower_ckpt")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_tower_ckpt.c")
    text = open(src).read()
    for name in _header_functions():
        assert name in text, f"{name} missing from abi_check_clip_tower_ckpt.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip tower ckpt ok" in r.stdout


def test_size_queries():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    saved, bwd = lib.tp_clip_tower_ckpt_saved_bytes, lib.tp_clip_tower_ckpt_backward_workspace_bytes
    for q in (saved, bwd):
        assert q(0, 1) == 0 and q(-1, 1) == 0 and q(1, 0) == 0 and q(1, 24) == 0 and q(1, -1) == 0
        assert q(N_PAST_LIMIT, 1) == 0 and q(N_PAST_LIMIT - 1, 1) > 0
        for k in (1, 4, 23):
            assert 0 < q(1, k) < q(2, k) < q(64, k)                                   # growing with the crops
    for n in (1, 3, 29, 231):
        for k in (2, 7, 23):
            assert saved(n, k) == k * saved(n, 1)
            assert bwd(n, k) == bwd(n, 1)                                             # one layer's scratch, whatever K
        # the scratch saved set and fc1's fp32 pre-activation on top of the backward's own workspace
        assert bwd(n, 1) >= lib.tp_clip_tower_backward_workspace_bytes(n, 1) + lib.tp_clip_tower_train_saved_bytes(n, 1) + n * 577 * 4096 * 4
        assert saved(n, 1) < lib.tp_clip_tower_train_saved_bytes(n, 1)
    # per layer: the layer's input (577 tokens x 1024 bf16 per crop) and the derived weights (q|k|v and fp32 biases, once per layer)
    per_crop = saved(2, 1) - saved(1, 1)
    assert 577 * 2048 <= per_crop <= 577 * 2048 + 1024
    assert saved(1, 1) - 577 * 2048 >= 3 * 1024 * 1024 * 2 + 9 * 1024 * 4


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    bad, small = _lib.TP_ERR_INVALID_ARGUMENT, _lib.TP_ERR_WORKSPACE_TOO_SMALL
    w = _lib.TpClipTowerWeights(*([4096] * 5))
    for i in range(23):
        w.layers[i] = _lib.TpClipTowerLayer(*([4096] * 16))
    outs = (C.c_void_p * 4)(4096, 8192, 12288, 16384)
    cs = 3 * 336 * 336
    sb, wsb, bwsb = lib.tp_clip_tower_ckpt_saved_bytes(1, 2), lib.tp_clip_tower_workspace_bytes(1), lib.tp_clip_tower_ckpt_backward_workspace_bytes(1, 2)

    def fwd(packed=4096, w=w, crops=4096, n=1, k=2, outs=outs, saved=4096, sb=sb, ws=4096, wsb=wsb):
        return lib.tp_clip_tower_forward_ckpt(packed, C.byref(w) if w is not None else None, crops, n, cs, k, outs, saved, sb, ws, wsb, None)

    for kwargs in ({"packed": None}, {"w": None}, {"crops": None}, {"n": 0}, {"n": N_PAST_LIMIT}, {"k": 0}, {"k": 24}, {"outs": None},
                   {"saved": None}, {"saved": 4096 + 16}, {"ws": None}, {"outs": (C.c_void_p * 4)(4096, 4096, 12288, 16384)}):
        assert fwd(**kwargs) == bad, kwargs
    assert fwd(sb=sb - 1) == small and fwd(wsb=wsb - 1) == small
    # the inference workspace is all the checkpointed forward needs; the training forward's query is not asked
    assert wsb < lib.tp_clip_tower_train_workspace_bytes(1, 2)
    d_outs = (C.c_void_p * 4)(None, None, None, 4096)
    grads = (_lib.TpClipTowerLayerGrads * 2)()

    def bwd(w=w, saved=4096, n=1, k=2, d_outs=d_outs, grads=grads, ws=4096, wsb=bwsb):
        return lib.tp_clip_tower_backward_ckpt(C.byref(w) if w is not None else None, saved, n, k, d_outs, grads, ws, wsb, None)

    for kwargs in ({"w": None}, {"saved": None}, {"saved": 4096 + 16}, {"n": 0}, {"k": 0}, {"k": 24}, {"d_outs": None}, {"grads": None},
                   {"ws": None}, {"ws": 4096 + 64}, {"d_outs": (C.c_void_p * 4)(None, 4096 + 2, None, 4096)}):
        assert bwd(**kwargs) == bad, kwargs
    assert bwd(wsb=bwsb - 1) == small
    assert bwd(wsb=lib.tp_clip_tower_backward_workspace_bytes(1, 2)) == small           # the non-checkpointed backward's is too small
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


def test_mode_follows_the_wrapped_models_switch():
    from tokenpacker_b200 import CLIPVisionTowerB200
    from tokenpacker_b200.tower import wants_gradient_checkpointing
    model = _fake_model()
    t = CLIPVisionTowerB200(model, trainable_layers=2)
    assert model.training and not wants_gradient_checkpointing(t.vision_model)          # no switch: no checkpointing
    model.gradient_checkpointing = True
    assert wants_gradient_checkpointing(t.vision_model)
    model.eval()                                                                         # transformers recomputes only in training
    assert not wants_gradient_checkpointing(t.vision_model)
    model.train()
    model.gradient_checkpointing = False
    assert not wants_gradient_checkpointing(t.vision_model)
    # a flag on a submodule counts, as transformers sets it on the encoder
    outer = torch.nn.Sequential(torch.nn.Identity(), torch.nn.Sequential(model))
    model.gradient_checkpointing = 1
    assert wants_gradient_checkpointing(outer)
    assert not hasattr(t, "gradient_checkpointing")                                     # the tower has no switch of its own


def test_mode_follows_transformers_gradient_checkpointing_enable():
    transformers = pytest.importorskip("transformers")
    from tokenpacker_b200.tower import wants_gradient_checkpointing
    cfg = transformers.CLIPVisionConfig(hidden_size=32, intermediate_size=64, num_attention_heads=2, num_hidden_layers=2, image_size=28,
                                        patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
    model = transformers.CLIPVisionModel(cfg).train()
    assert not wants_gradient_checkpointing(model)
    model.gradient_checkpointing_enable()
    assert model.is_gradient_checkpointing and wants_gradient_checkpointing(model)
    model.eval()
    assert not wants_gradient_checkpointing(model)
    model.train()
    assert wants_gradient_checkpointing(model)
    model.gradient_checkpointing_disable()
    assert not wants_gradient_checkpointing(model)
