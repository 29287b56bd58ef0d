"""The CLIP vision tower, host side (no CUDA): the torch oracle against transformers' CLIPVisionModel and against a committed fixture
written from it; include/tokenpacker_b200_clip_tower.h, its exports and its ctypes binding agree; a plain-C consumer links it; the C
entry points refuse bad arguments before any CUDA call; CLIPVisionTowerB200 refuses configurations it does not implement."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import clip_tower_oracle as cto

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower.h")
GOLDEN = os.path.join(ROOT, "tests", "golden", "clip_tower_l3.npz")


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_oracle_matches_transformers():
    transformers = pytest.importorskip("transformers")
    cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=3,
                                        image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
    model = transformers.CLIPVisionModel(cfg).eval()
    w = cto.make_weights(3, seed=4)
    missing, unexpected = model.load_state_dict({"vision_model." + k: v for k, v in w.items()}, strict=False)
    assert not unexpected and all(k.startswith("vision_model.post_layernorm") or "position_ids" in k for k in missing), (missing, unexpected)
    images = cto.make_images(1, seed=5)
    with torch.no_grad():
        hs = model(pixel_values=images, output_hidden_states=True).hidden_states
        ours = cto.forward(w, images, 3, torch.float32)
    for i in range(4):
        ref = hs[i].double()
        err = float((ours[i].double() - ref).norm() / ref.norm())
        assert err < 1e-5, (i, err)


def test_oracle_matches_the_committed_fixture():
    """tests/golden/clip_tower_l3.npz (oracle/gen_golden_clip_tower.py): sampled rows of transformers' hidden_states[0..3]"""
    z = np.load(GOLDEN)
    w = cto.make_weights(3, seed=int(z["weight_seed"]))
    images = cto.make_images(1, seed=int(z["image_seed"]))
    with torch.no_grad():
        ours = cto.forward(w, images, 3, torch.float64)
    rows = torch.from_numpy(z["rows"])
    for i in range(4):
        ref = torch.from_numpy(z[f"hs{i}"]).double()
        got = ours[i][0, rows]
        err = float((got - ref).norm() / ref.norm())
        assert err < 1e-5, (i, err)


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_clip_tower_forward", "tp_clip_tower_pack_weights", "tp_clip_tower_packed_bytes", "tp_clip_tower_workspace_bytes"]
    assert sorted(_lib.CLIP_TOWER_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES, _lib.LAYERS_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        n = 0 if params.strip() == "void" else len(params.split(","))
        assert n == len(_lib.CLIP_TOWER_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"
    # the struct mirrors the header: 5 + 23 x 16 pointers
    assert C.sizeof(_lib.TpClipTowerWeights) == (5 + 23 * 16) * C.sizeof(C.c_void_p)


def test_plain_c_consumer_of_the_clip_tower_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_tower")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_tower.c")
    text = open(src).read()
    for name in _header_functions():
        assert f"{name}" in text, f"{name} missing from abi_check_clip_tower.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip tower ok" in r.stdout


def test_sizes():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    per_layer = 3072 * 1024 * 2 + (3072 + 1024 + 4096 + 1024) * 4  # q|k|v bf16, the biases fp32
    assert per_layer * 23 <= lib.tp_clip_tower_packed_bytes() <= per_layer * 23 * 1.01 + 2 * 1024 * 1024
    assert lib.tp_clip_tower_workspace_bytes(0) == 0
    assert lib.tp_clip_tower_workspace_bytes(-1) == 0
    w1, w5 = lib.tp_clip_tower_workspace_bytes(1), lib.tp_clip_tower_workspace_bytes(5)
    assert 0 < w1 < w5 and w5 >= 5 * 577 * 1024 * 2 * 11


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    bad, small = _lib.TP_ERR_INVALID_ARGUMENT, _lib.TP_ERR_WORKSPACE_TOO_SMALL
    w = _lib.TpClipTowerWeights(*([4096] * 5))
    for i in range(23):
        w.layers[i] = _lib.TpClipTowerLayer(*([4096] * 16))
    outs = (C.c_void_p * 4)(4096, 8192, 12288, 16384)
    cs = 3 * 336 * 336
    ws_bytes = lib.tp_clip_tower_workspace_bytes(1)

    def fwd(packed=4096, w=w, crops=4096, n=1, cs=cs, outs=outs, ws=4096, wsb=ws_bytes):
        return lib.tp_clip_tower_forward(packed, C.byref(w) if w is not None else None, crops, n, cs, outs, ws, wsb, None)

    assert fwd(packed=None) == bad
    assert fwd(w=None) == bad
    assert fwd(crops=None) == bad
    assert fwd(n=0) == bad
    assert fwd(cs=cs - 1) == bad
    assert fwd(outs=None) == bad
    assert fwd(outs=(C.c_void_p * 4)(4096, None, 12288, 16384)) == bad
    assert fwd(outs=(C.c_void_p * 4)(4096, 8192 + 2, 12288, 16384)) == bad
    assert fwd(outs=(C.c_void_p * 4)(4096, 4096, 12288, 16384)) == bad       # one destination twice
    assert fwd(ws=None) == bad
    assert fwd(wsb=ws_bytes - 1) == small
    holey = _lib.TpClipTowerWeights(*([4096] * 5))
    for i in range(23):
        holey.layers[i] = _lib.TpClipTowerLayer(*([4096] * 16))
    holey.layers[7].fc2_w = None
    assert fwd(w=holey) == bad
    for field in ("class_emb", "pos_emb", "pre_ln_w", "pre_ln_b"):               # read 16 bytes at a time: 2-byte views are refused
        odd = _lib.TpClipTowerWeights(*([4096] * 5))
        for i in range(23):
            odd.layers[i] = _lib.TpClipTowerLayer(*([4096] * 16))
        setattr(odd, field, 4096 + 2)
        assert fwd(w=odd) == bad, field
    odd.pre_ln_b = 4096
    odd.layers[3].ln2_w = 4096 + 2
    assert fwd(w=odd) == bad
    assert lib.tp_clip_tower_pack_weights(C.byref(odd), 4096, lib.tp_clip_tower_packed_bytes(), None) == bad
    assert lib.tp_clip_tower_pack_weights(C.byref(holey), 4096, lib.tp_clip_tower_packed_bytes(), None) == bad
    assert lib.tp_clip_tower_pack_weights(C.byref(w), 4096, lib.tp_clip_tower_packed_bytes() - 1, None) == small
    assert lib.tp_clip_tower_pack_weights(None, 4096, lib.tp_clip_tower_packed_bytes(), None) == bad


class _Cfg(cto.FakeCLIPVisionModel.Config):
    pass


@pytest.mark.parametrize("field,value", [("hidden_size", 768), ("intermediate_size", 3072), ("num_attention_heads", 12),
                                         ("num_hidden_layers", 22), ("patch_size", 16), ("image_size", 224), ("hidden_act", "gelu"),
                                         ("layer_norm_eps", 1e-6)])
def test_refuses_other_configurations(field, value):
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = torch.nn.Linear(1, 1)
    model.config = _Cfg()
    setattr(model.config, field, value)
    with pytest.raises(NotImplementedError):
        CLIPVisionTowerB200(model)


def test_refuses_a_model_without_the_parameters_or_config():
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = torch.nn.Linear(1, 1)
    with pytest.raises(NotImplementedError):
        CLIPVisionTowerB200(model)
    model.config = _Cfg()
    with pytest.raises(NotImplementedError, match="missing"):
        CLIPVisionTowerB200(model)


def test_python_refuses_bad_input_before_device_work():
    from tokenpacker_b200 import CLIPVisionTowerB200
    w = {k: v.bfloat16() for k, v in cto.make_weights(0, seed=0).items()}
    for i in range(23):                                               # tiny stand-ins: only names and config are looked at here
        for key in cto.layer_keys(i).values():
            w[key] = torch.zeros(1, dtype=torch.bfloat16)
    t = CLIPVisionTowerB200(cto.FakeCLIPVisionModel(w))
    with pytest.raises(ValueError):
        t.hidden_states(torch.zeros(1, 3, 224, 224))
    with pytest.raises(ValueError):
        t.hidden_states(torch.zeros(3, 336, 336))
    with pytest.raises(NotImplementedError, match="forward only"):
        t.hidden_states(torch.zeros(1, 3, 336, 336, requires_grad=True))
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU path"):
            t.hidden_states(torch.zeros(1, 3, 336, 336))
