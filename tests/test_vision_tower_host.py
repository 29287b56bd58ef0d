"""LLaVA's vision-tower seam, host side (no CUDA): include/tokenpacker_b200_clip_tower_interleaved.h, its exports and its ctypes
binding agree; a plain-C consumer links it; the interleaved entry points refuse bad arguments before any CUDA call; the drop-in
``CLIPVisionTower`` has the reference's surface and state_dict keys and refuses what it cannot run; ``build_vision_tower`` with
``delay_load`` and ``load_model`` works from a ``save_pretrained`` directory."""
import ctypes as C
import os
import re
import shutil
import subprocess
from types import SimpleNamespace

import pytest
import torch

from oracle import clip_tower_oracle as cto

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower_interleaved.h")


def _header_functions(path=HEADER):
    text = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_clip_tower_forward_interleaved", "tp_clip_tower_forward_interleaved_f16"]
    assert sorted(_lib.CLIP_TOWER_INTERLEAVED_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES, _lib.LAYERS_SIGNATURES,
                  _lib.CLIP_TOWER_SIGNATURES, _lib.CLIP_TOWER_F16_SIGNATURES, _lib.CLIP_TOWER_TRAIN_SIGNATURES,
                  _lib.CLIP_TOWER_CKPT_SIGNATURES, _lib.CLIP_TOWER_EMBED_SIGNATURES, _lib.CROP_GRAD_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.CLIP_TOWER_INTERLEAVED_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"
    assert '#include "tokenpacker_b200_clip_tower_f16.h"' in open(HEADER).read()
    # the dense entry points are declared as before
    assert sorted(_header_functions(os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower.h"))) == sorted(_lib.CLIP_TOWER_SIGNATURES)
    assert sorted(_header_functions(os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower_f16.h"))) == \
        sorted(_lib.CLIP_TOWER_F16_SIGNATURES)


def test_plain_c_consumer_of_the_interleaved_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_tower_interleaved")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_tower_interleaved.c")
    text = open(src).read()
    for name in _header_functions():
        assert name in text, f"{name} missing from abi_check_clip_tower_interleaved.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip tower interleaved ok" in r.stdout


def test_entry_points_refuse_bad_arguments_through_the_binding():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    w = _lib.TpClipTowerWeights(*([4096] * len(_lib.CLIP_TOWER_FIELDS)))
    for i in range(_lib.CLIP_TOWER_LAYERS):
        w.layers[i] = _lib.TpClipTowerLayer(*([4096] * len(_lib.CLIP_TOWER_LAYER_FIELDS)))
    cs, P, bad = 3 * 336 * 336, 4096, _lib.TP_ERR_INVALID_ARGUMENT
    ws = lib.tp_clip_tower_workspace_bytes(1)
    f16 = lib.tp_clip_tower_forward_interleaved_f16
    bf16 = lib.tp_clip_tower_forward_interleaved
    assert bf16(P, C.byref(w), P, -1, cs, P, P, ws, None) == bad
    assert bf16(P, C.byref(w), P, 0, cs, P, P, ws, None) == bad
    assert bf16(P, C.byref(w), P, 1, cs, None, P, ws, None) == bad
    assert bf16(P, C.byref(w), P, 1, cs, P + 8, P, ws, None) == bad                  # output 16-byte aligned
    assert f16(P, C.byref(w), P, _lib.TP_CLIP_CROPS_F16, 1, cs, P + 2, P, ws, None) == bad
    assert f16(P, C.byref(w), P, 0, 1, cs, P, P, ws, None) == bad                     # crops dtype
    assert f16(P, C.byref(w), P, _lib.TP_CLIP_CROPS_BF16, 1, cs, P, P, ws - 1, None) == _lib.TP_ERR_WORKSPACE_TOO_SMALL
    # past the batch the workspace size query serves (fc1's 4 x 577 n rows must stay below 2^31)
    n_max = (1 << 31) // (577 * 4)
    assert lib.tp_clip_tower_workspace_bytes(n_max) > 0 and lib.tp_clip_tower_workspace_bytes(n_max + 1) == 0
    assert bf16(P, C.byref(w), P, n_max + 1, cs, P, P, 1 << 62, None) == bad
    w.layers[16].ln1_b = None
    assert bf16(P, C.byref(w), P, 1, cs, P, P, ws, None) == bad


def _fake_model(dtype=torch.bfloat16):
    w = {k: v.to(dtype) for k, v in cto.make_weights(0, seed=0).items()}
    for i in range(23):                                               # tiny stand-ins: only names and config are looked at here
        for key in cto.layer_keys(i).values():
            w[key] = torch.zeros(1, dtype=dtype)
    return cto.FakeCLIPVisionModel(w)


def _args(select_layer=-2, select_feature=None):
    args = SimpleNamespace(mm_vision_select_layer=select_layer)
    if select_feature is not None:
        args.mm_vision_select_feature = select_feature
    return args


def test_surface_of_a_wrapped_model():
    from tokenpacker_b200 import CLIPVisionTower
    model = _fake_model()
    t = CLIPVisionTower(model, _args())
    assert t.is_loaded and t.vision_tower is model and t.image_processor is None
    assert t.select_layer == -2 and t.select_feature == "patch"
    assert t.config is model.config and t.hidden_size == 1024 and t.num_patches == 576
    assert t.dtype == torch.bfloat16 and t.device == torch.device("cpu")
    d = t.dummy_feature
    assert d.shape == (1, 1024) and d.dtype == torch.bfloat16 and not d.any()
    # the reference's keys: its only submodule is the CLIPVisionModel, as self.vision_tower
    assert list(t.state_dict()) == ["vision_tower." + k for k in model.state_dict()]
    assert [n for n, _ in t.named_children()] == ["vision_tower"]
    t.half()
    assert t.dtype == torch.float16 and t.dummy_feature.dtype == torch.float16


@pytest.mark.parametrize("layer,block", [(12, 0), (16, 1), (22, 2), (23, 3), (-13, 0), (-9, 1), (-3, 2), (-2, 3)])
def test_select_layer_names_one_of_the_four_hidden_states(layer, block):
    from tokenpacker_b200 import CLIPVisionTower
    assert CLIPVisionTower(_fake_model(), _args(layer))._block == block          # 24 layers: hidden_states[-2] is [23]


@pytest.mark.parametrize("layer", [-1, 24, 0, 11, 13, 21, -26, 25, -12, True, "23", None, 23.0])
def test_other_select_layers_are_refused_at_construction(layer):
    from tokenpacker_b200 import CLIPVisionTower
    with pytest.raises(NotImplementedError, match=r"12, 16, 22, 23"):
        CLIPVisionTower(_fake_model(), _args(layer))


def test_forward_refusals():
    from tokenpacker_b200 import CLIPVisionTower
    crops = torch.zeros(1, 3, 336, 336, dtype=torch.bfloat16)
    t = CLIPVisionTower(_fake_model(), _args(-2, "cls"))
    with pytest.raises(ValueError, match="Unexpected select feature: cls"):
        t(crops)
    t = CLIPVisionTower(_fake_model(), _args(-2, "cls_patch"))
    with pytest.raises(TypeError, match="list"):
        t([crops[0], crops[0]])
    with pytest.raises(RuntimeError, match="no CPU path"):                   # accepted: it fails only for want of a GPU
        t(crops)
    with pytest.raises(ValueError, match=r"\[N,3,336,336\]"):
        t(torch.zeros(1, 3, 224, 224))


def test_interleaved_hidden_states_refusals():
    from tokenpacker_b200 import CLIPVisionTowerB200
    t = CLIPVisionTowerB200(_fake_model())
    with pytest.raises(ValueError, match=r"\[N,3,336,336\]"):
        t.interleaved_hidden_states(torch.zeros(3, 336, 336))
    with pytest.raises(NotImplementedError, match="inference only"):
        t.interleaved_hidden_states(torch.zeros(1, 3, 336, 336, requires_grad=True))
    with pytest.raises(RuntimeError, match="no CPU path"):
        t.interleaved_hidden_states(torch.zeros(1, 3, 336, 336))
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU path"):
        t.interleaved_hidden_states(torch.zeros(1, 3, 336, 336, requires_grad=True))


def test_build_vision_tower_refuses_unknown_towers():
    from tokenpacker_b200 import build_vision_tower
    for name in ("facebook/dinov2-large", "/no/such/dir", None):
        with pytest.raises(ValueError, match="Unknown vision tower"):
            build_vision_tower(SimpleNamespace(mm_vision_tower=name, mm_vision_select_layer=-2))


@pytest.fixture(scope="module")
def clip_dir(tmp_path_factory):
    """A CLIP-ViT-L/14-336-shaped CLIPVisionModel (bf16, uninitialised values) and its image processor, saved with save_pretrained."""
    transformers = pytest.importorskip("transformers")
    cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=24,
                                        patch_size=14, image_size=336, projection_dim=768)
    with torch.device("meta"):
        model = transformers.CLIPVisionModel(cfg)
    model = model.to_empty(device="cpu").to(torch.bfloat16)
    path = tmp_path_factory.mktemp("clip-vit-large-patch14-336")
    model.save_pretrained(str(path))
    transformers.CLIPImageProcessor(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336}).save_pretrained(str(path))
    return str(path), list(model.state_dict())


def test_delay_load_then_load_model(clip_dir):
    from tokenpacker_b200 import build_vision_tower
    path, keys = clip_dir
    cfg = SimpleNamespace(mm_vision_tower=path, mm_vision_select_layer=-2, mm_vision_select_feature="patch")
    t = build_vision_tower(cfg, delay_load=True)
    assert not t.is_loaded and t.vision_tower_name == path
    assert t.config.hidden_size == 1024 and t.hidden_size == 1024 and t.num_patches == 576
    assert list(t.state_dict()) == []                                    # only the config, as the reference keeps
    t.load_model()
    assert t.is_loaded and type(t.vision_tower).__name__ == "CLIPVisionModel"
    assert type(t.image_processor).__name__.startswith("CLIPImageProcessor")
    assert t.image_processor.crop_size["height"] == 336
    assert not any(p.requires_grad for p in t.vision_tower.parameters())
    assert t.config is t.vision_tower.config and t.dtype == t.vision_tower.dtype and t.device == t.vision_tower.device


def test_state_dict_keys_are_those_of_the_reference(clip_dir):
    from tokenpacker_b200 import build_vision_tower
    transformers = pytest.importorskip("transformers")
    path, keys = clip_dir
    t = build_vision_tower(SimpleNamespace(vision_tower=path, mm_vision_select_layer=23))
    assert t.is_loaded and t._block == 3
    with torch.device("meta"):
        real = transformers.CLIPVisionModel(transformers.CLIPVisionConfig.from_pretrained(path))
    assert list(t.state_dict()) == ["vision_tower." + k for k in real.state_dict()] == ["vision_tower." + k for k in keys]
    t.load_state_dict(t.state_dict())                                     # a checkpoint of the reference module loads as it is


def test_delay_load_checks_the_config(tmp_path):
    transformers = pytest.importorskip("transformers")
    from tokenpacker_b200 import CLIPVisionTower
    transformers.CLIPVisionConfig(hidden_size=768, intermediate_size=3072, num_attention_heads=12, num_hidden_layers=12, patch_size=16,
                                  image_size=224).save_pretrained(str(tmp_path))
    with pytest.raises(NotImplementedError, match="CLIP-ViT-L/14-336"):
        CLIPVisionTower(str(tmp_path), _args(), delay_load=True)
