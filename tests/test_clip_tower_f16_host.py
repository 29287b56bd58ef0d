"""The fp16 CLIP tower, host side (no CUDA): include/tokenpacker_b200_clip_tower_f16.h, its exports and its ctypes binding agree; a
plain-C consumer links it; the two entry points refuse bad arguments before any CUDA call; the tile engine refuses f16 / bf16 mixes
before any launch; CLIPVisionTowerB200 validates ``dtype=``; the oracle's fp16 eager tower keeps the bf16 one's rounding points."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import clip_tower_f16_oracle as ct16
from oracle import clip_tower_oracle as cto

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower_f16.h")
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_clip_tower_f16_hooks.so")


def _header_functions(path=HEADER):
    text = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_clip_tower_forward_f16", "tp_clip_tower_pack_weights_f16"]
    assert sorted(_lib.CLIP_TOWER_F16_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES, _lib.LAYERS_SIGNATURES,
                  _lib.CLIP_TOWER_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.CLIP_TOWER_F16_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"
    text = open(HEADER).read()
    assert '#include "tokenpacker_b200_clip_tower.h"' in text
    for name, value in (("TP_CLIP_CROPS_BF16", _lib.TP_CLIP_CROPS_BF16), ("TP_CLIP_CROPS_F16", _lib.TP_CLIP_CROPS_F16)):
        assert re.search(rf"#define {name} {value}\b", text), name
    # the bf16 tower's header is unchanged in what it declares
    assert sorted(_header_functions(os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower.h"))) == sorted(_lib.CLIP_TOWER_SIGNATURES)


def test_plain_c_consumer_of_the_f16_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_tower_f16")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_tower_f16.c")
    text = open(src).read()
    for name in _header_functions():
        assert name in text, f"{name} missing from abi_check_clip_tower_f16.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip tower f16 ok" in r.stdout


def _weights(value=4096):
    from tokenpacker_b200 import _lib
    w = _lib.TpClipTowerWeights(*([value] * 5))
    for i in range(23):
        w.layers[i] = _lib.TpClipTowerLayer(*([value] * 16))
    return w


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    bad, small = _lib.TP_ERR_INVALID_ARGUMENT, _lib.TP_ERR_WORKSPACE_TOO_SMALL
    w = _weights()
    outs = (C.c_void_p * 4)(4096, 8192, 12288, 16384)
    cs = 3 * 336 * 336
    ws_bytes = lib.tp_clip_tower_workspace_bytes(1)

    def fwd(packed=4096, w=w, crops=4096, dt=_lib.TP_CLIP_CROPS_F16, n=1, cs=cs, outs=outs, ws=4096, wsb=ws_bytes):
        return lib.tp_clip_tower_forward_f16(packed, C.byref(w) if w is not None else None, crops, dt, n, cs, outs, ws, wsb, None)

    for dt in (0, 3, -1, 16):                                               # 1 = bf16 crops, 2 = f16 crops; nothing else
        assert fwd(dt=dt) == bad, dt
    for dt in (_lib.TP_CLIP_CROPS_BF16, _lib.TP_CLIP_CROPS_F16):
        assert fwd(dt=dt, wsb=ws_bytes - 1) == small                        # every other argument valid: only the size is refused
        assert fwd(dt=dt, packed=None) == bad
        assert fwd(dt=dt, packed=4096 + 128) == bad                         # 256-byte alignment
        assert fwd(dt=dt, w=None) == bad
        assert fwd(dt=dt, crops=None) == bad
        assert fwd(dt=dt, crops=4096 + 1) == bad
        assert fwd(dt=dt, n=0) == bad
        assert fwd(dt=dt, n=-3) == bad
        assert fwd(dt=dt, cs=cs - 1) == bad
        assert fwd(dt=dt, outs=None) == bad
        assert fwd(dt=dt, outs=(C.c_void_p * 4)(4096, None, 12288, 16384)) == bad
        assert fwd(dt=dt, outs=(C.c_void_p * 4)(4096, 8192 + 2, 12288, 16384)) == bad   # misaligned
        assert fwd(dt=dt, outs=(C.c_void_p * 4)(4096, 8192, 12288, 8192)) == bad       # one destination twice
        assert fwd(dt=dt, ws=None) == bad
        assert fwd(dt=dt, ws=4096 + 64) == bad
    holey = _weights()
    holey.layers[7].fc2_w = None
    assert fwd(w=holey) == bad
    odd = _weights()
    odd.pos_emb = 4096 + 2
    assert fwd(w=odd) == bad
    assert lib.tp_clip_tower_pack_weights_f16(C.byref(odd), 4096, lib.tp_clip_tower_packed_bytes(), None) == bad
    assert lib.tp_clip_tower_pack_weights_f16(C.byref(holey), 4096, lib.tp_clip_tower_packed_bytes(), None) == bad
    assert lib.tp_clip_tower_pack_weights_f16(C.byref(w), 4096, lib.tp_clip_tower_packed_bytes() - 1, None) == small
    assert lib.tp_clip_tower_pack_weights_f16(C.byref(w), 4096 + 16, lib.tp_clip_tower_packed_bytes(), None) == bad
    assert lib.tp_clip_tower_pack_weights_f16(None, 4096, lib.tp_clip_tower_packed_bytes(), None) == bad


def test_engine_refuses_mixed_f16_and_bf16_launches():
    """A group (one launch_gemms call), a chain and a pair-kernel group that mix a bf16 and an f16 item are refused before any CUDA
    call (each instantiation reads and writes one 16-bit format)."""
    from tokenpacker_b200 import _lib
    hooks = C.CDLL(HOOKS)
    hooks.tpc_mixed_precision.restype = C.c_int
    hooks.tpc_mixed_precision.argtypes = [C.c_int]
    for how in (0, 1, 2):
        assert hooks.tpc_mixed_precision(how) == _lib.TP_ERR_INVALID_ARGUMENT, how


def _tiny_model():
    w = {k: v.bfloat16() for k, v in cto.make_weights(0, seed=0).items()}
    for i in range(23):                                                   # tiny stand-ins: only names and config are looked at here
        for key in cto.layer_keys(i).values():
            w[key] = torch.zeros(1, dtype=torch.bfloat16)
    return cto.FakeCLIPVisionModel(w)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.int8, torch.uint8, "float16", torch.float8_e4m3fn])
def test_dtype_validation(dtype):
    from tokenpacker_b200 import CLIPVisionTowerB200
    with pytest.raises(ValueError, match="dtype"):
        CLIPVisionTowerB200(_tiny_model(), dtype=dtype)


def test_dtype_choices_and_refusals():
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _tiny_model()
    assert CLIPVisionTowerB200(model).dtype == torch.bfloat16
    assert CLIPVisionTowerB200(model, dtype=torch.bfloat16).dtype == torch.bfloat16
    t = CLIPVisionTowerB200(model, dtype=torch.float16)
    assert t.dtype == torch.float16
    with pytest.raises(ValueError):
        t.hidden_states(torch.zeros(1, 3, 224, 224, dtype=torch.float16))
    with pytest.raises(NotImplementedError, match="forward only"):
        t.hidden_states(torch.zeros(1, 3, 336, 336, requires_grad=True))
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU path"):
            t.hidden_states(torch.zeros(1, 3, 336, 336, dtype=torch.float16))


def test_f16_eager_oracle_rounds_where_the_bf16_one_does():
    """forward_eager is one function for both 16-bit formats: on a tiny 1-layer tower the fp16 restatement returns fp16 tensors and
    agrees with the fp64 network far more closely than the bf16 one (unit roundoff 2^-11 against 2^-8); forward_bf16_eager is that
    function at bf16."""
    w = cto.round_bf16(cto.make_weights(1, seed=3))
    images = cto.make_images(1, seed=4)
    with torch.no_grad():
        ref = cto.forward(w, images.double(), 1, torch.float64)
        h16 = ct16.forward_f16_eager(w, images, 1)
        hb = cto.forward_bf16_eager(w, images, 1)
        hb2 = ct16.forward_eager(w, images, 1, torch.bfloat16)
    assert all(h.dtype == torch.float16 for h in h16) and all(h.dtype == torch.bfloat16 for h in hb)
    for a, b in zip(hb, hb2):
        assert torch.equal(a, b)
    for i in range(2):
        e16 = float((h16[i].double() - ref[i]).norm() / ref[i].norm())
        eb = float((hb[i].double() - ref[i]).norm() / ref[i].norm())
        assert e16 < eb / 3, (i, e16, eb)
