"""Gradients to the pixels, host side (no CUDA): include/tokenpacker_b200_clip_tower_crop_grad.h, its exports and its ctypes binding
agree; a plain-C consumer links it; the tower's ``input_grad`` flag and its refusals; the fp64 tiling oracle against
torch.autograd.gradcheck; and the HD backward plan's inverse-tap tables, applied in fp64, against the oracle's adjoint."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import clip_tower_oracle as cto
from oracle import crop_grad_oracle as cgo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower_crop_grad.h")


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_clip_tower_backward_crops", "tp_hd_tile_batch_backward", "tp_hd_tile_batch_backward_plan"]
    assert sorted(_lib.CROP_GRAD_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES, _lib.LAYERS_SIGNATURES,
                  _lib.CLIP_TOWER_SIGNATURES, _lib.CLIP_TOWER_F16_SIGNATURES, _lib.CLIP_TOWER_TRAIN_SIGNATURES, _lib.CLIP_TOWER_CKPT_SIGNATURES,
                  _lib.CLIP_TOWER_EMBED_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.CROP_GRAD_SIGNATURES[name][1]), name
    text = open(HEADER).read()
    body = re.search(r"typedef struct tp_hd_image_grad \{(.*?)\}", text, flags=re.S).group(1)
    assert re.findall(r"(\w+)[,;]", body) == [f for f, _ in _lib.TpHdImageGrad._fields_]
    assert int(re.search(r"#define TP_CROP_GRAD_BF16 (\d+)", text).group(1)) == _lib.TP_CROP_GRAD_BF16
    assert int(re.search(r"#define TP_CROP_GRAD_F32 (\d+)", text).group(1)) == _lib.TP_CROP_GRAD_F32
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"


def test_plain_c_consumer_of_the_crop_grad_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_tower_crop_grad")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_tower_crop_grad.c")
    text = open(src).read()
    for name in _header_functions():
        assert name in text, f"{name} missing from abi_check_clip_tower_crop_grad.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip tower crop grad ok" in r.stdout


def _fake_model():
    w = {k: v.bfloat16() for k, v in cto.make_weights(0, seed=0).items()}
    for i in range(23):                                               # tiny stand-ins: only names and config are looked at here
        for key in cto.layer_keys(i).values():
            w[key] = torch.zeros(1, dtype=torch.bfloat16)
    return cto.FakeCLIPVisionModel(w)


def test_input_grad_flag():
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _fake_model()
    t = CLIPVisionTowerB200(model)
    assert t.input_grad is False
    crops = torch.zeros(1, 3, 336, 336, requires_grad=True)
    with pytest.raises(NotImplementedError, match="forward only"):          # the default refuses crops that require grad, as before
        t.hidden_states(crops)
    for bad in (1, "yes", None):
        with pytest.raises(ValueError, match="input_grad"):
            t.input_grad = bad
    t.input_grad = True
    assert t.input_grad and "input_grad" not in str(list(t.state_dict()))
    with pytest.raises(RuntimeError, match="no CPU path"):                  # accepted: it fails only for want of a GPU
        t.hidden_states(crops)
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU path"):
        t.hidden_states(crops)
    f16 = CLIPVisionTowerB200(model, dtype=torch.float16)
    with pytest.raises(ValueError, match="fp16 tower is forward only"):
        f16.input_grad = True
    assert f16.input_grad is False


# (h, w, patch_num): 1 x 1 grids (no thumbnail), wide and tall grids, every patch_num, extreme aspect ratios
TILE_CASES = [(8, 8, 9), (12, 11, 16), (5, 7, 9), (20, 400, 9), (400, 20, 16), (100, 30, 25), (3, 90, 25), (61, 17, 16)]


@pytest.mark.parametrize("h,w,pn", TILE_CASES[:4])
def test_tiling_oracle_passes_gradcheck(h, w, pn):
    g = torch.Generator().manual_seed(h * 1000 + w)
    image = torch.randn(3, h, w, generator=g, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda x: cgo.tile(x, pn)[0], (image,), fast_mode=True, eps=1e-6, atol=1e-8, rtol=1e-6)


def _apply_tables(taps, off, n, dense_out):
    """The table at ``off`` (over n indices) as a dense [n, dense_out] fp64 matrix M: M[s, d] = sum of the weights of entries (d, w)."""
    counts = taps[off:off + n + 1]
    ent = taps[off + n + 1:off + n + 1 + 2 * counts[n]].reshape(-1, 2)
    m = np.zeros((n, dense_out))
    for s in range(n):
        for d, wbits in ent[counts[s]:counts[s + 1]]:
            m[s, d] += float(np.array([wbits], dtype=np.int32).view(np.float32)[0])
    return m


@pytest.mark.parametrize("h,w,pn", TILE_CASES)
def test_backward_plan_tables_are_the_adjoint_of_the_tiling(h, w, pn):
    """d image = Ry^T (d canvas + Ty^T d thumb Tx) Rx with the plan's tables as the matrices, against the fp64 oracle's autograd."""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    hs, ws = (C.c_int64 * 1)(h), (C.c_int64 * 1)(w)
    hb, wb, nc = (C.c_int * 1)(), (C.c_int * 1)(), C.c_int64(0)
    desc = (_lib.TpHdImage * 1)()
    assert lib.tp_hd_tile_batch_plan(hs, ws, None, 1, pn, desc, None, hb, wb, C.byref(nc)) == 0
    words, most = C.c_int64(0), C.c_int64(0)
    assert lib.tp_hd_tile_batch_backward_plan(desc, 1, None, None, None, C.byref(words), C.byref(most)) == 0
    assert most.value == h * w
    taps = np.zeros(words.value, dtype=np.int32)
    grads = (_lib.TpHdImageGrad * 1)()
    assert lib.tp_hd_tile_batch_backward_plan(desc, 1, None, grads, taps.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(words),
                                              C.byref(most)) == 0
    im, g = desc[0], grads[0]
    hb, wb = hb[0], wb[0]
    rng = np.random.default_rng(h * 7 + w)
    d_crops = rng.standard_normal((nc.value, 3, 336, 336))
    canvas = np.zeros((3, 336 * hb, 336 * wb))
    for i in range(hb):
        for j in range(wb):
            canvas[:, 336 * i:336 * (i + 1), 336 * j:336 * (j + 1)] = d_crops[i * wb + j]
    ry = _apply_tables(taps, g.row_taps, h, im.h_r)
    rx = _apply_tables(taps, g.col_taps, w, im.w_r)
    d_canvas = canvas[:, :im.h_r, :im.w_r]
    if hb * wb > 1:
        ty = _apply_tables(taps, g.thumb_row_taps, im.h_r, im.h_t)
        tx = _apply_tables(taps, g.thumb_col_taps, im.w_r, im.w_t)
        d_canvas = d_canvas + np.einsum("yi,cij,xj->cyx", ty, d_crops[-1][:, :im.h_t, :im.w_t], tx, optimize=True)
    else:
        assert g.thumb_row_taps == -1 and g.thumb_col_taps == -1 and nc.value == 1
    got = np.einsum("sy,cyx,tx->cst", ry, d_canvas, rx, optimize=True)
    image = torch.zeros(3, h, w, dtype=torch.float64)
    want = cgo.tile_gradients([image], torch.from_numpy(d_crops), pn)[0].numpy()
    rel = np.sqrt(((got - want) ** 2).mean()) / np.sqrt((want ** 2).mean())
    assert rel < 1e-4, rel                                   # fp32 tap coordinates against fp64 ones
