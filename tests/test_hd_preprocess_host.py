"""Decoded 8-bit HD input, host side (no CUDA): the normalisation table against the reference's own ``preprocess`` (fixture), the
oracle and torchvision; the oracle's ToTensor + Normalize + tiling against the fixture; argument validation of
tp_hd_preprocess_batch and hd_preprocess_batch before any device work."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import hd_oracle as hdo
from oracle import hd_preprocess_oracle as hpo


def _ramp():
    return np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)        # [1, 256, 3]: byte u at column u, every channel


def test_table_matches_reference_and_oracle(golden_dir):
    from tokenpacker_b200.hd import norm_table
    t = norm_table()
    assert t.dtype == torch.float32 and tuple(t.shape) == (3, 256)
    ref = np.load(os.path.join(golden_dir, "hd_preprocess_u8.npz"))["table"]
    np.testing.assert_array_equal(t.numpy().view(np.uint32), ref.view(np.uint32))                      # bit for bit, all 768
    np.testing.assert_array_equal(t.numpy().view(np.uint32), hpo.preprocess_u8(_ramp())[:, 0, :].view(np.uint32))


def test_table_matches_torchvision():
    tv = pytest.importorskip("torchvision.transforms")
    from PIL import Image
    from tokenpacker_b200.hd import CLIP_MEAN, CLIP_STD, norm_table
    pre = tv.Compose([tv.ToTensor(), tv.Normalize(CLIP_MEAN, CLIP_STD)])
    ref = pre(Image.fromarray(_ramp()))[:, 0, :]
    assert torch.equal(norm_table().view(torch.int32), ref.contiguous().view(torch.int32))


def test_oracle_preprocess_and_tile_match_reference_fixture(golden_dir):
    """hd_preprocess_oracle.preprocess_u8 followed by hd_oracle.hd_tile reproduces the reference's preprocess + tiling block on every case,
    within the tolerance of the float32 fixture (hd_tile.npz's)."""
    g = np.load(os.path.join(golden_dir, "hd_preprocess_u8.npz"))
    for ci in range(int(g["n_cases"])):
        h, w, patch_num, hb, wb, seed = (int(v) for v in g[f"case{ci}_meta"])
        px = hpo.u8_test_image(h, w, seed)
        if seed < 0:
            for c in range(3):
                assert np.unique(px[:, :, c]).size == 256         # every byte value in every channel
        crops, ohb, owb = hdo.hd_tile(hpo.preprocess_u8(px)[None], patch_num)
        assert (ohb, owb) == (hb, wb)
        np.testing.assert_allclose(crops[:, :, ::37, ::41], g[f"case{ci}_probe"], atol=3e-6)
        ab = np.abs(crops.astype(np.float64)).sum(axis=(1, 2, 3))
        np.testing.assert_allclose(ab, g[f"case{ci}_abs"], rtol=1e-6)
        assert np.all(np.abs(crops.astype(np.float64).sum(axis=(1, 2, 3)) - g[f"case{ci}_sum"]) <= 1e-6 * ab)   # relative to the magnitude


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    p = C.c_void_p(16)          # never dereferenced: every call below is refused before any CUDA work
    bad = _lib.TP_ERR_INVALID_ARGUMENT
    assert lib.tp_hd_preprocess_batch(None, p, p, 1, p, 0, p, None) == bad
    assert lib.tp_hd_preprocess_batch(p, None, p, 1, p, 0, p, None) == bad
    assert lib.tp_hd_preprocess_batch(p, p, None, 1, p, 0, p, None) == bad
    assert lib.tp_hd_preprocess_batch(p, p, p, 1, None, 0, p, None) == bad
    assert lib.tp_hd_preprocess_batch(p, p, p, 1, p, 0, None, None) == bad
    for dt in (-1, 2, 3):
        assert lib.tp_hd_preprocess_batch(p, p, p, 1, p, dt, p, None) == bad
    assert lib.tp_hd_preprocess_batch(p, p, p, -1, p, 1, p, None) == bad
    assert lib.tp_hd_preprocess_batch(p, p, p, 1 << 40, p, 1, p, None) == bad        # more CTAs than a grid holds
    assert lib.tp_hd_preprocess_batch(p, p, p, 0, p, 1, p, None) == _lib.TP_OK         # nothing to do, nothing launched
    assert C.sizeof(_lib.TpHdU8Source) == 32


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U8_HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_hd_u8.h")


def _u8_header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(U8_HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(", text)))


def test_u8_header_binding_and_exports_agree():
    """include/tokenpacker_b200_hd_u8.h only adds: its entry points are exported, bound by _lib.HD_U8_SIGNATURES, and none of
    them is also declared by tokenpacker_b200.h."""
    from tokenpacker_b200 import _lib
    names = _u8_header_functions()
    assert names == ["tp_hd_preprocess_batch"]
    assert sorted(_lib.HD_U8_SIGNATURES) == names
    assert not set(names) & set(_lib.SIGNATURES)
    raw = C.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"


def test_plain_c_consumer_of_the_u8_header(tmp_path):
    """The header is C99, its entry points link from plain C, and argument validation runs without a GPU
    (tests/abi_c/abi_check_hd_u8.c)."""
    import shutil
    import subprocess
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_hd_u8")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_hd_u8.c")
    text = open(src).read()
    for name in _u8_header_functions():
        assert f"&{name}" in text, f"{name} missing from abi_check_hd_u8.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi hd_u8 ok" in r.stdout


def test_python_argument_errors_before_device_work():
    from tokenpacker_b200 import hd_preprocess_batch
    img = torch.zeros(20, 30, 3, dtype=torch.uint8)
    with pytest.raises(TypeError):
        hd_preprocess_batch([img.float()])
    with pytest.raises(ValueError):
        hd_preprocess_batch([torch.zeros(20, 30, dtype=torch.uint8)])
    with pytest.raises(ValueError):
        hd_preprocess_batch([torch.zeros(1, 20, 30, 3, dtype=torch.uint8)])
    with pytest.raises(ValueError):
        hd_preprocess_batch([torch.zeros(20, 30, 4, dtype=torch.uint8)])
    with pytest.raises(ValueError):
        hd_preprocess_batch([img], layout="CHW")                   # [20,30,3] has 20 channels as CHW
    with pytest.raises(ValueError):
        hd_preprocess_batch([img], layout="NHWC")
    with pytest.raises(ValueError):
        hd_preprocess_batch([])
    for dt in (torch.float16, torch.float64, torch.uint8):
        with pytest.raises(ValueError):
            hd_preprocess_batch([img], dtype=dt)
    with pytest.raises(RuntimeError, match="no CPU path"):
        hd_preprocess_batch([img])
    with pytest.raises(RuntimeError, match="no CPU path"):
        hd_preprocess_batch([img.permute(2, 0, 1)], layout="CHW", dtype=torch.bfloat16)
