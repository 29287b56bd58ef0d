"""The JPEG decoder's host side, no GPU: the numpy oracle against PIL on the fixture matrix and on the committed fixtures, the refusal
reasons of jpeg_unsupported, the plan's geometry against the oracle's, and the header, binding and exports agreeing."""
import ctypes as C
import io
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_fixtures as jf  # noqa: E402
from oracle import jpeg_oracle as jo  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_jpeg.h")


@pytest.mark.parametrize("large", [False, True])
def test_oracle_equals_pil_on_the_matrix(large):
    for name, data in jf.matrix():
        hdr = jo.parse(data)
        if (hdr["h"] * hdr["w"] > 400_000) == large:
            assert np.array_equal(jo.decode(data), jf.pil_decode(data)), name


def test_oracle_equals_pil_at_narrow_chroma():
    """Chroma 1 or 2 samples wide takes libjpeg's plain replication instead of fancy upsampling."""
    for h, w in [(1, 2), (2, 1), (3, 3), (5, 3), (9, 4), (4, 5), (2, 9)]:
        for sub in ("422", "420"):
            for kind in jf.KINDS:
                data = jf.encode(jf.image(h, w, kind, h * 31 + w), sub, 50)
                assert np.array_equal(jo.decode(data), jf.pil_decode(data)), (h, w, sub, kind)


def test_committed_fixtures(golden_dir):
    import hashlib
    z = np.load(os.path.join(golden_dir, "jpeg_fixtures.npz"))
    names = list(z["names"])
    assert len(names) >= 10
    for i, name in enumerate(names):
        data = z[f"file_{i}"].tobytes()
        pil = jf.pil_decode(data)
        assert hashlib.sha256(pil.tobytes()).hexdigest() == str(z["sha256"][i]), name
        assert np.array_equal(jo.decode(data), pil), name


def _save(a, mode=None, **kw):
    b = io.BytesIO()
    im = Image.fromarray(a)
    if mode:
        im = im.convert(mode)
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def test_unsupported_reasons():
    from tokenpacker_b200 import jpeg_unsupported
    a = jf.image(40, 56, "grad", 1)
    ok = _save(a)
    files = [ok, _save(a, progressive=True), _save(a, "CMYK"), ok[:60], b"\x89PNG\r\n\x1a\n" + bytes(50), b"", _save(a, "L"), ok]
    got = jpeg_unsupported(files)
    assert got[0] is None and got[6] is None and got[7] is None
    assert got[1] == "progressive JPEG"
    assert got[2] == "CMYK, YCCK or RGB colour"
    assert got[3] == "malformed or truncated header"
    assert got[4] == got[5] == "not a JPEG file"
    # Adobe transform 0 (RGB-coded colour) and RGB component ids without JFIF
    rgb = _save(a, keep_rgb=True)
    assert jo.parse(ok) and jpeg_unsupported([rgb]) == ["CMYK, YCCK or RGB colour"]
    with pytest.raises(jo.Unsupported):
        jo.parse(rgb)


def test_unsupported_sampling_and_multi_scan():
    """4:4:0 (luma 1 x 2) is refused, and a sequential file with a second scan is refused."""
    from tokenpacker_b200 import jpeg_unsupported
    data = bytearray(_save(jf.image(32, 32, "noise", 2), subsampling=0))
    sof = data.index(b"\xff\xc0")
    assert data[sof + 11] == 0x11
    data[sof + 11] = 0x12                              # component 1: H = 1, V = 2
    assert jpeg_unsupported([bytes(data)]) == ["sampling factors other than 4:4:4, 4:2:2 and 4:2:0"]
    ok = _save(jf.image(16, 16, "grad", 3))
    sos = ok.index(b"\xff\xda")
    twice = ok[:-2] + ok[sos:]                         # the scan repeated before EOI
    assert jpeg_unsupported([twice]) == ["more than one scan"]


def test_plan_geometry_against_the_oracle():
    from tokenpacker_b200 import _lib
    from tokenpacker_b200.jpeg import _buffers
    named = [x for x in jf.matrix(big=False)][::7]
    ptrs, sizes, keep = _buffers([d for _, d in named])
    b = len(ptrs)
    rows = (_lib.TpJpegImage * b)()
    tot = _lib.TpJpegTotals()
    assert _lib.lib.tp_jpeg_plan((C.c_void_p * b)(*ptrs), (C.c_int64 * b)(*sizes), b, rows, None, None, C.byref(tot)) == 0
    blocks = pixels = 0
    for (name, data), im in zip(named, rows):
        hdr = jo.parse(data)
        assert (im.h, im.w, im.ncomp, im.mcus_x, im.mcus_y) == (hdr["h"], hdr["w"], len(hdr["comps"]), hdr["mcus_x"], hdr["mcus_y"]), name
        assert im.scan_bytes == len(hdr["scan_bytes"]), name
        assert im.n_segments == len(jo.unstuff(hdr["scan_bytes"])), name
        assert im.block0 == blocks and im.pixel0 == pixels
        blocks += im.n_blocks
        pixels += im.h * im.w
    assert (tot.blocks, tot.pixels, tot.output_bytes) == (blocks, pixels, 3 * pixels)
    assert _lib.lib.tp_jpeg_workspace_bytes(rows, b) == tot.workspace_bytes


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(", text)))


def test_jpeg_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    names = _header_functions()
    assert names == ["tp_jpeg_decode_batch", "tp_jpeg_plan", "tp_jpeg_reason_string", "tp_jpeg_workspace_bytes"]
    assert sorted(_lib.JPEG_SIGNATURES) == names
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name in names:
        params = re.search(rf"\b{name}\s*\(([^;]*?)\)\s*;", text, flags=re.S).group(1)
        assert len(params.split(",")) == len(_lib.JPEG_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"
    sizes = {"TpJpegImage": 168, "TpJpegHuff": 1424, "TpJpegTables": 8928, "TpJpegTotals": 40, "TpJpegStatus": 16}
    for cls, n in sizes.items():
        assert C.sizeof(getattr(_lib, cls)) == n, cls


def test_plain_c_consumer_of_the_jpeg_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_jpeg")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_jpeg.c")
    text = open(src).read()
    for name in _header_functions():
        assert f"&{name}" in text, f"{name} missing from abi_check_jpeg.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    f = tmp_path / "x.jpg"
    f.write_bytes(_save(jf.image(16, 24, "noise", 4), subsampling=2, restart_marker_blocks=1))
    r = subprocess.run([exe, str(f)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi jpeg ok" in r.stdout


def test_python_argument_errors_before_device_work():
    from tokenpacker_b200 import decode_jpeg_batch, jpeg_unsupported
    with pytest.raises(TypeError):
        jpeg_unsupported([np.zeros(10, np.float32)])
    with pytest.raises(TypeError):
        jpeg_unsupported(["a string"])
    with pytest.raises(ValueError):
        decode_jpeg_batch([])
    with pytest.raises(RuntimeError, match="no CPU path"):
        decode_jpeg_batch([b"\xff\xd8"], device="cpu")


def test_jfif_and_adobe_follow_libjpeg():
    """JFIF means YCbCr whatever the Adobe transform; without JFIF, transform 0 means RGB (refused) and any other YCbCr."""
    from tokenpacker_b200 import jpeg_unsupported
    base = jf.encode(jf.image(45, 61, "sat", 13), "420", 85)
    files = [jf.with_adobe(base, t) for t in (0, 1, 2)]
    assert jpeg_unsupported(files) == [None, None, None]
    for f in files:
        assert np.array_equal(jo.decode(f), jf.pil_decode(f))
    end = 4 + ((base[4] << 8) | base[5])
    no_jfif = [base[:2] + f[end:] for f in files]           # the APP0 segment removed
    assert jpeg_unsupported(no_jfif) == ["CMYK, YCCK or RGB colour", None, None]


def test_scan_order_other_than_the_frame_has_its_own_reason():
    from tokenpacker_b200 import jpeg_unsupported
    data = bytearray(jf.encode(jf.image(16, 16, "grad", 5), "444", 75))
    sos = data.index(b"\xff\xda")
    comps = [bytes(data[sos + 5 + 2 * k:sos + 7 + 2 * k]) for k in range(3)]
    data[sos + 5:sos + 11] = comps[1] + comps[0] + comps[2]
    assert jpeg_unsupported([bytes(data)]) == ["scan components not in frame order"]


def test_matrix_has_16_bit_quantisation_tables():
    names = [(n, d) for n, d in jf.matrix(big=False) if "dqt16" in n]
    assert len(names) >= 9
    for n, d in names:
        i = d.index(b"\xff\xdb")
        assert d[i + 4] >> 4 == 1, n                          # Pq = 1
