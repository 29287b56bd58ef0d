"""The PNG decoder's host side, no GPU: the oracle against zlib and PIL on the matrix and the committed fixtures, each PIL rule the
decoder restates, the refusal reasons of png_unsupported, the plan's geometry and workspace bound, and the header, binding and exports
agreeing (with a plain-C consumer)."""
import ctypes as C
import hashlib
import io
import os
import re
import shutil
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_fixtures as pf  # noqa: E402
import png_writer as pw  # noqa: E402
from oracle import png_oracle as po  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_png.h")


def test_oracle_equals_zlib_and_pil_on_the_matrix():
    for name, data in pf.matrix():
        hdr = po.parse(data)
        if hdr["raw_bytes"] > 120_000:
            continue
        raw, blocks, src = po.inflate(hdr["stream"])
        assert raw == zlib.decompress(hdr["stream"]), name
        assert blocks[0]["start_bit"] == 16 and blocks[-1]["final"] == 1 and sum(b["out_bytes"] for b in blocks) == len(raw)
        assert (src <= np.arange(len(src))).all()
        assert np.array_equal(po.decode(data), pf.pil_decode(data)), name


def test_committed_fixtures(golden_dir):
    z = np.load(os.path.join(golden_dir, "png_fixtures.npz"))
    assert len(z["names"]) >= 10
    for i, name in enumerate(z["names"]):
        data = z[f"file_{i}"].tobytes()
        pil = pf.pil_decode(data)
        assert hashlib.sha256(pil.tobytes()).hexdigest() == str(z["sha256"][i]), name
        assert np.array_equal(po.decode(data), pil), name


def _png(w, h, depth, ct, raw, extra=b"", palette=b""):
    return pw.png(w, h, depth, ct, zlib.compress(raw), palette=palette, extra=extra)


def test_pil_rules_the_oracle_restates():
    dec = pf.pil_decode
    # 2- and 4-bit gray scaled by 85 and 17; 1-bit gray is mode '1', 0 / 255
    f = _png(4, 1, 2, 0, b"\0" + bytes([0b00011011]))
    assert dec(f)[0, :, 0].tolist() == [0, 85, 170, 255] and np.array_equal(po.decode(f), dec(f))
    f = _png(4, 1, 4, 0, b"\0" + bytes([0x0F, 0x7A]))
    assert dec(f)[0, :, 0].tolist() == [0, 255, 119, 170] and np.array_equal(po.decode(f), dec(f))
    f = _png(4, 1, 1, 0, b"\0" + bytes([0b10100000]))
    assert Image.open(io.BytesIO(f)).mode == "1" and dec(f)[0, :, 0].tolist() == [255, 0, 255, 0]
    assert np.array_equal(po.decode(f), dec(f))
    # a palette index past PLTE is black; tRNS and alpha are dropped
    pal = bytes([10, 20, 30, 40, 50, 60])
    f = _png(2, 1, 8, 3, b"\0\0\5", palette=pal)
    assert dec(f).tolist() == [[[10, 20, 30], [0, 0, 0]]] and np.array_equal(po.decode(f), dec(f))
    f = pw.png(2, 1, 8, 3, zlib.compress(b"\0\0\1"), palette=pal)
    f2 = f[:f.index(b"IDAT") - 4] + pw.chunk(b"tRNS", b"\0") + f[f.index(b"IDAT") - 4:]
    assert dec(f2).tolist() == [[[10, 20, 30], [40, 50, 60]]] and np.array_equal(po.decode(f2), dec(f2))
    f = _png(1, 1, 8, 6, b"\0" + bytes([1, 2, 3, 0]))
    assert dec(f).tolist() == [[[1, 2, 3]]] and np.array_equal(po.decode(f), dec(f))
    f = _png(1, 1, 8, 4, b"\0" + bytes([77, 9]), extra=pw.chunk(b"gAMA", struct.pack(">I", 45455)) + pw.chunk(b"sRGB", b"\0"))
    assert dec(f).tolist() == [[[77, 77, 77]]] and np.array_equal(po.decode(f), dec(f))
    # IDAT CRCs are not checked; a bad Adler-32 and a filter type above 4 raise
    f = _png(1, 1, 8, 2, b"\0\1\2\3")
    k = f.index(b"IEND") - 8
    assert dec(f[:k] + bytes([f[k] ^ 1]) + f[k + 1:]).tolist() == [[[1, 2, 3]]]
    z = zlib.compress(b"\0\1\2\3")
    with pytest.raises(OSError):
        dec(pw.png(1, 1, 8, 2, z[:-1] + bytes([z[-1] ^ 1])))
    with pytest.raises(po.Corrupt):
        po.inflate(z[:-1] + bytes([z[-1] ^ 1]))
    with pytest.raises(OSError):
        dec(_png(1, 1, 8, 2, b"\5\1\2\3"))
    with pytest.raises(po.Corrupt):
        po.decode(_png(1, 1, 8, 2, b"\5\1\2\3"))
    # data past the last row is ignored, missing rows are zeros: PIL does not raise (the decoder reports a status)
    assert dec(_png(1, 1, 8, 2, b"\0\1\2\3" + b"\0" * 50)).tolist() == [[[1, 2, 3]]]
    assert dec(_png(1, 2, 8, 2, b"\0\1\2\3")).tolist() == [[[1, 2, 3]], [[0, 0, 0]]]
    with pytest.raises(po.Corrupt):
        po.decode(_png(1, 2, 8, 2, b"\0\1\2\3"))


def test_unsupported_reasons():
    from tokenpacker_b200 import png_unsupported
    ok = _png(2, 2, 8, 2, b"\0" + bytes(6) + b"\0" + bytes(6))
    bad_crc = bytearray(ok)
    bad_crc[8 + 8 + 13] ^= 1                                    # IHDR's CRC
    pal = _png(2, 1, 8, 3, b"\0\0\1", palette=bytes(6))
    bad_plte = bytearray(pal)
    k = pal.index(b"PLTE")
    bad_plte[k + 4 + 6] ^= 1
    big = pw.png(20000, 10000, 8, 0, zlib.compress(b""))
    big_ok = pw.png(89478485, 2, 1, 0, zlib.compress(b""))     # exactly 2 * MAX_IMAGE_PIXELS: PIL only warns
    acTL = ok[:33] + pw.chunk(b"acTL", bytes(8)) + ok[33:]
    zdict = pw.png(2, 2, 8, 2, bytes([0x78, 0xBB, 0, 0, 0, 1]) + b"\x03\x00" + bytes(8))
    method = pw.png(2, 2, 8, 2, bytes([0x79, (31 - (0x79 << 8) % 31) % 31]) + bytes(8))          # CM = 9
    short_trns = ok[:33] + pw.chunk(b"tRNS", b"\0\1") + ok[33:]
    files = [ok, b"GIF89a" + bytes(20), b"", ok[:40], bytes(bad_crc), bytes(bad_plte), pw.png(1, 1, 16, 0, zlib.compress(b"\0\0\0")),
             pw.png(1, 1, 8, 2, zlib.compress(b"\0\1\2\3"), interlace=1), acTL, zdict, big, big_ok, short_trns, method]
    got = png_unsupported(files)
    assert got[0] is None and got[11] is None
    assert got[1] == got[2] == "not a PNG file"
    assert got[3] == "malformed or truncated chunks"
    assert got[4] == got[5] == "bad chunk CRC"
    assert got[6] == "16-bit samples"
    assert got[7] == "interlaced PNG"
    assert got[8] == "animated PNG"
    assert got[9] == "unsupported zlib header"
    assert got[10] == "image too large"
    assert got[12] == "ancillary chunk PIL rejects"
    assert got[13] == "unsupported zlib header"
    # PIL raises on each refused file it is asked to decode (the 16-bit and interlaced files it reads, and big_ok is in scope)
    for i in (1, 2, 3, 4, 5, 10, 12):
        with pytest.raises(Exception):
            pf.pil_decode(files[i])


def test_plan_geometry_and_workspace_bound():
    from tokenpacker_b200 import _lib
    files = [d for _, d in pf.matrix()]
    b = len(files)
    bufs = [C.create_string_buffer(f, len(f)) for f in files]
    ptrs = (C.c_void_p * b)(*[C.addressof(x) for x in bufs])
    sizes = (C.c_int64 * b)(*[len(f) for f in files])
    images = (_lib.TpPngImage * b)()
    pal = (C.c_uint8 * (768 * b))()
    staged = (C.c_uint8 * (sum((len(f) + 15) // 16 * 16 for f in files) + 16))()
    tot = _lib.TpPngTotals()
    assert _lib.lib.tp_png_plan(ptrs, sizes, b, images, pal, staged, C.byref(tot)) == 0
    out = ws = 0
    for i, f in enumerate(files):
        im, hdr = images[i], po.parse(f)
        assert (im.h, im.w, im.depth, im.color_type, im.row_bytes, im.filter_bpp, im.raw_bytes) == (
            hdr["h"], hdr["w"], hdr["depth"], hdr["color_type"], hdr["row_bytes"], hdr["filter_bpp"], hdr["raw_bytes"])
        assert bytes(staged[im.stream_offset:im.stream_offset + im.stream_bytes]) == hdr["stream"]
        if im.color_type == 3:
            p = hdr["palette"]
            assert bytes(pal[768 * i:768 * i + len(p)]) == p and im.palette_entries == len(p) // 3
        assert im.out_offset == out
        out += im.h * im.w * 3
        s, r = im.stream_bytes, im.raw_bytes
        assert im.block_capacity == 8 * s // 10 + 2
        assert im.mask_offset >= ws and im.mask_offset % 16 == 0
        need = im.src_offset + 4 * r - im.mask_offset
        assert need <= 19.5 * s + 5 * r + 200
        assert im.spec_offset >= im.mask_offset + 4 * ((8 * s + 31) // 32)
        assert im.block_offset >= im.spec_offset + 20 * 4 * ((8 * s + 255) // 256)
        assert im.raw_offset >= im.block_offset + 20 * im.block_capacity and im.src_offset >= im.raw_offset + r
        ws = im.src_offset + 4 * r
    assert tot.output_bytes == out and tot.workspace_bytes == _lib.lib.tp_png_workspace_bytes(images, b) == ws
    assert tot.max_raw_bytes == max(po.parse(f)["raw_bytes"] for f in files)


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    import tokenpacker_b200 as tp
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = sorted(set(re.findall(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(", text)))
    assert names == sorted(_lib.PNG_SIGNATURES)
    raw = C.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n)
    assert "decode_png_batch" in tp.__all__ and "png_unsupported" in tp.__all__
    for code in range(10):
        assert _lib.lib.tp_png_reason_string(code) is not None
    assert _lib.lib.tp_png_reason_string(10) is None
    assert C.sizeof(_lib.TpPngImage) == 136 and C.sizeof(_lib.TpPngBlock) == 20 and C.sizeof(_lib.TpPngStatus) == 16
    for name, value in re.findall(r"(TP_PNG_STATUS_\w+) = (\d+)", text):
        assert getattr(_lib, name) == int(value)


def test_plain_c_consumer_of_the_png_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_png")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_png.c")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    f = tmp_path / "a.png"
    f.write_bytes(pw.png(24, 16, 8, 2, zlib.compress(bytes(16 * (24 * 3 + 1)))))
    r = subprocess.run([exe, str(f)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi png ok" in r.stdout


def test_limits_fixture_reaches_the_window_edge():
    """The hand-written limits stream holds matches of length 258 at distance 32768 and of length 3 and 258 at distance 1, a
    32768-distance match crossing a row boundary, and sources in the block before their own."""
    f = pf.limits_file()
    hdr = po.parse(f)
    raw, blocks, src = po.inflate(hdr["stream"])
    m = [x for b in blocks for x in b["matches"]]
    assert {(258, 32768), (258, 1), (3, 1)} <= {(n, d) for _, n, d in m}
    assert int((np.arange(len(src)) - src).max()) == 32768
    rb = hdr["row_bytes"] + 1
    assert any(p // rb != (p + n - 1) // rb for p, n, d in m if d == 32768)
    assert len(blocks) == 2 and any(p - d < blocks[1]["out_offset"] for p, n, d in blocks[1]["matches"])
    assert np.array_equal(po.decode(f), pf.pil_decode(f))
    small = pf.corrupt_set()[-1][0]                       # a distance one past the 256-byte window its zlib header declares
    with pytest.raises(po.Corrupt, match="too far back"):
        po.decode(small)


def test_idat_crcs_are_not_checked():
    """PIL reads no IDAT CRC, so a bad one on the first or a later IDAT is no reason to refuse; a bad CRC on a chunk before the
    first IDAT is."""
    from tokenpacker_b200 import png_unsupported
    z = zlib.compress(b"\0\1\2\3\0\4\5\6")
    f = pw.png(1, 2, 8, 2, z, idat_sizes=[3, 100])
    starts, i = [], 8
    while i + 12 <= len(f):
        starts.append(i)
        i += 12 + struct.unpack(">I", f[i:i + 4])[0]
    idats = [k for k in starts if f[k + 4:k + 8] == b"IDAT"]
    assert len(idats) == 2
    files = []
    for k in idats:
        end = k + 12 + struct.unpack(">I", f[k:k + 4])[0]
        b = bytearray(f)
        b[end - 1] ^= 1
        files.append(bytes(b))
        assert pf.pil_decode(files[-1]).tolist() == [[[1, 2, 3]], [[4, 5, 6]]]
    gama = f[:33] + pw.chunk(b"gAMA", struct.pack(">I", 45455)) + f[33:]
    bad = bytearray(gama)
    bad[33 + 8 + 4] ^= 1                                  # the gAMA chunk's CRC
    with pytest.raises(OSError):                          # PIL: cannot identify image file (broken PNG file)
        pf.pil_decode(bytes(bad))
    assert png_unsupported(files + [gama, bytes(bad)]) == [None, None, None, "bad chunk CRC"]
