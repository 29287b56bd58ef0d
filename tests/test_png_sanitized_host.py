"""The PNG decoder's scalar core (tokenpacker_b200/csrc/tp_png.cuh), which every GPU kernel of the decoder calls, compiled with
g++ -fsanitize=address,undefined into tests/csrc/tp_png_cpu_driver.cpp and run stage by stage over the fixture matrix, the
hand-written streams and seeded corruptions of them: bit flips, truncation at every chunk, block and row boundary, spliced IDAT
chunks, the file cut at every chunk boundary.  Each output must equal zlib's, the oracle's and PIL's, or carry a status or a refusal,
and the sanitisers must stay silent."""
import os
import random
import shutil
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_fixtures as pf  # noqa: E402
from oracle import png_oracle as po  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    d = tmp_path_factory.mktemp("png_driver")
    exe = str(d / "tp_png_cpu_driver")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-Wall", "-Wextra",
                    "-Werror", os.path.join(ROOT, "tests", "csrc", "tp_png_cpu_driver.cpp"), "-o", exe], check=True, capture_output=True,
                   text=True)
    return exe, d


def run(driver, files):
    """(reason, status, blocks, serial, candidates, inflated bytes or None, rgb or None) per file."""
    exe, d = driver
    paths = []
    for i, f in enumerate(files):
        p = str(d / f"in{i}.png")
        with open(p, "wb") as fh:
            fh.write(f)
        paths.append(p)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1")
    r = subprocess.run([exe] + paths, capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "Sanitizer" not in r.stderr, r.stderr[-3000:]
    out = []
    for p in paths:
        b = open(p + ".out", "rb").read()
        head = struct.unpack("<5i", b[:20])
        n = struct.unpack("<q", b[20:28])[0]
        body = b[28:]
        out.append(head + ((body[:n], body[n:]) if body else (None, None)))
    return out


def check(files, results, require_ok=False):
    for f, (reason, status, blocks, serial, cands, inflated, rgb) in zip(files, results):
        if reason != 0:
            continue
        hdr = po.parse(f)
        if status != 0:
            assert not require_ok, status
            continue
        assert inflated == zlib.decompress(hdr["stream"])          # zlib raises on every stream the decoder must report
        ref = po.convert(po.unfilter(inflated, hdr["h"], hdr["row_bytes"], hdr["filter_bpp"]), hdr)
        assert np.array_equal(np.frombuffer(rgb, np.uint8).reshape(hdr["h"], hdr["w"], 3), ref)
        assert np.array_equal(ref, pf.pil_decode(f))
        assert 1 <= blocks and serial <= blocks and cands >= 1


def test_matrix_under_sanitizers(driver):
    files = [d for _, d in pf.matrix()]
    res = run(driver, files)
    assert all(r[0] == 0 for r in res)
    check(files, res, require_ok=True)


def test_fixed_only_stream_is_all_fallbacks(driver):
    (f,) = [d for n, d in pf.hand_written() if n == "fixed-only"]
    (r,) = run(driver, [f])
    assert r[1] == 0 and r[3] == r[2] - 1      # every block but the first (always speculated) decoded by the chain itself


def _row_cuts(s, raw_bytes, row_bytes):
    """The stream offsets at which the inflated data first reaches each row's start: zlib fed one byte at a time."""
    d, got, cuts = zlib.decompressobj(), 0, []
    starts = iter(range(0, raw_bytes, row_bytes + 1))
    want = next(starts, None)
    for c in range(len(s)):
        got += len(d.decompress(s[c:c + 1]))
        while want is not None and got >= want:
            cuts.append(c + 1)
            want = next(starts, None)
    return cuts


def _chunk_starts(f):
    i, out = 8, []
    while i + 12 <= len(f):
        out.append(i)
        i += 12 + struct.unpack(">I", f[i:i + 4])[0]
    return out


def _corruptions(f, rng):
    hdr = po.parse(f)
    s = hdr["stream"]
    out = []
    idat = f.index(b"IDAT") + 4
    for _ in range(12):                                           # bit flips inside the image data
        b = bytearray(f)
        k = idat + rng.randrange(len(s) - 1)
        b[k] ^= 1 << rng.randrange(8)
        out.append(bytes(b))
    _, blocks, _ = po.inflate(s)
    cuts = {b["start_bit"] // 8 for b in blocks} | {(b["end_bit"] + 7) // 8 for b in blocks} | {2, len(s) - 4, len(s) - 1}
    cuts |= set(_row_cuts(s, hdr["raw_bytes"], hdr["row_bytes"]))
    for c in sorted(cuts):                                        # streams truncated at block and row boundaries, in whole chunks
        if 2 <= c < len(s):
            out.append(_rewrap(f, s[:c]))
    multi = _rewrap(f, s)
    for k in _chunk_starts(multi)[1:]:                            # the file truncated at every chunk boundary, and inside a header
        out += [multi[:k], multi[:k + 6]]
    idats = [k for k in _chunk_starts(multi) if multi[k + 4:k + 8] == b"IDAT"]
    if len(idats) > 2:                                            # spliced IDATs: the second chunk dropped, or repeated
        n1 = 12 + struct.unpack(">I", multi[idats[1]:idats[1] + 4])[0]
        out.append(multi[:idats[1]] + multi[idats[1] + n1:])
        out.append(multi[:idats[1] + n1] + multi[idats[1]:])
    out.append(_rewrap(f, s[:len(s) // 2] + s[len(s) // 3:]))     # a spliced stream
    return out


def _rewrap(f, stream):
    import png_writer as pw
    hdr = po.parse(f)
    return pw.png(hdr["w"], hdr["h"], hdr["depth"], hdr["color_type"], stream, palette=hdr["palette"] if hdr["color_type"] == 3 else b"",
                  idat_sizes=[50, 1, 4096])


def test_corruptions_are_exact_or_reported(driver):
    rng = random.Random(1234)
    files = []
    for name, f in pf.matrix():
        if name.startswith(("64x97", "level", "strategy", "stored", "fixed", "limits", "false", "chosen", "optimize")):
            files += _corruptions(f, rng)
    res = run(driver, files)
    check(files, res)
    assert sum(r[1] != 0 for r in res if r[0] == 0) > len(files) // 3


def test_gpu_corrupt_set_under_sanitizers(driver):
    """The corrupt streams the GPU tests run, each with the status it must report."""
    bad = pf.corrupt_set()
    res = run(driver, [f for f, _ in bad])
    assert [r[1] for r in res] == [st for _, st in bad]
