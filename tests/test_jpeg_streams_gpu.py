"""The JPEG decoder on streams Pillow never writes (tests/jpeg_streams.py), through the stage hook (tests/csrc/tp_jpeg_hooks.cu):
after stage 2 the int16 coefficients equal the writer's bit for bit, after stage 4 the bytes equal PIL's with status 0, and on
every crafted stream, valid or not, either the status is 0 and the bytes are PIL's or the file is refused or reported.  Coverage
is read back: every subsequence-boundary offset, a swallowed last subsequence in the workspace's records, and the chunk-straddling
bytes in the staged scan.  A camera-size batch takes the output and coefficient regions past 2^31 bytes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_fixtures as jf  # noqa: E402
import jpeg_streams as js  # noqa: E402
import jpeg_writer as jw  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_jpeg_hooks.so")

pytestmark = pytest.mark.gpu

# JpegSub (tp_jpeg.cuh): start, end, seg_end, entry_pos, exit_pos (int64); seg, entry_bk, exit_bk, started, bad, first (int32)
SUB = np.dtype([("start", "<i8"), ("end", "<i8"), ("seg_end", "<i8"), ("entry_pos", "<i8"), ("exit_pos", "<i8"), ("seg", "<i4"),
                ("entry_bk", "<i4"), ("exit_bk", "<i4"), ("started", "<i4"), ("bad", "<i4"), ("first", "<i4")])


@pytest.fixture(scope="module")
def hooks():
    h = C.CDLL(HOOKS)
    h.tpj_decode_stages.restype = C.c_int
    h.tpj_decode_stages.argtypes = [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p]
    h.tpj_subsequence_record_bytes.restype = C.c_int
    assert h.tpj_subsequence_record_bytes() == SUB.itemsize
    return h


@pytest.fixture(scope="module")
def valid():
    return js.valid_streams()


def _run(hooks, files, stage):
    """(plan rows, output bytes, workspace, status) on the device after the launches up to `stage`."""
    from tokenpacker_b200.jpeg import _plan_upload_launch

    def launch(out, ws, args, stream):
        assert hooks.tpj_decode_stages(*args, stage, stream) == 0
    rows, out, ws, status = _plan_upload_launch(files, "cuda", launch)
    torch.cuda.synchronize()
    return rows, out, ws, status.cpu().numpy()


def _coefs(ws, im, shapes):
    off, out = im.coef_offset, []
    for by, bx in shapes:
        n = by * bx * 128
        out.append(ws[off:off + n].cpu().numpy().view(np.int16).reshape(by, bx, 64))
        off += n
    return out


def _staged(files):
    """The host plan's staged scans and rows: the bytes the unstuff kernel reads."""
    from tokenpacker_b200 import _lib
    from tokenpacker_b200.jpeg import _buffers
    ptrs, sizes, keep = _buffers(files)
    b = len(ptrs)
    rows = (_lib.TpJpegImage * b)()
    tables = (_lib.TpJpegTables * b)()
    staged = np.zeros(sum(sizes) + 16 * b, np.uint8)
    tot = _lib.TpJpegTotals()
    assert _lib.lib.tp_jpeg_plan((C.c_void_p * b)(*ptrs), (C.c_int64 * b)(*sizes), b, rows, tables, staged.ctypes.data,
                                 C.byref(tot)) == 0
    return rows, staged


def test_stage2_coefficients_equal_the_writer(hooks, valid):
    files = [d for _, d, _ in valid]
    rows, _, ws, status = _run(hooks, files, 2)
    assert (status[:, 0] == 0).all(), status[:, 0].tolist()
    for (name, _, log), im in zip(valid, rows):
        got = _coefs(ws, im, [c.shape[:2] for c in log.coefs])
        for c, (g, want) in enumerate(zip(got, log.coefs)):
            assert np.array_equal(g, want), (name, c, int((g != want).sum()))
    # the boundary family: every offset d in 1 .. 31, and records whose predecessor's last code swallowed them whole
    i = next(k for k, (n, _, _) in enumerate(valid) if n == "boundaries-gray-dri1")
    assert js.boundary_offsets(valid[i][2]) >= set(range(1, 32))
    im = rows[i]
    subs = ws[im.sub_offset:im.sub_offset + SUB.itemsize * int(status[i, 2])].cpu().numpy().view(SUB)
    swallowed = subs[subs["entry_pos"] >= subs["end"]]
    assert len(swallowed) >= 1
    # such a record is always its interval's last, and the code that swallowed it ended on the interval's last bit
    assert (swallowed["entry_pos"] == swallowed["end"]).all() and (swallowed["end"] == swallowed["seg_end"]).all()
    assert (subs["end"] - subs["start"] <= js.SUB_BITS).all() and int(status[i, 1]) >= 1


def test_the_chunk_straddling_bytes_are_in_the_staged_scan(valid):
    named = [(n, d, log) for n, d, log in valid if n.startswith(("dense-ff00", "rst-across-chunk"))]
    rows, staged = _staged([d for _, d, _ in named])
    for (name, d, log), im in zip(named, rows):
        scan = staged[im.scan_offset:im.scan_offset + im.scan_bytes].tobytes()
        assert scan == d[log.scan_begin:log.scan_begin + im.scan_bytes], name
        second = scan[js.CHUNK]
        assert scan[js.CHUNK - 1] == 0xFF and (second == 0x00 if name.startswith("dense") else 0xD0 <= second <= 0xD7), name
        pairs = [p for p in range(7, len(scan) - 1, 8) if scan[p] == 0xFF and p % js.CHUNK != js.CHUNK - 1]
        assert any(scan[p + 1] == 0x00 for p in pairs) if name.startswith("dense") else any(0xD0 <= scan[p + 1] <= 0xD7 for p in pairs)


def test_stage4_bytes_equal_pil(hooks, valid):
    files = [d for _, d, _ in valid]
    rows, out, _, status = _run(hooks, files, 4)
    assert (status[:, 0] == 0).all(), status[:, 0].tolist()
    for (name, d, _), im in zip(valid, rows):
        got = out[im.out_offset:im.out_offset + im.h * im.w * 3].cpu().numpy().reshape(im.h, im.w, 3)
        assert np.array_equal(got, jf.pil_decode(d)), name


def _pil_or_none(d):
    try:
        return jf.pil_decode(d)
    except (OSError, SyntaxError, ValueError):
        return None


def test_contract_on_every_crafted_stream(valid):
    """Status 0 means PIL's bytes; anything PIL raises on is refused or reported; and the crafted breakages get their status."""
    from tokenpacker_b200 import decode_jpeg_batch, jpeg_unsupported
    crafted = js.contract_streams()
    named = [(n, d, "ok") for n, d, _ in valid] + [(n, d, e) for n, d, _, e in crafted]
    # a cut inside the dense stream's last block and a cut mid-scan: PIL raises on both
    dense = next(d for n, d, _ in valid if n.startswith("dense"))
    named += [("dense-cut", dense[:len(dense) - 40], None), ("dense-half", dense[:len(dense) // 2], None)]
    files = [d for _, d, _ in named]
    refused = jpeg_unsupported(files)
    keep = [k for k, r in enumerate(refused) if r is None]
    assert len(keep) == len(named)
    imgs, status = decode_jpeg_batch(files, return_status=True)
    st = status[:, 0].cpu().numpy()
    want = {"ok": 0, "restart": 2, "entropy": 1}
    for k, (name, d, exp) in enumerate(named):
        pil = _pil_or_none(d)
        if st[k] == 0:
            assert pil is not None, name
            assert np.array_equal(imgs[k].cpu().numpy(), pil), name
        if exp is not None:
            assert st[k] == want[exp], (name, int(st[k]))
        else:
            assert pil is None and st[k] != 0, name


def test_the_runs_past_63_agree_with_the_plain_coding(hooks):
    """The stage-2 coefficients of a run past 63 are the ones libjpeg keeps: the value at natural index 63."""
    crafted = {n: d for n, d, _, _ in js.contract_streams()}
    rows, _, ws, status = _run(hooks, [crafted["ac-run-past-63"], crafted["ac-zrl-past-63"]], 2)
    assert (status[:, 0] == 0).all()
    run, zrl = _coefs(ws, rows[0], [(2, 3)])[0], _coefs(ws, rows[1], [(2, 3)])[0]
    assert run[0, 1, 63] == -2 and run[0, 1, jw.ZIGZAG[59]] == 5 and np.count_nonzero(run[0, 1, 1:]) == 3
    assert zrl[0, 1, jw.ZIGZAG[55]] == 3 and np.count_nonzero(zrl[0, 1, 1:]) == 2


@pytest.fixture(scope="module")
def camera():
    return {sub: js.camera_stream(sub) for sub in ("422", "420")}


def test_camera_size_files(hooks, camera):
    for sub, (name, d, log) in camera.items():
        rows, out, ws, status = _run(hooks, [d], 4)
        assert status[0, 0] == 0 and status[0, 2] > 1000, (name, status[0].tolist())
        for c, (g, want) in enumerate(zip(_coefs(ws, rows[0], [x.shape[:2] for x in log.coefs]), log.coefs)):
            assert np.array_equal(g, want), (name, c)
        im = rows[0]
        got = out[im.out_offset:im.out_offset + im.h * im.w * 3].cpu().numpy().reshape(im.h, im.w, 3)
        assert np.array_equal(got, jf.pil_decode(d)), name
        del out, ws
        torch.cuda.empty_cache()


def test_batch_past_2_31_bytes(hooks, camera):
    """One batch of the 4:2:0 camera file repeated until the output and the coefficient regions each pass 2^31 bytes: the last file's
    coefficients and bytes are still exact."""
    name, d, log = camera["420"]
    per = 3024 * 4032 * 3
    n = (1 << 31) // per + 1
    rows, out, ws, status = _run(hooks, [d] * n, 4)
    last = rows[n - 1]
    assert last.out_offset + per > 1 << 31 and last.coef_offset - rows[0].coef_offset + last.n_blocks * 128 > 1 << 31
    assert (status[:, 0] == 0).all()
    for c, (g, want) in enumerate(zip(_coefs(ws, last, [x.shape[:2] for x in log.coefs]), log.coefs)):
        assert np.array_equal(g, want), c
    ref = torch.from_numpy(jf.pil_decode(d).reshape(-1)).cuda()
    for im in (rows[0], rows[n // 2], last):
        assert torch.equal(out[im.out_offset:im.out_offset + per], ref), im.out_offset
    first = out[:per]
    for im in rows:
        assert torch.equal(out[im.out_offset:im.out_offset + per], first)
    print(f"batch of {n}: output {out.numel() / 2**30:.2f} GiB, workspace {ws.numel() / 2**30:.2f} GiB, "
          f"peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    del out, ws
    torch.cuda.empty_cache()
