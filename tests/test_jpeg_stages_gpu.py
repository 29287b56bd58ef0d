"""The JPEG decoder stage by stage against oracle/jpeg_oracle.py, bit for bit (tests/csrc/tp_jpeg_hooks.cu runs the launches up to one
stage): the int16 coefficients after Huffman decoding and DC prediction, the component planes after the IDCT, the final bytes; and
each stage writes only its own regions of the workspace and the output."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_fixtures as jf  # noqa: E402
from oracle import jpeg_oracle as jo  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_jpeg_hooks.so")
SENTINEL = 0xA5

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def hooks():
    h = C.CDLL(HOOKS)
    h.tpj_decode_stages.restype = C.c_int
    h.tpj_decode_stages.argtypes = [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p]
    h.tpj_subsequence_record_bytes.restype = C.c_int
    return h


def _files():
    keep = ("1x1-", "7x13-", "17x33-", "333x517-")
    return [(n, d) for n, d in jf.matrix(big=False) if n.startswith(keep)][::3]


def _run(hooks, files, stage):
    from tokenpacker_b200.jpeg import _plan_upload_launch

    def launch(out, ws, args, stream):
        out.fill_(SENTINEL)
        ws.fill_(SENTINEL)
        assert hooks.tpj_decode_stages(*args, stage, stream) == 0
    rows, out, ws, status = _plan_upload_launch(files, "cuda", launch)
    torch.cuda.synchronize()
    return out.cpu().numpy(), ws.cpu().numpy(), status.cpu().numpy(), rows


def _regions(rows, status, sub_bytes, stage):
    """[start, end) byte ranges of the workspace stages 1 .. stage write."""
    r = []
    for i, im in enumerate(rows):
        if stage >= 1:
            unst = int(im.scan_bytes)                          # an upper bound of the unstuffed bytes
            r += [(im.unstuffed_offset, im.unstuffed_offset + unst), (im.seg_offset, im.seg_offset + 8 * (im.n_segments + 1)),
                  (im.sub_offset, im.sub_offset + sub_bytes * int(status[i, 2]))]
        if stage >= 2:
            r.append((im.coef_offset, im.coef_offset + 128 * im.n_blocks))
        if stage >= 3:
            r.append((im.plane_offset, im.plane_offset + 64 * im.n_blocks))
    return r


@pytest.mark.parametrize("stage", [1, 2, 3, 4])
def test_stage_against_oracle_and_regions(hooks, stage):
    named = _files()
    files = [d for _, d in named]
    out, ws, status, rows = _run(hooks, files, stage)
    assert (status[:, 0] == 0).all()
    touched = np.zeros(ws.size, bool)
    for a, b in _regions(rows, status, hooks.tpj_subsequence_record_bytes(), stage):
        touched[a:b] = True
    assert (ws[~touched] == SENTINEL).all(), "a stage wrote outside its regions"
    if stage < 4:
        assert (out == SENTINEL).all()
    for (name, data), im in zip(named, rows):
        hdr = jo.parse(data)
        if stage == 1:
            segs = jo.unstuff(hdr["scan_bytes"])
            starts = ws[im.seg_offset:im.seg_offset + 8 * (im.n_segments + 1)].view(np.int64)
            assert starts[0] == 0 and len(segs) >= im.n_segments, name
            for k in range(im.n_segments):
                got = ws[im.unstuffed_offset + starts[k]:im.unstuffed_offset + starts[k + 1]].tobytes()
                assert got == segs[k], (name, k)
            continue
        coefs = jo.coefficients(hdr)
        off = im.coef_offset
        planes = jo.planes(hdr, coefs) if stage >= 3 else None
        poff = im.plane_offset
        for c, ref in enumerate(coefs):
            n = ref.shape[0] * ref.shape[1]
            got = ws[off:off + n * 128].view(np.int16).reshape(ref.shape)
            assert np.array_equal(got, ref), (name, "coefficients", c)
            off += n * 128
            if planes is not None:
                p = planes[c]
                gotp = ws[poff:poff + p.size].reshape(p.shape)
                assert np.array_equal(gotp, p), (name, "plane", c)
                poff += p.size
        if stage == 4:
            got = out[im.out_offset:im.out_offset + im.h * im.w * 3].reshape(im.h, im.w, 3)
            assert np.array_equal(got, jo.rgb(hdr, planes)), name
            assert np.array_equal(got, jf.pil_decode(data)), name
