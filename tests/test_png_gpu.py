"""decode_png_batch on the GPU against PIL, byte for byte: the fixture matrix one file at a time and as one batch, repeated runs,
corrupt streams reported while the rest of their batch decodes, a refused file raising before any launch, the committed fixtures,
the all-fixed-block stream, each stage's output against the oracle, and decode followed by the GPU front ends against PIL decode
followed by the same calls."""
import ctypes as C
import hashlib
import os
import sys
import zlib

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_fixtures as pf  # noqa: E402
import png_writer as pw  # noqa: E402
from oracle import png_oracle as po  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def matrix():
    return pf.matrix()


def test_matrix_one_file_at_a_time(matrix):
    from tokenpacker_b200 import decode_png_batch
    for name, data in matrix:
        (got,) = decode_png_batch([data])
        assert got.dtype == torch.uint8 and got.is_cuda
        assert np.array_equal(got.cpu().numpy(), pf.pil_decode(data)), name


def test_matrix_as_one_batch_equals_per_file_and_repeats(matrix):
    from tokenpacker_b200 import decode_png_batch
    files = [d for _, d in matrix]
    forms = [f if i % 3 == 0 else (np.frombuffer(f, np.uint8) if i % 3 == 1 else torch.frombuffer(bytearray(f), dtype=torch.uint8))
             for i, f in enumerate(files)]
    first = [t.cpu().numpy() for t in decode_png_batch(forms)]
    for (name, data), got in zip(matrix, first):
        assert np.array_equal(got, pf.pil_decode(data)), name
    again, status = decode_png_batch(files, return_status=True)
    st = status.cpu().numpy()
    assert (st[:, 0] == 0).all() and (st[:, 1] >= 1).all() and (st[:, 2] <= st[:, 1]).all() and (st[:, 3] >= 1).all()
    for a, b in zip(first, again):
        assert np.array_equal(a, b.cpu().numpy())


def test_fixed_only_stream_is_all_chain_fallbacks():
    from tokenpacker_b200 import decode_png_batch
    (f,) = [d for n, d in pf.hand_written() if n == "fixed-only"]
    (img,), status = decode_png_batch([f], return_status=True)
    st = status.cpu().numpy()[0]
    assert st[0] == 0 and st[2] == st[1] - 1          # only the first block, always speculated, is not a fallback
    assert np.array_equal(img.cpu().numpy(), pf.pil_decode(f))


def test_corrupt_streams_report_status_and_others_decode(matrix):
    from tokenpacker_b200 import decode_png_batch
    good = [d for n, d in matrix if n.startswith("40x1344")][:3]
    bad = pf.corrupt_set()
    files = [good[0]] + [b for b, _ in bad] + [good[1], good[2]]
    imgs, status = decode_png_batch(files, return_status=True)
    st = status.cpu().numpy()
    for k, (_, want) in enumerate(bad):
        assert st[1 + k, 0] == want, (k, st[1 + k])
    for i, g in ((0, good[0]), (len(files) - 2, good[1]), (len(files) - 1, good[2])):
        assert st[i, 0] == 0 and np.array_equal(imgs[i].cpu().numpy(), pf.pil_decode(g))
    with pytest.raises(ValueError, match="file 1: incorrect data check"):
        decode_png_batch(files)


def test_refused_file_raises_before_any_launch(matrix):
    from tokenpacker_b200 import _lib, decode_png_batch
    ok = matrix[0][1]
    inter = pw.png(1, 1, 8, 2, zlib.compress(b"\0\1\2\3"), interlace=1)
    before = _lib.lib.tp_launch_count()
    with pytest.raises(ValueError, match="file 1: interlaced PNG"):
        decode_png_batch([ok, inter])
    assert _lib.lib.tp_launch_count() == before


def test_launch_count_follows_the_largest_raw_size(matrix):
    from tokenpacker_b200 import _lib, decode_png_batch
    files = [d for _, d in matrix[:20]]
    rows = [po.parse(f)["raw_bytes"] for f in files]
    before = _lib.lib.tp_launch_count()
    decode_png_batch(files)
    assert _lib.lib.tp_launch_count() - before == 5 + int(np.ceil(np.log2(max(rows))))


def test_committed_fixtures(golden_dir):
    from tokenpacker_b200 import decode_png_batch
    z = np.load(os.path.join(golden_dir, "png_fixtures.npz"))
    files = [z[f"file_{i}"].tobytes() for i in range(len(z["names"]))]
    for i, img in enumerate(decode_png_batch(files)):
        assert hashlib.sha256(img.cpu().numpy().tobytes()).hexdigest() == str(z["sha256"][i]), z["names"][i]


def _hooks():
    path = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_png_hooks.so")
    lib = C.CDLL(path)
    lib.tpp_decode_stages.restype = C.c_int
    lib.tpp_decode_stages.argtypes = [C.c_void_p] * 4 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p]
    return lib


def _region_ends(im):
    nbits = 8 * im.stream_bytes
    return {"mask": (im.mask_offset, im.mask_offset + 4 * ((nbits + 31) // 32)),
            "spec": (im.spec_offset, im.spec_offset + 20 * 4 * ((nbits + 255) // 256)),
            "blocks": (im.block_offset, im.block_offset + 20 * im.block_capacity),
            "raw": (im.raw_offset, im.raw_offset + im.raw_bytes), "src": (im.src_offset, im.src_offset + 4 * im.raw_bytes)}


@pytest.mark.parametrize("name", ["stored-fixed-dynamic", "limits-across-boundaries", "false-candidate", "level9", "40x1344-photo-RGB",
                                  "strategy-huffman-ct6"])
def test_stages_against_the_oracle(matrix, name):
    """Each stage through the hook library, for a two-file batch (the file and a second one after it): the candidates hold every
    true dynamic block start, the chain's block table is the oracle's, the second decode's literals and sources match, the resolved
    bytes are zlib's, the unfiltered rows and the final bytes PIL's.  Canaries: the workspace is filled with 0x5A and the output with
    0xA5 first; every gap between regions, the rest of each block table, the regions of stages not yet run and the workspace's tail
    keep their fill, for both files, so that no stage writes outside its own file's regions."""
    from tokenpacker_b200 import _lib, png as P
    hooks = _hooks()
    files = [dict(matrix)[name], dict(matrix)["64x97-photo-RGBA"]]
    refs = []
    for data in files:
        hdr = po.parse(data)
        refs.append((hdr,) + po.inflate(hdr["stream"]))
    for stage in range(1, 6):
        def launch(out, workspace, args, stream):
            out.fill_(0xA5)
            workspace.fill_(0x5A)
            assert hooks.tpp_decode_stages(*args, stage, stream) == 0
        rows, out, ws, status = P._plan_upload_launch(files, "cuda", launch)
        torch.cuda.synchronize()
        w = ws.cpu().numpy()
        o = out.cpu().numpy()
        sts = status.cpu().numpy()
        ends = []
        for f, (data, (hdr, raw_ref, blocks_ref, src_ref)) in enumerate(zip(files, refs)):
            im, st, reg = rows[f], sts[f], _region_ends(rows[f])
            ends.append(reg["src"][1])
            nbits = 8 * im.stream_bytes
            mask = np.frombuffer(w[reg["mask"][0]:reg["mask"][1]].tobytes(), np.uint32)
            cand = np.unpackbits(mask.view(np.uint8), bitorder="little")[:nbits]
            for b in blocks_ref:
                if b["type"] == 2:
                    assert cand[b["start_bit"]], b
            assert st[3] == cand.sum()
            order = ["mask", "spec", "blocks", "raw", "src"]
            for a, b in zip(order, order[1:]):                     # gaps between regions
                assert (w[reg[a][1]:reg[b][0]] == 0x5A).all(), (stage, a, b)
            if stage == 1:
                assert (w[reg["blocks"][0]:reg["src"][1]] == 0x5A).all()
                continue
            assert st[0] == 0 and st[1] == len(blocks_ref)
            tab = np.frombuffer(w[im.block_offset:im.block_offset + 20 * st[1]].tobytes(), np.uint32).reshape(-1, 5)
            for row, b in zip(tab, blocks_ref):
                assert (row[0], row[1], row[2], row[3], row[4] & 1, (row[4] >> 1) & 3) == (
                    b["start_bit"], b["end_bit"], b["out_offset"], b["out_bytes"], b["final"], b["type"])
            assert (w[im.block_offset + 20 * st[1]:reg["blocks"][1]] == 0x5A).all()
            if stage == 2:
                assert (w[reg["raw"][0]:reg["src"][1]] == 0x5A).all()
                continue
            rawb = w[reg["raw"][0]:reg["raw"][1]]
            if stage == 3:
                src = np.frombuffer(w[reg["src"][0]:reg["src"][1]].tobytes(), np.uint32).astype(np.int64)
                assert np.array_equal(src, src_ref)
                lit = src_ref == np.arange(len(src_ref))
                assert np.array_equal(rawb[lit], np.frombuffer(raw_ref, np.uint8)[lit])
            if stage == 4:
                assert rawb.tobytes() == raw_ref
            if stage == 5:
                rows_ref = po.unfilter(raw_ref, hdr["h"], hdr["row_bytes"], hdr["filter_bpp"])
                assert np.array_equal(rawb.reshape(hdr["h"], -1)[:, 1:], rows_ref)
                got = o[im.out_offset:im.out_offset + im.h * im.w * 3].reshape(im.h, im.w, 3)
                assert np.array_equal(got, pf.pil_decode(data))
        assert rows[1].mask_offset >= ends[0] and (w[ends[0]:rows[1].mask_offset] == 0x5A).all()
        end = _lib.lib.tp_png_workspace_bytes(rows, 2)
        assert end == ends[1] and (w[end:] == 0x5A).all()
        if stage < 5:
            assert (o == 0xA5).all()
        else:
            assert (o[rows[1].out_offset + rows[1].h * rows[1].w * 3:] == 0xA5).all()


@pytest.mark.parametrize("front", ["hd", "clip"])
def test_decode_then_front_end_equals_pil_then_front_end(matrix, front):
    from tokenpacker_b200 import clip_preprocess_batch, decode_png_batch, hd_preprocess_batch
    files = [d for n, d in matrix if n.startswith(("40x1344", "64x97"))][:8]
    gpu = decode_png_batch(files)
    pil = [torch.from_numpy(pf.pil_decode(f)).cuda() for f in files]
    if front == "hd":
        a, b = hd_preprocess_batch(gpu), hd_preprocess_batch(pil)
        a, b = a[0] if isinstance(a, tuple) else a, b[0] if isinstance(b, tuple) else b
    else:
        a, b = clip_preprocess_batch(gpu), clip_preprocess_batch(pil)
    assert torch.equal(a, b)
