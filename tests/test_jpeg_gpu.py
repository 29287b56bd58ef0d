"""decode_jpeg_batch on the GPU against PIL, bit for bit: the fixture matrix one file at a time and as one mixed batch, repeated runs,
a stream whose subsequences need several synchronisation rounds, a truncated entropy-coded segment, and decode followed by the GPU
front ends against PIL decode followed by the same calls."""
import io
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_fixtures as jf  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def matrix():
    return jf.matrix()


def test_matrix_one_file_at_a_time(matrix):
    from tokenpacker_b200 import decode_jpeg_batch
    for name, data in matrix:
        (got,) = decode_jpeg_batch([data])
        assert got.dtype == torch.uint8 and got.is_cuda
        assert np.array_equal(got.cpu().numpy(), jf.pil_decode(data)), name


def test_matrix_as_one_batch_equals_per_file_and_repeats(matrix):
    from tokenpacker_b200 import decode_jpeg_batch
    files = [d for _, d in matrix]
    # the three input forms
    forms = [f if i % 3 == 0 else (np.frombuffer(f, np.uint8) if i % 3 == 1 else torch.frombuffer(bytearray(f), dtype=torch.uint8))
             for i, f in enumerate(files)]
    first = [t.cpu().numpy() for t in decode_jpeg_batch(forms)]
    for (name, data), got in zip(matrix, first):
        assert np.array_equal(got, jf.pil_decode(data)), name
    again, status = decode_jpeg_batch(files, return_status=True)
    assert status[:, 0].abs().sum().item() == 0
    for a, b in zip(first, again):
        assert np.array_equal(a, b.cpu().numpy())


def _flat_gray(h, w, value=128):
    b = io.BytesIO()
    Image.fromarray(np.full((h, w), value, np.uint8)).save(b, "JPEG", quality=75)
    return b.getvalue()


def test_periodic_stream_needs_several_rounds():
    """A flat image codes every block alike (a 6-bit period against 1024-bit subsequences), so a speculative decode that starts out
    of phase can stay out of phase: the rounds must carry the true state forward, and the result must not depend on how many run."""
    from tokenpacker_b200 import decode_jpeg_batch
    files = [_flat_gray(512, 2048), _flat_gray(64, 64, 37)]
    imgs, status = decode_jpeg_batch(files, return_status=True)
    st = status.cpu().numpy()
    assert (st[:, 0] == 0).all()
    for f, g in zip(files, imgs):
        assert np.array_equal(g.cpu().numpy(), jf.pil_decode(f))
    print("sync rounds", st[:, 1].tolist(), "subsequences", st[:, 2].tolist())
    assert st[0, 1] >= 2


def test_truncated_entropy_segment_is_reported_and_others_decode(matrix):
    from tokenpacker_b200 import decode_jpeg_batch
    good = [d for n, d in matrix if n.startswith("333x517-420")][:2]
    whole = jf.encode(jf.image(333, 517, "noise", 3), "420", 90)
    cut = whole[:len(whole) // 2]                  # the header is whole, the scan stops half way
    files = [good[0], cut, good[1]]
    imgs, status = decode_jpeg_batch(files, return_status=True)
    st = status.cpu().numpy()
    assert st[1, 0] == 1 and st[0, 0] == 0 and st[2, 0] == 0
    assert np.array_equal(imgs[0].cpu().numpy(), jf.pil_decode(good[0]))
    assert np.array_equal(imgs[2].cpu().numpy(), jf.pil_decode(good[1]))
    with pytest.raises(ValueError, match="file 1: corrupt or truncated"):
        decode_jpeg_batch(files)
    with pytest.raises(OSError):
        jf.pil_decode(cut)                         # PIL refuses the file too


def test_refused_file_raises_before_any_launch():
    from tokenpacker_b200 import decode_jpeg_batch
    b = io.BytesIO()
    Image.fromarray(jf.image(40, 40, "grad", 1)).save(b, "JPEG", progressive=True)
    with pytest.raises(ValueError, match="file 1: progressive JPEG"):
        decode_jpeg_batch([_flat_gray(8, 8), b.getvalue()])


@pytest.mark.parametrize("h,w", [(333, 517), (1345, 224), (640, 480)])
def test_decode_then_front_ends_equal_pil_then_front_ends(h, w):
    from tokenpacker_b200 import decode_jpeg_batch, hd_preprocess_batch, clip_preprocess_batch
    files = [jf.encode(jf.image(h, w, k, 7), "420", 90) for k in ("grad", "noise")] + [jf.encode(jf.image(w, h, "edges", 8), "gray", 80)]
    ours = decode_jpeg_batch(files)
    ref = [torch.from_numpy(jf.pil_decode(f)).cuda() for f in files]
    a, hb_a, wb_a = hd_preprocess_batch(ours, dtype=torch.bfloat16)
    b, hb_b, wb_b = hd_preprocess_batch(ref, dtype=torch.bfloat16)
    assert (hb_a, wb_a) == (hb_b, wb_b) and torch.equal(a, b)
    for mode in ("pad", "square"):
        assert torch.equal(clip_preprocess_batch(ours, mode), clip_preprocess_batch(ref, mode))


def test_committed_fixtures_on_the_gpu(golden_dir):
    import hashlib
    from tokenpacker_b200 import decode_jpeg_batch
    z = np.load(os.path.join(golden_dir, "jpeg_fixtures.npz"))
    files = [z[f"file_{i}"] for i in range(len(z["names"]))]    # uint8 numpy arrays
    for i, got in enumerate(decode_jpeg_batch(files)):
        assert hashlib.sha256(got.cpu().numpy().tobytes()).hexdigest() == str(z["sha256"][i]), str(z["names"][i])


def test_files_cut_short_at_the_tail_are_reported_where_the_oracle_raises(matrix):
    """The last one or two scan bytes and the EOI dropped: a file whose last needed block read past the end reports status 1 (the
    oracle raises, and so does PIL); one whose dropped bytes were only padding decodes as the oracle decodes it."""
    from oracle import jpeg_oracle as jo
    from tokenpacker_b200 import decode_jpeg_batch
    small = [d for n, d in matrix if not n.startswith(("1000x", "1345x"))][::2]
    files = [d[:-cut] for cut in (3, 4) for d in small]
    imgs, status = decode_jpeg_batch(files, return_status=True)
    st = status[:, 0].cpu().numpy()
    raised = 0
    for i, f in enumerate(files):
        try:
            ref = jo.decode(f)
        except ValueError:
            raised += 1
            assert st[i] == 1, i
            continue
        assert st[i] == 0 and np.array_equal(imgs[i].cpu().numpy(), ref), i
    assert raised > len(files) // 4


def _restart_file(rows=True):
    kw = {"restart_marker_rows": 1} if rows else {"restart_marker_blocks": 2}
    return jf.encode(jf.image(96, 128, "noise", 11), "420", 90, **kw)


def test_restart_markers_missing_report_their_status():
    from tokenpacker_b200 import decode_jpeg_batch
    whole = _restart_file()
    ok = jf.encode(jf.image(50, 70, "grad", 12), "444", 80)
    imgs, status = decode_jpeg_batch([ok, whole[:len(whole) // 2], whole], return_status=True)
    st = status[:, 0].cpu().numpy()
    assert st.tolist() == [0, 2, 0]
    assert np.array_equal(imgs[0].cpu().numpy(), jf.pil_decode(ok))
    assert np.array_equal(imgs[2].cpu().numpy(), jf.pil_decode(whole))


def test_corrupt_middle_interval_is_reported():
    """One restart interval's entropy bytes replaced by stuffed 0xFF bytes (all ones: no valid code), the markers kept."""
    from tokenpacker_b200 import decode_jpeg_batch
    whole = _restart_file(rows=False)
    sos = whole.index(b"\xff\xda")
    rst = [i for i in range(sos, len(whole) - 1) if whole[i] == 0xFF and 0xD0 <= whole[i + 1] <= 0xD7]
    a, b = rst[len(rst) // 2] + 2, rst[len(rst) // 2 + 1]
    bad = whole[:a] + b"\xff\x00" * ((b - a) // 2) + whole[a + 2 * ((b - a) // 2):]
    imgs, status = decode_jpeg_batch([whole, bad], return_status=True)
    assert status[:, 0].tolist() == [0, 1]
    assert np.array_equal(imgs[0].cpu().numpy(), jf.pil_decode(whole))


def test_speculative_errors_do_not_travel_down_the_chain():
    """On natural content most speculative decodes synchronise within their subsequence; an error met while decoding speculatively
    must not be handed on one subsequence per round, which would make the rounds as many as the subsequences."""
    from tokenpacker_b200 import decode_jpeg_batch
    files = []
    for n, (h, w, sub) in enumerate([(600, 800, "420"), (480, 640, "444"), (700, 500, "gray")]):
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        base = np.stack([128 + 100 * np.sin(xx / 37 + c) * np.cos(yy / 53 - c) for c in range(3)], 2)
        a = np.clip(base + np.random.default_rng(n).normal(0, 6, (h, w, 3)), 0, 255).astype(np.uint8)
        files.append(jf.encode(a, sub, 90))
    imgs, status = decode_jpeg_batch(files, return_status=True)
    st = status.cpu().numpy()
    for i, f in enumerate(files):
        assert st[i, 0] == 0 and np.array_equal(imgs[i].cpu().numpy(), jf.pil_decode(f))
        assert st[i, 2] >= 100 and st[i, 1] <= st[i, 2] // 8, st[i].tolist()


def test_jfif_with_adobe_transform_decodes_as_ycbcr():
    """libjpeg reads a JFIF file as YCbCr whatever its Adobe transform; a transform other than 0 without JFIF is YCbCr too."""
    from tokenpacker_b200 import decode_jpeg_batch
    base = jf.encode(jf.image(45, 61, "sat", 13), "420", 85)
    files = [jf.with_adobe(base, t) for t in (0, 1, 2)]
    for f, got in zip(files, decode_jpeg_batch(files)):
        assert np.array_equal(got.cpu().numpy(), jf.pil_decode(f))
