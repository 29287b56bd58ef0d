"""Decoded 8-bit HD input on the GPU (hd_preprocess_batch / tp_hd_preprocess_batch): the reference fixture, bit identity with
hd_tile_batch on the host-normalised float32 image, bf16 output, source layouts and strided views, byte coverage, and writes that
stay inside the output."""
import os

import numpy as np
import pytest
import torch

from oracle import hd_oracle as hdo
from oracle import hd_preprocess_oracle as hpo

pytestmark = pytest.mark.gpu


def _u8(px, layout="HWC"):
    t = torch.from_numpy(np.ascontiguousarray(px)).cuda()
    return t if layout == "HWC" else t.permute(2, 0, 1).contiguous()


def _normalised(u8_hwc):
    """The float32 [3,h,w] image that ToTensor + Normalize make of uint8 [h,w,3] (table lookup; the table is torchvision's bits)."""
    from tokenpacker_b200.hd import norm_table
    table = norm_table().cuda()
    return torch.stack([table[c][u8_hwc[:, :, c].long()] for c in range(3)])


def _config3_sizes():
    g = torch.Generator().manual_seed(0)                 # bench.py's configs[3] batch: 32 seeded sizes, patch_num 9 -> 231 crops
    hs = torch.randint(224, 1345, (32,), generator=g).tolist()
    ws = torch.randint(224, 1345, (32,), generator=g).tolist()
    return list(zip(hs, ws))


def _oracle_random_sizes():
    rng = np.random.default_rng(99)                      # the ten sizes of test_hd_gpu.py::test_tile_matches_oracle_random_sizes
    sizes = [(244, 1002, 9), (500, 700, 16), (1300, 900, 9), (77, 1411, 25), (1123, 1277, 25)]
    sizes += [(int(rng.integers(40, 1500)), int(rng.integers(40, 1500)), (9, 16, 25)[i % 3]) for i in range(5)]
    return sizes


def _fixture_cases(golden_dir):
    g = np.load(os.path.join(golden_dir, "hd_preprocess_u8.npz"))
    return g, [tuple(int(v) for v in g[f"case{ci}_meta"]) for ci in range(int(g["n_cases"]))]


def _assert_same_as_tile_batch(pixels, patch_num):
    """hd_preprocess_batch(uint8) == hd_tile_batch(host-normalised float32), bit for bit, as one batch and image by image."""
    from tokenpacker_b200 import hd_preprocess_batch, hd_tile_batch
    u8 = [_u8(px) for px in pixels]
    f32 = [_normalised(t) for t in u8]
    crops, hb, wb = hd_preprocess_batch(u8, patch_num)
    ref, rhb, rwb = hd_tile_batch(f32, patch_num)
    assert (hb, wb) == (rhb, rwb) and crops.dtype == torch.float32
    assert torch.equal(crops, ref)
    off = 0
    for t, f in zip(u8, f32):
        one, ohb, owb = hd_preprocess_batch([t], patch_num)
        assert torch.equal(one, hd_tile_batch([f], patch_num)[0])
        assert torch.equal(one, crops[off:off + one.shape[0]])
        off += one.shape[0]
    assert off == crops.shape[0]
    return crops, hb, wb


def test_matches_reference_fixture(golden_dir):
    """The reference's own preprocess + tiling block (model_vqa.py:62,88-123 on PIL images), within test_hd_gpu.py's tolerance
    for the tiling fixture: 3e-6 absolute on the probes, 1e-6 relative on the sums (the kernel contracts to fma where ATen's CPU
    code rounds, and vice versa)."""
    from tokenpacker_b200 import hd_preprocess_batch
    g, cases = _fixture_cases(golden_dir)
    for ci, (h, w, patch_num, hb, wb, seed) in enumerate(cases):
        crops, ohb, owb = hd_preprocess_batch([_u8(hpo.u8_test_image(h, w, seed))], patch_num)
        assert (ohb, owb) == ([hb], [wb])
        c = crops.cpu().numpy()
        assert c.shape == (hdo.n_crops(hb, wb), 3, 336, 336)
        np.testing.assert_allclose(c[:, :, ::37, ::41], g[f"case{ci}_probe"], atol=3e-6)
        ab = np.abs(c.astype(np.float64)).sum(axis=(1, 2, 3))
        np.testing.assert_allclose(ab, g[f"case{ci}_abs"], rtol=1e-6)
        assert np.all(np.abs(c.astype(np.float64).sum(axis=(1, 2, 3)) - g[f"case{ci}_sum"]) <= 1e-6 * ab)


def test_bit_identity_fixture_sizes_every_patch_num(golden_dir):
    _, cases = _fixture_cases(golden_dir)
    pixels = [hpo.u8_test_image(h, w, seed) for h, w, _, _, _, seed in cases]
    for patch_num in (9, 16, 25):
        _assert_same_as_tile_batch(pixels, patch_num)


def test_bit_identity_random_sizes():
    rng = np.random.default_rng(7)
    by_patch = {}
    for h, w, patch_num in _oracle_random_sizes():
        by_patch.setdefault(patch_num, []).append(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8))
    for patch_num, pixels in by_patch.items():
        _assert_same_as_tile_batch(pixels, patch_num)


def test_bit_identity_config3_batch_and_bf16():
    """The full configs[3] batch (32 images, 231 crops); the bf16 crops are the float32 crops rounded to nearest even."""
    from tokenpacker_b200 import hd_preprocess_batch
    rng = np.random.default_rng(11)
    pixels = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in _config3_sizes()]
    crops, hb, wb = _assert_same_as_tile_batch(pixels, 9)
    assert crops.shape[0] == 231
    u8 = [_u8(px) for px in pixels]
    b16, bhb, bwb = hd_preprocess_batch(u8, 9, dtype=torch.bfloat16)
    assert b16.dtype == torch.bfloat16 and (bhb, bwb) == (hb, wb)
    assert torch.equal(b16.view(torch.int16), crops.to(torch.bfloat16).view(torch.int16))


def test_one_by_one_grid_has_no_thumbnail():
    from tokenpacker_b200 import hd_preprocess_batch
    px = np.random.default_rng(3).integers(0, 256, size=(336, 336, 3), dtype=np.uint8)
    crops, hb, wb = _assert_same_as_tile_batch([px, hpo.u8_test_image(300, 280, 4)], 9)
    assert (hb[0], wb[0]) == (1, 1)
    one, _, _ = hd_preprocess_batch([_u8(px)], 9)
    assert one.shape[0] == 1                              # train.py:718: no thumbnail for a single crop
    b16, _, _ = hd_preprocess_batch([_u8(px)], 9, dtype=torch.bfloat16)
    assert torch.equal(b16.view(torch.int16), one.to(torch.bfloat16).view(torch.int16))


def test_layouts_and_views_agree():
    """HWC, CHW, a sub-window of a larger buffer (every stride differs from the contiguous one) and a permute view give the same bits."""
    from tokenpacker_b200 import hd_preprocess_batch
    rng = np.random.default_rng(21)
    sizes = [(500, 700), (1088, 900), (240, 1300)]
    for dt in (torch.float32, torch.bfloat16):
        pixels = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
        hwc = [_u8(px) for px in pixels]
        ref, hb, wb = hd_preprocess_batch(hwc, 9, dtype=dt)
        chw, _, _ = hd_preprocess_batch([t.permute(2, 0, 1).contiguous() for t in hwc], 9, dtype=dt, layout="CHW")
        perm, _, _ = hd_preprocess_batch([t.permute(2, 0, 1) for t in hwc], 9, dtype=dt, layout="CHW")
        windows = []
        for t in hwc:
            h, w, _ = t.shape
            big = torch.randint(0, 256, (h + 9, w + 13, 5), dtype=torch.uint8, device="cuda")
            big[4:4 + h, 7:7 + w, 1:4] = t
            windows.append(big[4:4 + h, 7:7 + w, 1:4])   # strides (5 (w + 13), 5, 1), offset into the buffer
        win, _, _ = hd_preprocess_batch(windows, 9, dtype=dt)
        chw_windows = []
        for t in hwc:
            h, w, _ = t.shape
            big = torch.randint(0, 256, (4, h + 3, w + 6), dtype=torch.uint8, device="cuda")
            big[1:4, 2:2 + h, 5:5 + w] = t.permute(2, 0, 1)
            chw_windows.append(big[1:4, 2:2 + h, 5:5 + w])
        cwin, _, _ = hd_preprocess_batch(chw_windows, 9, dtype=dt, layout="CHW")
        for other in (chw, perm, win, cwin):
            assert torch.equal(other, ref)


def test_byte_coverage_and_constant_images():
    """Every byte value in every channel (ramps), and constant 0 / 255 images: bit identity with the float32 path, and the content
    of a constant image is that constant's normalised value wherever no padding is involved."""
    from tokenpacker_b200 import hd_preprocess_batch
    from tokenpacker_b200.hd import hd_fit, hd_grid, norm_table
    ramps = [hpo.u8_test_image(h, w, -1) for h, w in ((256, 256), (300, 457), (17, 1200))]
    for px in ramps:
        for c in range(3):
            assert np.unique(px[:, :, c]).size == 256
    consts = [np.full((h, w, 3), v, dtype=np.uint8) for v in (0, 255) for h, w in ((500, 700), (336, 336))]
    _assert_same_as_tile_batch(ramps + consts, 9)
    table = norm_table()
    for px in consts:
        h, w = px.shape[:2]
        v = int(px[0, 0, 0])
        crops, hb, wb = hd_preprocess_batch([_u8(px)], 9)
        (h_r, w_r), _ = hd_fit(h, w, *hd_grid(h, w, 9))
        canvas = crops[0]                                 # the first crop lies wholly inside the resized content here
        assert h_r >= 336 and w_r >= 336
        for c in range(3):
            # the bilinear weights sum to 1 up to rounding: a few float32 ulps of the constant, never the padding's 0.0
            want = float(table[c, v])
            assert float((canvas[c] - want).abs().max()) <= 1e-6 * abs(want)


def _call_abi_into(out_full, u8, patch_num, out_dtype):
    """The launch of hd_preprocess_batch re-issued through the C ABI into a caller-owned output."""
    from tokenpacker_b200 import hd_preprocess_batch
    from tokenpacker_b200._lib import lib
    _, hb, wb, (tables, src_off, table_off, n, table) = hd_preprocess_batch(u8, patch_num, _return_launch=True)
    stream = torch.cuda.current_stream().cuda_stream
    st = lib.tp_hd_preprocess_batch(tables.data_ptr(), tables.data_ptr() + src_off, tables.data_ptr() + table_off, n, table.data_ptr(),
                                    out_dtype, out_full.data_ptr(), stream)
    torch.cuda.synchronize()
    return st, hb, wb, n


def test_writes_stay_inside_the_output():
    """Into a NaN-filled output with one sentinel crop after the end: every element of every crop is written, the sentinel is left
    alone, and the thumbnail is exactly 0 past its fitted size (train.py:728), as the canvas is past its resized content (:710)."""
    from tokenpacker_b200 import hd_preprocess_batch
    from tokenpacker_b200._lib import TP_OK
    from tokenpacker_b200.hd import hd_fit
    rng = np.random.default_rng(5)
    sizes = [(500, 700), (336, 336), (1300, 250), (901, 333)]
    u8 = [_u8(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)) for h, w in sizes]
    for out_dtype, dt, bits in ((0, torch.float32, torch.int32), (1, torch.bfloat16, torch.int16)):
        ref, _, _ = hd_preprocess_batch(u8, 9, dtype=dt)
        n = ref.shape[0]
        out = torch.full((n + 1, 3, 336, 336), float("nan"), dtype=dt, device="cuda")
        fill = out[n].clone()
        st, hb, wb, n2 = _call_abi_into(out, u8, 9, out_dtype)
        assert st == TP_OK and n2 == n
        assert not torch.isnan(out[:n]).any()
        assert torch.equal(out[:n].view(bits), ref.view(bits))
        assert torch.equal(out[n].view(bits), fill.view(bits))
        off = 0
        for (h, w), a, b in zip(sizes, hb, wb):
            (h_r, w_r), (h_t, w_t) = hd_fit(h, w, a, b)
            k = hdo.n_crops(a, b)
            canvas = out[off:off + a * b].view(a, b, 3, 336, 336).permute(2, 0, 3, 1, 4).reshape(3, a * 336, b * 336)
            assert not canvas[:, h_r:].float().any() and not canvas[:, :, w_r:].float().any()
            if k > a * b:
                thumb = out[off + a * b]
                assert not thumb[:, h_t:].float().any() and not thumb[:, :, w_t:].float().any()
            off += k
        assert off == n
