"""Non-HD CLIP input on the GPU (clip_preprocess_batch / tp_clip_preprocess_batch): the processor fixture by digest, the numpy oracle
bit for bit on the configs[3] sizes in both modes, batched against per-image calls, bf16, source layouts and strided views, byte and
clipping coverage, extreme sizes, writes and reads that stay inside their image, and run-to-run identity.  Every comparison is exact."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import clip_preprocess_oracle as cpo

pytestmark = pytest.mark.gpu


def _u8(px, layout="HWC"):
    t = torch.from_numpy(np.ascontiguousarray(px)).cuda()
    return t if layout == "HWC" else t.permute(2, 0, 1).contiguous()


def _assert_oracle(pixels, mode, out):
    """out [3, 336, 336] float32 (CUDA) equals the oracle bit for bit."""
    ref = cpo.clip_preprocess(pixels, mode)
    got = out.cpu().numpy()
    if not np.array_equal(got.view(np.uint32), ref.view(np.uint32)):
        bad = np.argwhere(got.view(np.uint32) != ref.view(np.uint32))
        pytest.fail(f"{pixels.shape} {mode}: {len(bad)} values differ, first at {tuple(bad[0])}: {got[tuple(bad[0])]} vs {ref[tuple(bad[0])]}")


def _config3_sizes():
    g = torch.Generator().manual_seed(0)                 # bench.py's configs[3] batch: 32 seeded sizes 224..1344
    hs = torch.randint(224, 1345, (32,), generator=g).tolist()
    ws = torch.randint(224, 1345, (32,), generator=g).tolist()
    return list(zip(hs, ws))


def test_matches_processor_fixture(golden_dir):
    """The reference's expand2square + the slow CLIP processor (fixture), by SHA-256 of the float32 output; batched per mode."""
    from tokenpacker_b200 import clip_preprocess_batch
    g = np.load(os.path.join(golden_dir, "clip_preprocess_u8.npz"))
    cases = [tuple(int(v) for v in g[f"case{ci}_meta"]) for ci in range(int(g["n_cases"]))]
    for mi, mode in enumerate(cpo.MODES):
        idx = [ci for ci, c in enumerate(cases) if c[2] == mi]
        out = clip_preprocess_batch([_u8(cpo.test_image(cases[ci][0], cases[ci][1], cases[ci][3])) for ci in idx], mode)
        assert out.dtype == torch.float32 and tuple(out.shape) == (len(idx), 3, 336, 336)
        host = out.cpu().numpy()
        for j, ci in enumerate(idx):
            assert hashlib.sha256(host[j].tobytes()).hexdigest() == str(g[f"case{ci}_sha256"]), cases[ci]
            np.testing.assert_array_equal(host[j][:, ::37, ::41].view(np.uint32), g[f"case{ci}_probe"].view(np.uint32))


@pytest.mark.parametrize("mode", cpo.MODES)
def test_config3_sizes_match_oracle_batched_and_per_image(mode):
    from tokenpacker_b200 import clip_preprocess_batch
    rng = np.random.default_rng(11)
    pixels = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in _config3_sizes()]
    imgs = [_u8(p) for p in pixels]
    out = clip_preprocess_batch(imgs, mode)
    assert tuple(out.shape) == (32, 3, 336, 336)
    for i, p in enumerate(pixels):
        _assert_oracle(p, mode, out[i])
    for i, t in enumerate(imgs[:8]):
        assert torch.equal(clip_preprocess_batch([t], mode)[0].view(torch.int32), out[i].view(torch.int32))
    bf = clip_preprocess_batch(imgs, mode, dtype=torch.bfloat16)
    assert bf.dtype == torch.bfloat16
    assert torch.equal(bf.view(torch.int16), out.to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize("mode", cpo.MODES)
def test_layouts_and_strided_views(mode):
    from tokenpacker_b200 import clip_preprocess_batch
    rng = np.random.default_rng(12)
    px = rng.integers(0, 256, size=(413, 701, 3), dtype=np.uint8)
    ref = clip_preprocess_batch([_u8(px)], mode)
    big = torch.from_numpy(rng.integers(0, 256, size=(500, 900, 3), dtype=np.uint8)).cuda()
    big[37:37 + 413, 101:101 + 701] = _u8(px)
    wide = torch.zeros((413, 701, 5), dtype=torch.uint8, device="cuda")          # channel stride 1, column stride 5
    wide[:, :, 1:4] = _u8(px)
    planes = torch.zeros((3, 413, 800), dtype=torch.uint8, device="cuda")        # CHW with a row pitch of 800
    planes[:, :, :701] = _u8(px, "CHW")
    for imgs, layout in (([_u8(px, "CHW")], "CHW"), ([big[37:37 + 413, 101:101 + 701]], "HWC"), ([wide[:, :, 1:4]], "HWC"),
                         ([planes[:, :, :701]], "CHW"), ([_u8(px).permute(2, 0, 1)], "CHW"), ([_u8(px, "CHW").permute(1, 2, 0)], "HWC")):
        assert torch.equal(clip_preprocess_batch(imgs, mode, layout=layout).view(torch.int32), ref.view(torch.int32)), layout


def _checkerboard(h, w):
    y, x = np.indices((h, w))
    return np.repeat((((y + x) % 2) * 255).astype(np.uint8)[:, :, None], 3, axis=2)


@pytest.mark.parametrize("mode", cpo.MODES)
def test_byte_and_clipping_coverage(mode):
    """Every byte in every channel, constant 0 / 255, a one-pixel checkerboard (the negative lobes clip at 0 and 255), and the pad
    background next to saturated pixels."""
    from tokenpacker_b200 import clip_preprocess_batch
    ramp = cpo.test_image(517, 389, -1)
    cases = [ramp, cpo.test_image(336, 336, -1), np.zeros((300, 451, 3), np.uint8), np.full((451, 300, 3), 255, np.uint8),
             _checkerboard(640, 480), _checkerboard(150, 150), _checkerboard(200, 150), np.full((100, 700, 3), 255, np.uint8),
             np.zeros((700, 101, 3), np.uint8)]
    out = clip_preprocess_batch([_u8(p) for p in cases], mode)
    for p, o in zip(cases, out):
        _assert_oracle(p, mode, o)
    # the 150 x 150 checkerboard is the same canvas in both modes; its upscale overshoots to -24 .. 279 before the clip
    xmin, _, k = cpo.coeffs(150, 336)
    acc = sum(_checkerboard(150, 150)[:, np.minimum(xmin + j, 149), 0].astype(np.int64) * k[:, j] for j in range(k.shape[1]))
    assert ((acc + (1 << 21)) >> 22).min() < 0 and ((acc + (1 << 21)) >> 22).max() > 255


@pytest.mark.parametrize("mode", cpo.MODES)
def test_extreme_sizes(mode):
    """1 x 1, 1 x 4000, 4000 x 3000 and an 8000-pixel side (97 taps on the 8000 x 8000 pad canvas)."""
    from tokenpacker_b200 import clip_preprocess_batch
    rng = np.random.default_rng(13)
    cases = [rng.integers(0, 256, size=s, dtype=np.uint8) for s in ((1, 1, 3), (1, 4000, 3), (4000, 3000, 3), (8000, 2999, 3))]
    out = clip_preprocess_batch([_u8(p) for p in cases], mode)
    for p, o in zip(cases, out):
        _assert_oracle(p, mode, o)


@pytest.mark.parametrize("mode", cpo.MODES)
def test_confinement_poisoned_workspace_and_sentinels(mode):
    """The workspace is filled with 0xFF before the launches and the output sits between NaN sentinel images of a larger buffer: the
    sentinels stay untouched and the result is unchanged, so no read of an unwritten workspace row and no write outside its image."""
    from tokenpacker_b200 import clip_preprocess_batch
    from tokenpacker_b200._lib import check, lib
    rng = np.random.default_rng(14)
    sizes = [(480, 640), (336, 336), (120, 90), (1000, 333), (336, 777)]
    imgs = [_u8(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)) for h, w in sizes]
    ref, (dev, soff, coff, plan, ws, table) = clip_preprocess_batch(imgs, mode, _return_launch=True)
    torch.cuda.synchronize()
    tabs = dev.clone()                                            # the staging buffer is shared by later calls
    ws.fill_(0xFF)
    framed = torch.full((len(sizes) + 2, 3, 336, 336), float("nan"), device="cuda")
    check(lib.tp_clip_preprocess_batch(C.addressof(plan), tabs.data_ptr(), tabs.data_ptr() + soff, tabs.data_ptr() + coff, len(sizes),
                                       table.data_ptr(), 0, framed[1:].data_ptr(), ws.data_ptr(), ws.numel(),
                                       torch.cuda.current_stream().cuda_stream), "tp_clip_preprocess_batch")
    torch.cuda.synchronize()
    assert torch.isnan(framed[0]).all() and torch.isnan(framed[-1]).all()
    assert torch.equal(framed[1:-1].view(torch.int32), ref.view(torch.int32))


def test_two_runs_identical():
    from tokenpacker_b200 import clip_preprocess_batch
    rng = np.random.default_rng(15)
    imgs = [_u8(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)) for h, w in _config3_sizes()[:12]]
    for mode in cpo.MODES:
        a = clip_preprocess_batch(imgs, mode, dtype=torch.bfloat16)
        b = clip_preprocess_batch(imgs, mode, dtype=torch.bfloat16)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
