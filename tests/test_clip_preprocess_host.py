"""Non-HD CLIP input, host side (no CUDA): the numpy oracle against Pillow's resample and the slow CLIP processor, bit for bit; the
oracle against the committed processor fixture; the library's plan (tp_clip_preprocess_plan) against the oracle; argument
validation of the C entry points, from Python and from a plain-C consumer; and Python's checks before any device work."""
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import clip_preprocess_oracle as cpo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_u8.h")

# (in, out) sizes of one axis: downscales to about 25x, upscales, identity, a 1-pixel source
RESAMPLE_SIZES = [(8400, 336), (4000, 160), (1000, 40), (1344, 336), (1000, 336), (677, 336), (337, 336), (336, 336), (335, 336),
                  (200, 336), (90, 336), (17, 401), (2, 336), (1, 336), (1, 1), (5, 3)]
# (h, w) of the plan and pipeline checks
PLAN_SIZES = [(1, 1), (1, 4000), (4000, 1), (30, 600), (90, 120), (120, 90), (335, 336), (336, 336), (336, 337), (336, 500),
              (700, 336), (480, 640), (640, 480), (500, 333), (333, 500), (1344, 224), (224, 1344), (3000, 4000), (8000, 2999),
              (32768, 32768), (32768, 1)]


def test_oracle_resample_matches_pillow():
    """cpo.resize == PIL.Image.resize(BICUBIC, reducing_gap=None) on both axes together and on one axis only."""
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(21)
    pairs = [(a, b) for a, b in zip(RESAMPLE_SIZES, RESAMPLE_SIZES[3:] + RESAMPLE_SIZES[:3])]
    n = 0
    for (ih, oh), (iw, ow) in pairs:
        if ih * iw > 4_000_000:                                       # keep the source small; the output sizes are unchanged
            iw = max(1, 4_000_000 // ih)
        img = rng.integers(0, 256, size=(ih, iw, 3), dtype=np.uint8)
        for th, tw in ((oh, ow), (ih, ow), (oh, iw)):                 # both axes, horizontal only, vertical only
            ref = np.asarray(Image.fromarray(img).resize((tw, th), Image.BICUBIC, reducing_gap=None))
            np.testing.assert_array_equal(cpo.resize(img, th, tw), ref, err_msg=f"{(ih, iw)} -> {(th, tw)}")
            n += 1
    assert n == 3 * len(pairs)


def _pil_expand2square(pil, background):
    """The pad canvas built with PIL's own operations (Image.new + paste), as expand2square does."""
    from PIL import Image
    w, h = pil.size
    if w == h:
        return pil
    out = Image.new(pil.mode, (max(w, h), max(w, h)), background)
    out.paste(pil, (0, (w - h) // 2) if w > h else ((h - w) // 2, 0))
    return out


def test_oracle_pipeline_matches_slow_clip_processor():
    """The oracle == expand2square (pad) + transformers' slow CLIP processor with the openai/clip-vit-large-patch14-336 configuration,
    bit for bit, on seeded sizes in both modes."""
    pytest.importorskip("PIL")
    pytest.importorskip("transformers")
    try:
        from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil as Slow    # transformers >= 5
    except ImportError:
        from transformers import CLIPImageProcessor as Slow                                                # 4.x: the PIL processor
    from PIL import Image
    from oracle.gen_golden_clip_preprocess import PROCESSOR
    proc = Slow(**PROCESSOR)
    rng = np.random.default_rng(22)
    sizes = [(int(rng.integers(40, 1400)), int(rng.integers(40, 1400))) for _ in range(8)] + [(336, 600), (900, 336), (77, 1500)]
    for h, w in sizes:
        px = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        for mode in cpo.MODES:
            pil = Image.fromarray(px)
            if mode == "pad":
                pil = _pil_expand2square(pil, cpo.BACKGROUND)
            ref = proc.preprocess(pil, return_tensors="np")["pixel_values"][0]
            got = cpo.clip_preprocess(px, mode)
            assert ref.dtype == np.float32
            np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32), err_msg=f"{(h, w)} {mode}")


def test_oracle_matches_processor_fixture(golden_dir):
    """Digests and probes of every fixture case, and the processor's table == hd.norm_table() == cpo.table() in all 768 entries."""
    from tokenpacker_b200.hd import norm_table
    g = np.load(os.path.join(golden_dir, "clip_preprocess_u8.npz"))
    modes = set()
    for ci in range(int(g["n_cases"])):
        h, w, mi, seed = (int(v) for v in g[f"case{ci}_meta"])
        out = cpo.clip_preprocess(cpo.test_image(h, w, seed), cpo.MODES[mi])
        assert hashlib.sha256(out.tobytes()).hexdigest() == str(g[f"case{ci}_sha256"]), (h, w, cpo.MODES[mi])
        np.testing.assert_array_equal(out[:, ::37, ::41].view(np.uint32), g[f"case{ci}_probe"].view(np.uint32))
        np.testing.assert_array_equal(out.astype(np.float64).sum(axis=(1, 2)), g[f"case{ci}_sum"])
        modes.add(mi)
    assert modes == {0, 1}
    np.testing.assert_array_equal(g["table"].view(np.uint32), norm_table().numpy().view(np.uint32))
    np.testing.assert_array_equal(g["table"].view(np.uint32), cpo.table().view(np.uint32))
    ramp = cpo.test_image(336, 336, -1)
    assert all(np.unique(ramp[:, :, c]).size == 256 for c in range(3))


def _plan(sizes, mode):
    from tokenpacker_b200.clip import clip_preprocess_plan
    return clip_preprocess_plan(sizes, mode)


@pytest.mark.parametrize("mode", cpo.MODES)
def test_plan_matches_oracle(mode):
    """Geometry, bounds, int32 weights and row ranges of the library's plan == the oracle's, for every size; the tables are
    deduplicated by (input size, output size, first kept output); the workspace is the sum of the row ranges."""
    images, co, ws = _plan(PLAN_SIZES, mode)
    co = np.asarray(co, dtype=np.int64)
    keys, rows = {}, 0
    for (h, w), im in zip(PLAN_SIZES, images):
        g = cpo.geometry(h, w, mode)
        got = {k: getattr(im, k) for k in ("canvas_h", "canvas_w", "pad_y", "pad_x", "top", "left")}
        assert got == {k: g[k] for k in got} and (im.h, im.w) == (h, w)
        assert (im.resized_h, im.resized_w) == (g["rh"], g["rw"])
        for axis, in_size, out_size, first, ks, off in (("x", g["canvas_w"], g["rw"], g["left"], im.ksize_x, im.coeff_x),
                                                        ("y", g["canvas_h"], g["rh"], g["top"], im.ksize_y, im.coeff_y)):
            if in_size == out_size:
                assert ks == 0 and off == -1, (h, w, axis)
                continue
            xmin, n, k = cpo.coeffs(in_size, out_size)
            xmin, n, k = xmin[first:first + 336], n[first:first + 336], k[first:first + 336]
            assert ks == k.shape[1], (h, w, axis)
            tab = co[off:off + (2 + ks) * 336]
            np.testing.assert_array_equal(tab[:336], xmin)
            np.testing.assert_array_equal(tab[336:672], n)
            np.testing.assert_array_equal(tab[672:].reshape(ks, 336).T, k, err_msg=f"{(h, w)} {axis}")
            assert keys.setdefault((in_size, out_size, first), off) == off               # one table per key
            if axis == "y":                                     # the canvas rows the kept output rows read
                assert im.row0 == int(xmin.min())
                assert im.rows == (int((xmin + n).max()) - im.row0 if im.ksize_x else 0)
        if im.ksize_y == 0:
            assert im.row0 == g["top"] and im.rows == (336 if im.ksize_x else 0)
        assert im.workspace_row == rows and im.workspace_offset == rows * 336 * 3
        rows += im.rows
    assert ws == rows * 336 * 3
    assert len(co) == sum((2 + cpo.coeffs(i, o)[2].shape[1]) * 336 for i, o, _ in keys)
    if mode == "pad":
        assert len(keys) < sum(1 for h, w in PLAN_SIZES if max(h, w) != 336)          # both axes of a canvas share one table


def test_plan_dedup_across_images():
    """Repeated sizes add no table; in pad mode both orientations of one size share the canvas's table."""
    _, co1, _ = _plan([(480, 640)], "pad")
    _, co2, _ = _plan([(480, 640), (640, 480), (480, 640), (640, 640)], "pad")
    assert len(co1) == len(co2) == (2 + 9) * 336
    _, co3, _ = _plan([(480, 640), (640, 480)], "square")
    assert len(co3) == 2 * (2 + 7) * 336     # 480 -> 336 and 640 -> 448 from 56 on (7 taps each), shared by the transposed size


def test_plan_and_batch_argument_errors():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    bad = _lib.TP_ERR_INVALID_ARGUMENT
    a = (C.c_int64 * 2)(100, 200)
    n, ws = C.c_int64(0), C.c_size_t(0)
    for mode in (-1, 2, 7):
        assert lib.tp_clip_preprocess_plan(a, a, 2, mode, None, None, C.byref(n), C.byref(ws)) == bad
    assert lib.tp_clip_preprocess_plan(None, a, 2, 1, None, None, C.byref(n), C.byref(ws)) == bad
    assert lib.tp_clip_preprocess_plan(a, None, 2, 1, None, None, C.byref(n), C.byref(ws)) == bad
    assert lib.tp_clip_preprocess_plan(a, a, 2, 1, None, None, None, C.byref(ws)) == bad
    assert lib.tp_clip_preprocess_plan(a, a, 2, 1, None, None, C.byref(n), None) == bad
    assert lib.tp_clip_preprocess_plan(a, a, -1, 1, None, None, C.byref(n), C.byref(ws)) == bad
    for h, w in ((0, 5), (5, 0), (-3, 5), (32769, 5), (5, 32769)):
        s = (C.c_int64 * 1)(h), (C.c_int64 * 1)(w)
        assert lib.tp_clip_preprocess_plan(s[0], s[1], 1, 0, None, None, C.byref(n), C.byref(ws)) == bad, (h, w)
    assert lib.tp_clip_preprocess_plan(a, a, 0, 1, None, None, C.byref(n), C.byref(ws)) == _lib.TP_OK and n.value == 0 and ws.value == 0

    images, co, need = _plan([(480, 640), (336, 336), (90, 120)], "pad")
    host = (_lib.TpClipImage * 3)(*images)
    p = C.c_void_p(16)          # never dereferenced: every call below is refused before any CUDA work
    hp = C.addressof(host)
    args = [hp, p, p, p, 3, p, 0, p, p, need, None]
    for i in (0, 1, 2, 3, 5, 7):
        a2 = list(args)
        a2[i] = None
        assert lib.tp_clip_preprocess_batch(*a2) == bad, i
    for dt in (-1, 2):
        assert lib.tp_clip_preprocess_batch(hp, p, p, p, 3, p, dt, p, p, need, None) == bad
    assert lib.tp_clip_preprocess_batch(hp, p, p, p, -1, p, 0, p, p, need, None) == bad
    assert lib.tp_clip_preprocess_batch(hp, p, p, p, 1 << 40, p, 0, p, p, need, None) == bad          # more CTAs than a grid holds
    assert lib.tp_clip_preprocess_batch(hp, p, p, p, 3, p, 0, p, p, need - 1, None) == _lib.TP_ERR_WORKSPACE_TOO_SMALL
    assert lib.tp_clip_preprocess_batch(hp, p, p, p, 3, p, 0, p, None, need, None) == bad              # a workspace is needed
    assert lib.tp_clip_preprocess_batch(hp, p, p, p, 0, p, 1, p, None, 0, None) == _lib.TP_OK          # nothing to do, nothing launched
    assert C.sizeof(_lib.TpClipImage) == 88


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(", text)))


def test_clip_header_binding_and_exports_agree():
    """include/tokenpacker_b200_clip_u8.h only adds: its entry points are exported, bound by _lib.CLIP_U8_SIGNATURES with as many
    arguments as the header declares, and declared by no other header."""
    from tokenpacker_b200 import _lib
    names = _header_functions()
    assert names == ["tp_clip_preprocess_batch", "tp_clip_preprocess_plan"]
    assert sorted(_lib.CLIP_U8_SIGNATURES) == names
    assert not set(names) & (set(_lib.SIGNATURES) | set(_lib.HD_U8_SIGNATURES) | set(_lib.INPUT_GRAD_SIGNATURES))
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name in names:
        params = re.search(rf"\b{name}\s*\(([^;]*?)\)\s*;", text, flags=re.S).group(1)
        assert len(params.split(",")) == len(_lib.CLIP_U8_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"


def test_plain_c_consumer_of_the_clip_header(tmp_path):
    """The header is C99, its entry points link from plain C, and the plan and argument validation run without a GPU
    (tests/abi_c/abi_check_clip_u8.c)."""
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_u8")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_u8.c")
    text = open(src).read()
    for name in _header_functions():
        assert f"&{name}" in text, f"{name} missing from abi_check_clip_u8.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip_u8 ok" in r.stdout


def test_python_argument_errors_before_device_work():
    from tokenpacker_b200 import clip_preprocess_batch
    img = torch.zeros(20, 30, 3, dtype=torch.uint8)
    with pytest.raises(ValueError):
        clip_preprocess_batch([img], "slice")
    with pytest.raises(ValueError):
        clip_preprocess_batch([img], None)
    with pytest.raises(TypeError):
        clip_preprocess_batch([img.float()])
    with pytest.raises(ValueError):
        clip_preprocess_batch([torch.zeros(20, 30, dtype=torch.uint8)])
    with pytest.raises(ValueError):
        clip_preprocess_batch([img], layout="CHW")                   # [20,30,3] has 20 channels as CHW
    with pytest.raises(ValueError):
        clip_preprocess_batch([])
    for dt in (torch.float16, torch.float64):
        with pytest.raises(ValueError):
            clip_preprocess_batch([img], dtype=dt)
    with pytest.raises(RuntimeError, match="no CPU path"):
        clip_preprocess_batch([img], "square")
    with pytest.raises(RuntimeError, match="no CPU path"):
        clip_preprocess_batch([img.permute(2, 0, 1)], "pad", torch.bfloat16, "CHW")
