"""LLaVA's vision-tower seam on the H100: the interleaved forward (include/tokenpacker_b200_clip_tower_interleaved.h) and the drop-in
``CLIPVisionTower`` built on it.  Every comparison is bit for bit against the dense forward (``tp_clip_tower_forward`` / ``_f16``,
``CLIPVisionTowerB200.hidden_states``), which the tower's own tests hold against fp64 and transformers.

1. Each 1024-column block of the interleaved buffer equals the matching dense output, at N = 1, 3, 29, 64 and 231 in bf16 and fp16,
   inside a sentinel-filled buffer whose guard crops stay untouched, with the dense forward's launch count.
2. Past 32-bit element offsets (N = 910): picked crops equal a dense forward of those crops alone.
3. ``forward(images)`` equals (hs[j][:, 1:], torch.cat(hs, 2)[:, 1:]) cast to images.dtype, for bf16 / fp32 crops, the bf16 / fp16
   towers, both select_feature modes and every select_layer block; feat and feat_multi are views of one buffer.
4. The encode step: TokenPackerB200.forward(dropin(images)) equals forward_hidden_states on the tower's hidden states (bf16, and the
   fp16 evaluation composition).
5. Memory at 64 crops: the drop-in allocates one [N, 577, 4096] buffer where hidden_states + torch.cat allocate two, and its peak is
   not above theirs (both peaks are the tower's workspace plus one such buffer: the concatenation runs after the workspace is freed).
"""
import ctypes as C

import pytest
import torch

from oracle import clip_tower_oracle as cto
from oracle import tokenpacker_oracle as tpo

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SENTINEL = -12345                                     # 0xCFC7: a NaN in neither bf16 nor f16


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


@pytest.fixture(scope="module")
def weights():
    return cto.make_weights(23, seed=0, device=DEV)


@pytest.fixture(scope="module")
def crops():
    return cto.make_images(231, seed=1, device=DEV).to(torch.bfloat16)


def _model(weights, dtype):
    return cto.FakeCLIPVisionModel({k: v.to(dtype) for k, v in weights.items()})


@pytest.fixture(scope="module")
def towers(weights):
    from tokenpacker_b200 import CLIPVisionTowerB200
    return {dt: CLIPVisionTowerB200(_model(weights, dt), dtype=dt) for dt in (torch.bfloat16, torch.float16)}


def _interleaved_into(tower, images, out):
    """tp_clip_tower_forward_interleaved(_f16) of images into out (a [N, 577, 4096] view); returns the launch count."""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    n = images.shape[0]
    packed, (w, _) = tower._packed_weights(images.device)
    ws_bytes = lib.tp_clip_tower_workspace_bytes(n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=images.device)
    stream = torch.cuda.current_stream().cuda_stream
    before = lib.tp_launch_count()
    if tower.dtype == torch.float16:
        status = lib.tp_clip_tower_forward_interleaved_f16(packed.data_ptr(), C.byref(w), images.data_ptr(), _lib.TP_CLIP_CROPS_BF16, n,
                                                           images.stride(0), out.data_ptr(), ws.data_ptr(), ws_bytes, stream)
    else:
        status = lib.tp_clip_tower_forward_interleaved(packed.data_ptr(), C.byref(w), images.data_ptr(), n, images.stride(0), out.data_ptr(),
                                                       ws.data_ptr(), ws_bytes, stream)
    assert status == 0, lib.tp_strerror(status)
    return lib.tp_launch_count() - before


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n", [1, 3, 29, 64, 231])
def test_interleaved_blocks_equal_the_dense_outputs(towers, crops, n, dtype):
    from tokenpacker_b200 import _lib
    tower, images = towers[dtype], crops[:n]
    tower._packed_weights(images.device)                     # the derived cache exists before either launch count is taken
    with torch.no_grad():
        before = _lib.lib.tp_launch_count()
        hs = tower.hidden_states(images)
        dense_launches = _lib.lib.tp_launch_count() - before
        buf = torch.full((n + 2, 577, 4096), SENTINEL, dtype=torch.int16, device=DEV).view(dtype)     # guard crops 0 and n + 1
        launches = _interleaved_into(tower, images, buf[1:n + 1])
    torch.cuda.synchronize()
    assert launches == dense_launches
    for j, h in enumerate(hs):
        assert _same(buf[1:n + 1, :, 1024 * j:1024 * (j + 1)], h), (n, j)
    guard = buf[[0, n + 1]].view(torch.int16)
    assert bool((guard == SENTINEL).all())
    assert _same(torch.cat(hs, 2), buf[1:n + 1])
    for h in hs:
        assert h.dtype == dtype and bool(torch.isfinite(h.float()).all())


def test_past_32_bit_offsets(towers, crops):
    """N = 910: element offsets into the output reach 910 * 577 * 4096 > 2^31 (from crop 909 on)."""
    n = 910
    tower = towers[torch.bfloat16]
    images = crops[torch.arange(n, device=DEV) % crops.shape[0]]
    with torch.no_grad():
        buf = tower.interleaved_hidden_states(images)
    assert buf.shape == (n, 577, 4096) and buf.dtype == torch.bfloat16
    picked = [0, 455, 908, 909]
    assert (picked[-1] * 577 * 4096) > 2 ** 31
    with torch.no_grad():
        hs = tower.hidden_states(images[picked])
    torch.cuda.synchronize()
    for j, h in enumerate(hs):
        assert _same(buf[picked, :, 1024 * j:1024 * (j + 1)], h), j
    del buf


def _args(layer, feature):
    from types import SimpleNamespace
    return SimpleNamespace(mm_vision_select_layer=layer, mm_vision_select_feature=feature)


@pytest.mark.parametrize("tower_dtype", [torch.bfloat16, torch.float16], ids=["bf16_tower", "fp16_tower"])
@pytest.mark.parametrize("crops_dtype", [torch.bfloat16, torch.float32], ids=["bf16_crops", "fp32_crops"])
@pytest.mark.parametrize("feature,layer,block", [("patch", -2, 3), ("cls_patch", -2, 3), ("patch", 12, 0), ("cls_patch", -9, 1),
                                                 ("patch", 22, 2)])
def test_dropin_forward_equals_feature_select_on_hidden_states(towers, crops, tower_dtype, crops_dtype, feature, layer, block):
    from tokenpacker_b200 import CLIPVisionTower
    images = cto.make_images(5, seed=7, device=DEV).to(crops_dtype)
    dropin = CLIPVisionTower(towers[tower_dtype].vision_model, _args(layer, feature))
    assert dropin.dtype == tower_dtype
    feat, feat_multi = dropin(images)
    with torch.no_grad():
        hs = towers[tower_dtype].hidden_states(images)
    rows = slice(1, None) if feature == "patch" else slice(None)
    assert _same(feat, hs[block][:, rows].to(crops_dtype))
    assert _same(feat_multi, torch.cat(hs, 2)[:, rows].to(crops_dtype))
    assert feat.shape == (5, 576 if feature == "patch" else 577, 1024) and feat_multi.shape[2] == 4096
    # views of one buffer: feat is the selected layer's column block of feat_multi
    assert feat.untyped_storage().data_ptr() == feat_multi.untyped_storage().data_ptr()
    assert feat.data_ptr() == feat_multi.data_ptr() + 1024 * block * feat.element_size()
    assert feat.stride() == feat_multi.stride() and feat_multi.stride()[1:] == (4096, 1)
    assert not feat.requires_grad and not feat_multi.requires_grad


def test_dropin_follows_the_model_precision_and_keeps_one_cache(weights, crops):
    from tokenpacker_b200 import CLIPVisionTower
    dropin = CLIPVisionTower(_model(weights, torch.bfloat16), _args(-2, "patch"))
    images = crops[:2]
    a = dropin(images)
    bf16_tower = dropin._towers[torch.bfloat16]
    packed = bf16_tower._packed
    assert packed is not None
    dropin(images)
    assert bf16_tower._packed is packed                                   # not rebuilt by every call
    dropin.to(dtype=torch.float16)                                        # what the evaluation scripts do
    assert dropin.dtype == torch.float16
    b = dropin(images)
    assert bf16_tower._packed is None and dropin._towers[torch.float16]._packed is not None
    with torch.no_grad():
        hs16 = dropin._towers[torch.float16].hidden_states(images)
    assert _same(b[1], torch.cat(hs16, 2)[:, 1:].to(torch.bfloat16))
    assert not _same(a[1], b[1])
    dropin.to(dtype=torch.bfloat16)
    dropin(images)
    assert dropin._towers[torch.float16]._packed is None and bf16_tower._packed is not None


def _projector(seed):
    from tokenpacker_b200 import TokenPackerB200
    params = {k: tpo.round_bf16(v) for k, v in tpo.make_params(4096, seed=seed).items()}
    m = TokenPackerB200(hidden_size=4096, scale_factor=2)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    return m.to(DEV, torch.bfloat16).eval()


def test_encode_step_equals_forward_hidden_states(towers, crops):
    from tokenpacker_b200 import CLIPVisionTower
    proj = _projector(3)
    images = crops[:29]
    with torch.no_grad():
        dropin = CLIPVisionTower(towers[torch.bfloat16].vision_model, _args(-2, "patch"))
        got = proj(dropin(images))
        want = proj.forward_hidden_states(towers[torch.bfloat16].hidden_states(images))
        assert got.shape == (29, 144, 4096) and _same(got, want)
        # the evaluation composition: an fp16 tower fed bf16 crops, its outputs cast to bf16 for the bf16 projector
        dropin16 = CLIPVisionTower(towers[torch.float16].vision_model, _args(-2, "patch"))
        got16 = proj(dropin16(images))
        want16 = proj.forward_hidden_states([h.to(torch.bfloat16) for h in towers[torch.float16].hidden_states(images)])
        assert _same(got16, want16)


def test_peak_memory_below_hidden_states_and_cat(towers, crops):
    from tokenpacker_b200 import CLIPVisionTower
    images = crops[:64]
    tower = towers[torch.bfloat16]
    dropin = CLIPVisionTower(tower.vision_model, _args(-2, "patch"))

    def measure(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        total = torch.cuda.memory_stats()["allocated_bytes.all.allocated"]
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            out = fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, torch.cuda.memory_stats()["allocated_bytes.all.allocated"] - total, out

    with torch.no_grad():                                                 # the derived caches exist before either arm is measured
        dropin(images[:1])
        tower.hidden_states(images[:1])

    def cat_arm():
        hs = tower.hidden_states(images)
        return hs[3][:, 1:], torch.cat(hs, 2)[:, 1:]

    p_dropin, alloc_dropin, a = measure(lambda: dropin(images))
    p_cat, alloc_cat, b = measure(cat_arm)
    assert _same(a[0], b[0]) and _same(a[1], b[1])
    buf_bytes = 64 * 577 * 4096 * 2
    ws_bytes = lib_workspace_bytes(64)
    slack = 8 << 20                                   # the caching allocator may hand out a cached block up to 1 MB larger than asked
    assert abs(alloc_dropin - (ws_bytes + buf_bytes)) < slack, (alloc_dropin, ws_bytes, buf_bytes)
    assert abs(alloc_cat - (ws_bytes + 2 * buf_bytes)) < slack, (alloc_cat, ws_bytes, buf_bytes)
    assert p_dropin <= p_cat + slack, (p_dropin, p_cat)


def lib_workspace_bytes(n):
    from tokenpacker_b200 import _lib
    return _lib.lib.tp_clip_tower_workspace_bytes(n)
