"""Gradients to the pixels on the GPU (``CLIPVisionTowerB200.input_grad``, ``hd_tile_batch`` / ``hd_tile`` under autograd,
include/tokenpacker_b200_clip_tower_crop_grad.h): the crops' gradient against the fp64 autograd oracle; parameter gradients with the bits
of the step without input_grad; checkpointing, repetition, crop dtypes and crop views; the 231-crop HD batch; the tiling backward
against fp64 and batched against per-image; one end-to-end image gradient through the projector; the launches the step adds."""
import pytest
import torch

from oracle import clip_tower_oracle as cto
from oracle import crop_grad_oracle as cgo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GATE = 1e-2                                                 # rel-RMS of d(crops), of the order of the embedding stage's gradients


@pytest.fixture(scope="module")
def weights():
    return cto.round_bf16(cto.make_weights(23, seed=11, device=DEV))


def _model(w, layers=False, embed=False):
    model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    for name, p in model.named_parameters():
        p.requires_grad_(layers if "encoder.layers." in name else embed)
    return model


def _d_outs(n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return {j: (torch.randn(n, 577, 1024, generator=g, device=DEV) * 0.1).bfloat16() for j in cto.OUT_LAYERS}


def _backward(outs, d_outs):
    pairs = [(o, d_outs[j]) for o, j in zip(outs, cto.OUT_LAYERS) if d_outs[j] is not None and o.requires_grad]
    torch.autograd.backward([o for o, _ in pairs], [d for _, d in pairs])
    torch.cuda.synchronize()


def _rel(got, ref):
    ref = ref.double()
    return float((got.double() - ref).norm() / ref.norm().clamp_min(1e-300))


def _crop_step(tower, images, d_outs):
    x = images.detach().clone().requires_grad_(True)
    _backward(tower.hidden_states(x), d_outs)
    return x.grad


def _oracle(w, images, d_outs):
    d = {j: None if v is None else v.double() for j, v in d_outs.items()}
    return cgo.crop_gradients_chunked(w, images.double(), d, chunk=4, device=DEV)


@pytest.mark.parametrize("n", [1, 3, 29, 64], ids=["N1", "N3", "N29-splitk", "N64"])
def test_crop_gradient_against_fp64_oracle(weights, n):
    from tokenpacker_b200 import CLIPVisionTowerB200
    t = CLIPVisionTowerB200(_model(weights))
    t.input_grad = True
    images = cto.make_images(n, seed=40 + n, device=DEV).bfloat16().float()
    d_outs = _d_outs(n, 50 + n)
    got = _crop_step(t, images, d_outs)
    assert got.dtype == torch.float32 and got.shape == images.shape and torch.isfinite(got).all()
    ref = _oracle(weights, images, d_outs)
    err = _rel(got, ref)
    worst = max(_rel(got[i], ref[i]) for i in range(n))
    print(f"N={n}: d(crops) rel-RMS {err:.2e}, worst crop {worst:.2e}")
    assert err < GATE and worst < 2 * GATE, (err, worst)


def _param_grads(model):
    return {name: p.grad.clone() for name, p in model.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("k,embed", [(0, False), (4, False), (23, True)], ids=["frozen", "K4", "K23-embed"])
def test_parameter_gradients_keep_their_bits(weights, k, embed):
    """Every parameter gradient is bit-identical to the step without input_grad; checkpointing and repetition change no bit of d(crops)."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _model(weights, layers=k > 0, embed=embed)
    t = CLIPVisionTowerB200(model, trainable_layers=k, train_embeddings=embed)
    n = 2
    images = cto.make_images(n, seed=60, device=DEV).bfloat16()
    d_outs = _d_outs(n, 61)
    d_outs[16] = None
    with torch.no_grad():
        ref_outs = CLIPVisionTowerB200(model).hidden_states(images)
    plain = None
    if k > 0:
        _backward(t.hidden_states(images), d_outs)
        plain = _param_grads(model)
        model.zero_grad(set_to_none=True)
    t.input_grad = True
    crop_grads = []
    for checkpointing in (False, True, False):
        model.gradient_checkpointing = checkpointing
        x = images.detach().clone().requires_grad_(True)
        outs = t.hidden_states(x)
        for a, b, j in zip(outs, ref_outs, cto.OUT_LAYERS):
            assert torch.equal(a, b) and a.requires_grad, j
        _backward(outs, d_outs)
        crop_grads.append(x.grad)
        if plain is not None:
            got = _param_grads(model)
            assert got.keys() == plain.keys()
            for name in plain:
                assert torch.equal(got[name], plain[name]), (checkpointing, name)
            model.zero_grad(set_to_none=True)
        else:
            assert not _param_grads(model)
    assert crop_grads[0].dtype == torch.bfloat16
    assert torch.equal(crop_grads[0], crop_grads[1]) and torch.equal(crop_grads[0], crop_grads[2])


def test_crop_dtypes_and_views(weights):
    """fp32 crops get the fp32 gradient, bf16 crops its rounding; a crop view with a wider crop stride gets the same bits."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    t = CLIPVisionTowerB200(_model(weights))
    t.input_grad = True
    n = 3
    images = cto.make_images(n, seed=70, device=DEV).bfloat16()
    d_outs = _d_outs(n, 71)
    g32 = _crop_step(t, images.float(), d_outs)
    g16 = _crop_step(t, images, d_outs)
    assert g32.dtype == torch.float32 and g16.dtype == torch.bfloat16
    assert torch.equal(g16, g32.bfloat16())
    base = torch.zeros(n, 4, 336, 336, device=DEV)
    base[:, 1:] = images.float()
    view = base[:, 1:].detach().requires_grad_(True)
    assert view.stride(0) == 4 * 336 * 336
    _backward(t.hidden_states(view), d_outs)
    assert torch.equal(view.grad, g32)


def test_hd_batch_231_crops(weights):
    """231 crops (the HD batch: 133k patch rows, split-K weight gradients), the whole tower training with checkpointing: every
    parameter gradient keeps its bits, and the gradient of the first and last crops matches fp64."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    n = 231
    model = _model(weights, layers=True, embed=True)
    model.gradient_checkpointing = True
    t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    images = cto.make_images(n, seed=80, device=DEV).bfloat16().float()
    d_outs = _d_outs(n, 81)
    _backward(t.hidden_states(images), d_outs)
    plain = _param_grads(model)
    model.zero_grad(set_to_none=True)
    t.input_grad = True
    got = _crop_step(t, images, d_outs)
    after = _param_grads(model)
    assert after.keys() == plain.keys() and all(torch.equal(after[k], plain[k]) for k in plain)
    assert torch.isfinite(got).all()
    pick = [0, 1, n - 2, n - 1]
    ref = _oracle(weights, images[pick], {j: d[pick] for j, d in d_outs.items()})
    err = _rel(got[pick], ref)
    print(f"N=231: d(crops) rel-RMS {err:.2e} on crops {pick}")
    assert err < GATE, err


HD_SIZES = [(500, 300), (336, 336), (120, 900), (1000, 620)]


def _hd_images(seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(3, h, w, generator=g, device=DEV) for h, w in HD_SIZES]


def test_hd_tile_backward_against_fp64_and_per_image():
    from tokenpacker_b200 import hd
    images = [im.requires_grad_(True) for im in _hd_images(90)]
    crops, hb, wb = hd.hd_tile_batch(images, patch_num=9)
    with torch.no_grad():
        plain, hb0, wb0 = hd.hd_tile_batch([im.detach() for im in images], patch_num=9)
    assert torch.equal(crops.detach(), plain) and (hb, wb) == (hb0, wb0) and crops.requires_grad
    d = torch.randn(crops.shape, generator=torch.Generator(device=DEV).manual_seed(91), device=DEV)
    crops.backward(d)
    want = cgo.tile_gradients(images, d.cpu(), 9)
    c0 = 0
    for im, ref, b_h, b_w in zip(images, want, hb, wb):
        err = _rel(im.grad.cpu(), ref)
        assert im.grad.dtype == torch.float32 and err < 1e-4, (tuple(im.shape), err)
        single = im.detach().clone().requires_grad_(True)
        c, h1, w1 = hd.hd_tile(single, patch_num=9)
        assert (h1, w1) == (b_h, b_w)
        nc = c.shape[0]
        c.backward(d[c0:c0 + nc])
        assert torch.equal(single.grad, im.grad), tuple(im.shape)
        c0 += nc
    again = [im.detach().clone().requires_grad_(True) for im in images]
    hd.hd_tile_batch(again, patch_num=9)[0].backward(d)
    assert all(torch.equal(a.grad, b.grad) for a, b in zip(again, images))


def test_end_to_end_image_gradient_through_the_projector(weights):
    """two images -> hd_tile_batch -> tower -> forward_hidden_states_packed -> loss: image.grad against the fp64 chain (the tower's and
    the tiling's oracles, fed the hidden-state gradients the projector's own backward gives)."""
    from oracle import tokenpacker_oracle as tpo
    from tokenpacker_b200 import CLIPVisionTowerB200, TokenPackerB200, hd
    hidden = 256
    params = {k: tpo.round_bf16(v) for k, v in tpo.make_params(hidden, seed=1).items()}
    proj = TokenPackerB200(hidden_size=hidden, scale_factor=2)
    proj.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    proj = proj.to(DEV, torch.bfloat16)
    proj.requires_grad_(False)
    proj.input_grad = True
    tower = CLIPVisionTowerB200(_model(weights))
    tower.input_grad = True
    g = torch.Generator(device=DEV).manual_seed(95)
    images = [torch.randn(3, 200, 150, generator=g, device=DEV).requires_grad_(True),
              torch.randn(3, 90, 300, generator=g, device=DEV).requires_grad_(True)]
    crops, hb, wb = hd.hd_tile_batch(images, patch_num=9)
    crops.retain_grad()
    hs = tower.hidden_states(crops)
    d_hs = [None] * 4
    for i, h in enumerate(hs):
        h.register_hook(lambda grad, i=i: d_hs.__setitem__(i, grad.detach().clone()))
    sep = torch.randn(hidden, generator=g, device=DEV).bfloat16()
    ret = torch.randn(hidden, generator=g, device=DEV).bfloat16()
    packed, _ = proj.forward_hidden_states_packed(hs, hb, wb, sep, ret)
    packed.float().square().mean().backward()
    torch.cuda.synchronize()
    d_outs = {j: d for j, d in zip(cto.OUT_LAYERS, d_hs)}
    d_crops = _oracle(weights, crops.detach(), d_outs)
    assert _rel(crops.grad, d_crops) < GATE
    want = cgo.tile_gradients(images, d_crops.cpu(), 9)
    for im, ref in zip(images, want):
        err = _rel(im.grad.cpu(), ref)
        print(f"end to end: image {tuple(im.shape)} d(image) rel-RMS {err:.2e}")
        assert err < GATE, err


def test_launch_count(weights):
    """The pixel-gradient step adds the crop-gradient GEMM and the col2im store to the whole-tower step (and, on the HD path, the
    tiling backward); it keeps the step's workspace."""
    from tokenpacker_b200 import CLIPVisionTowerB200, _lib, hd
    lib = _lib.lib
    model = _model(weights, layers=True, embed=True)
    t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    n = 2
    images = cto.make_images(n, seed=100, device=DEV).bfloat16().float()
    d_outs = _d_outs(n, 101)
    model.requires_grad_(False)
    counts = {}
    for crop_grad in (False, True):
        t.input_grad = crop_grad
        x = images.detach().clone().requires_grad_(crop_grad)
        if not crop_grad:
            for name, p in model.named_parameters():                  # the whole-tower step without crop gradients: all layers, no wgrads
                p.requires_grad_("pre_layrnorm" in name)
        outs = t.hidden_states(x)
        torch.cuda.synchronize()
        c0 = lib.tp_launch_count()
        _backward(outs, d_outs)
        counts[crop_grad] = lib.tp_launch_count() - c0
        model.requires_grad_(False)
    # without crop gradients: pre_layrnorm's backward and its parameter reduction; with them (no parameter gradient): pre_layrnorm's
    # backward, the dgrad GEMM and the col2im store
    assert counts[True] == counts[False] + 1, counts
    image = torch.randn(3, 500, 300, device=DEV, requires_grad=True)
    crops = hd.hd_tile_batch([image])[0]
    torch.cuda.synchronize()
    c0 = lib.tp_launch_count()
    crops.backward(torch.ones_like(crops))
    torch.cuda.synchronize()
    assert lib.tp_launch_count() - c0 == 1
