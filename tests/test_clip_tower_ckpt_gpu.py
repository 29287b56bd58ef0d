"""Gradient checkpointing for the CLIP tower's trainable layers on the GPU (include/tokenpacker_b200_clip_tower_ckpt.h, chosen by the
wrapped model's ``gradient_checkpointing`` switch): the outputs have the inference bits and every parameter gradient the bits of the
non-checkpointed step; the mode is fixed when the graph is built; what is kept between forward and backward and the step's peak memory;
composition with the preprocessing and the projector."""
import pytest
import torch

from oracle import clip_tower_oracle as cto

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MiB = 1 << 20


@pytest.fixture(scope="module")
def weights():
    return cto.round_bf16(cto.make_weights(23, seed=11, device=DEV))


def _model(w, trainable_from):
    model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    for name, p in model.named_parameters():
        if "encoder.layers." in name and int(name.split("encoder.layers.")[1].split(".")[0]) >= trainable_from:
            p.requires_grad_(True)
    return model


def _grads(model):
    return {name: None if p.grad is None else p.grad.clone() for name, p in model.named_parameters() if p.requires_grad}


def _clear(model):
    for p in model.parameters():
        p.grad = None


def _backward(outs, d_outs):
    """d(sum_j <hidden_states[j], d_outs[j]>) without materialising the products: the four gradients go straight to autograd."""
    pairs = [(o, d_outs[j]) for o, j in zip(outs, cto.OUT_LAYERS) if d_outs[j] is not None and o.requires_grad]
    torch.autograd.backward([o for o, _ in pairs], [d for _, d in pairs])
    torch.cuda.synchronize()


@pytest.mark.parametrize("n,k", [(2, 1), (2, 3), (2, 23), (29, 2)], ids=["N2-K1", "N2-K3", "N2-K23", "N29-K2-splitk"])
def test_checkpointed_step_has_the_bits_of_the_plain_step(weights, n, k):
    from tokenpacker_b200 import CLIPVisionTowerB200
    first = 23 - k
    model = _model(weights, first)
    frozen = []
    if k == 3:                                                                        # parameters frozen inside a trainable layer get None
        named = dict(model.named_parameters())
        frozen = ["vision_model." + cto.layer_keys(21)[key] for key in ("mlp.fc1.weight", "self_attn.q_proj.bias", "layer_norm2.weight")]
        for name in frozen:
            named[name].requires_grad_(False)
    t = CLIPVisionTowerB200(model, trainable_layers=k)
    images = cto.make_images(n, seed=60 + n, device=DEV).bfloat16()
    with torch.no_grad():
        ref_outs = CLIPVisionTowerB200(model).hidden_states(images)
    g = torch.Generator(device=DEV).manual_seed(70 + k)
    d_outs = {j: (torch.randn(n, 577, 1024, generator=g, device=DEV) * 0.1).bfloat16() for j in cto.OUT_LAYERS}
    d_outs[16] = None                                                                 # an output the loss does not use

    def step(checkpointing):
        model.gradient_checkpointing = checkpointing
        outs = t.hidden_states(images)
        for a, b, j in zip(outs, ref_outs, cto.OUT_LAYERS):
            assert torch.equal(a, b), j
            assert a.requires_grad == (j - 1 >= first), j
        assert outs[3].grad_fn.checkpoint == checkpointing
        _backward(outs, d_outs)

    step(False)
    plain = _grads(model)
    _clear(model)
    step(True)
    ckpt = _grads(model)
    assert set(plain) == set(ckpt) and len(ckpt) == 16 * k - len(frozen)
    for name in plain:
        assert plain[name] is not None and torch.equal(ckpt[name], plain[name]), name
    for name, p in model.named_parameters():
        if not p.requires_grad:
            assert p.grad is None, name
    step(True)                                                                        # accumulates like any autograd gradient
    for name, p in model.named_parameters():
        if p.requires_grad:
            assert torch.equal(p.grad, 2 * ckpt[name]), name


def test_mode_is_fixed_when_the_graph_is_built(weights):
    from tokenpacker_b200 import CLIPVisionTowerB200, _lib
    lib = _lib.lib
    n, k = 2, 2
    model = _model(weights, 23 - k)
    t = CLIPVisionTowerB200(model, trainable_layers=k)
    images = cto.make_images(n, seed=85, device=DEV).bfloat16()
    g = torch.Generator(device=DEV).manual_seed(86)
    d_outs = {j: (torch.randn(n, 577, 1024, generator=g, device=DEV) * 0.1).bfloat16() for j in cto.OUT_LAYERS}
    with torch.no_grad():
        t.hidden_states(images)                                                       # derived cache built
        c0 = lib.tp_launch_count()
        t.hidden_states(images)
        torch.cuda.synchronize()
        inference_launches = lib.tp_launch_count() - c0

    def step(on_forward, on_backward):
        _clear(model)
        model.gradient_checkpointing = on_forward
        c0 = lib.tp_launch_count()
        outs = t.hidden_states(images)
        torch.cuda.synchronize()
        c1 = lib.tp_launch_count()
        model.gradient_checkpointing = on_backward
        _backward(outs, d_outs)
        return c1 - c0, lib.tp_launch_count() - c1, _grads(model), outs

    fwd_on, bwd_on, grads_on, outs = step(True, True)
    saved = outs[3].grad_fn.saved
    assert saved.numel() == lib.tp_clip_tower_ckpt_saved_bytes(n, k)                  # checkpoints only between forward and backward
    fwd_plain, bwd_plain, grads_plain, _ = step(False, False)
    fwd_switched, bwd_switched, grads_switched, _ = step(True, False)                 # switched off between forward and backward
    # the checkpointed forward is the inference schedule plus packing each trainable layer's derived weights (two launches per layer)
    assert fwd_on == fwd_switched == inference_launches + 2 * k
    assert fwd_plain != fwd_on
    # the backward follows the forward's mode: the recompute's launches on top of the plain backward's
    assert bwd_switched == bwd_on > bwd_plain
    for name in grads_on:
        assert torch.equal(grads_switched[name], grads_on[name]) and torch.equal(grads_plain[name], grads_on[name]), name
    # and the other way round: switched on after a plain forward, the backward stays plain
    _, bwd_late, grads_late, _ = step(False, True)
    assert bwd_late == bwd_plain and all(torch.equal(grads_late[name], grads_on[name]) for name in grads_on)


def test_checkpointed_step_memory(weights):
    """29 crops, 12 trainable layers.  Between forward and backward the step keeps the checkpoints and the four outputs; its peak adds
    the backward's workspace and the parameter gradients the backward returns (16 tensors per layer, 302 MB at K = 12).  Both are well
    below the non-checkpointed step's peak, measured here too."""
    from tokenpacker_b200 import CLIPVisionTowerB200, _lib
    lib = _lib.lib
    n, k = 29, 12
    model = _model(weights, 23 - k)
    t = CLIPVisionTowerB200(model, trainable_layers=k)
    images = cto.make_images(n, seed=87, device=DEV).bfloat16()
    g = torch.Generator(device=DEV).manual_seed(88)
    d_outs = {j: (torch.randn(n, 577, 1024, generator=g, device=DEV) * 0.1).bfloat16() for j in cto.OUT_LAYERS}
    out_bytes = n * 577 * 1024 * 2
    param_grad_bytes = sum(p.numel() * p.element_size() for p in model.parameters() if p.requires_grad)
    saved_bytes = lib.tp_clip_tower_ckpt_saved_bytes(n, k)
    bound = saved_bytes + lib.tp_clip_tower_ckpt_backward_workspace_bytes(n, k) + 2 * 4 * out_bytes + param_grad_bytes + 64 * MiB
    peaks = {}
    for checkpointing in (False, True):
        model.gradient_checkpointing = checkpointing
        _clear(model)
        _backward(t.hidden_states(images), d_outs)                                    # warm-up: derived cache and allocator
        _clear(model)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        start = torch.cuda.memory_allocated()
        outs = t.hidden_states(images)
        torch.cuda.synchronize()
        kept = torch.cuda.memory_allocated() - start
        if checkpointing:
            assert outs[3].grad_fn.saved.numel() == saved_bytes
            assert saved_bytes + 4 * out_bytes <= kept <= saved_bytes + 4 * out_bytes + MiB, (kept, saved_bytes)
        else:
            assert outs[3].grad_fn.saved.numel() == lib.tp_clip_tower_train_saved_bytes(n, k)
        _backward(outs, d_outs)
        peaks[checkpointing] = torch.cuda.max_memory_allocated() - start
        del outs
    print(f"N={n} K={k}: peak above start {peaks[True] / 1e9:.2f} GB checkpointed (bound {bound / 1e9:.2f} GB), "
          f"{peaks[False] / 1e9:.2f} GB not; checkpoints {saved_bytes / 1e9:.2f} GB")
    assert peaks[True] < bound
    assert peaks[True] < peaks[False]


def test_uint8_images_through_tower_and_projector_backward(weights):
    """Decoded images -> hd_preprocess_batch -> tower (last 2 layers trainable, checkpointing on) -> packed projector output with
    input_grad -> loss -> backward: the tower's and the projector's gradients have the bits of the same chain without checkpointing."""
    from tokenpacker_b200 import CLIPVisionTowerB200, TokenPackerB200, hd_preprocess_batch
    g = torch.Generator(device=DEV).manual_seed(91)
    images = [torch.randint(0, 256, (h_, w_, 3), generator=g, device=DEV, dtype=torch.uint8) for h_, w_ in ((336, 336), (400, 600))]
    torch.manual_seed(7)
    proj = TokenPackerB200(hidden_size=1024, scale_factor=2).to(DEV, torch.bfloat16).train()
    proj.input_grad = True
    sep, ret = torch.randn(1024, device=DEV).bfloat16(), torch.randn(1024, device=DEV).bfloat16()
    model = _model(weights, 21)
    t = CLIPVisionTowerB200(model, trainable_layers=2)
    with torch.no_grad():
        crops, hb, wb = hd_preprocess_batch(images, patch_num=9, dtype=torch.bfloat16)

    def chain(checkpointing):
        model.gradient_checkpointing = checkpointing
        _clear(model)
        for p in proj.parameters():
            p.grad = None
        hs = t.hidden_states(crops)
        assert hs[3].grad_fn.checkpoint == checkpointing
        proj.forward_hidden_states_packed(list(hs), hb, wb, sep, ret)[0].float().square().mean().backward()
        torch.cuda.synchronize()
        tower = _grads(model)
        projector = {name: p.grad.clone() for name, p in proj.named_parameters() if p.grad is not None}
        return tower, projector

    tower_plain, proj_plain = chain(False)
    tower_ckpt, proj_ckpt = chain(True)
    assert proj_plain and set(proj_plain) == set(proj_ckpt)
    assert len(tower_plain) == 32 and all(v is not None for v in tower_plain.values())
    for name in tower_plain:
        assert torch.equal(tower_ckpt[name], tower_plain[name]), name
    for name in proj_plain:
        assert torch.equal(proj_ckpt[name], proj_plain[name]), name
