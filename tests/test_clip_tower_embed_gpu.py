"""Training the whole CLIP tower on the GPU (``CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)``,
include/tokenpacker_b200_clip_tower_embed.h): all 373 parameter gradients against the fp64 autograd oracle; the outputs and the 368
layer gradients have the bits of the 23-layer step without the embedding stage; checkpointing, repetition, None output gradients and
accumulation change no bits; frozen layers and frozen embedding parameters; launches and memory; composition with the preprocessing
and the projector."""
import pytest
import torch

from oracle import clip_tower_embed_oracle as cte
from oracle import clip_tower_oracle as cto
from oracle import clip_tower_train_oracle as ctt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MiB = 1 << 20
GATE = 1.5e-2                                               # rel-RMS per gradient tensor, as for the layers (DESIGN.md §9.1)
GATE_QK = 2.5e-2                                            # q_proj / k_proj: the reason is in DESIGN.md §9.1
EMBED_NAMES = ["vision_model." + k for k in cte.EMBED_KEYS]


@pytest.fixture(scope="module")
def weights():
    return cto.round_bf16(cto.make_weights(23, seed=11, device=DEV))


def _model(w, layers=True, embed=True):
    model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    for name, p in model.named_parameters():
        p.requires_grad_(layers if "encoder.layers." in name else embed)
    return model


def _grads(model):
    return {name: None if p.grad is None else p.grad.clone() for name, p in model.named_parameters() if p.requires_grad}


def _clear(model):
    for p in model.parameters():
        p.grad = None


def _backward(outs, d_outs):
    pairs = [(o, d_outs[j]) for o, j in zip(outs, cto.OUT_LAYERS) if d_outs[j] is not None and o.requires_grad]
    torch.autograd.backward([o for o, _ in pairs], [d for _, d in pairs])
    torch.cuda.synchronize()


def _d_outs(n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return {j: (torch.randn(n, 577, 1024, generator=g, device=DEV) * 0.1).bfloat16() for j in cto.OUT_LAYERS}


def _rel(got, ref):
    ref = ref.double()
    return float((got.double() - ref).norm() / ref.norm().clamp_min(1e-300))


def _oracle(w, images, d_outs):
    d = {j: None if v is None else v.double() for j, v in d_outs.items()}
    n = images.shape[0]
    if n <= 3:
        eg, lg, _ = cte.parameter_gradients(w, images.double(), d, device=DEV)
    else:
        eg, lg = cte.parameter_gradients_chunked(w, images.double(), d, chunk=4, device=DEV)
    return eg, lg


@pytest.mark.parametrize("n", [1, 3, 29], ids=["N1", "N3", "N29-splitk"])
def test_all_373_gradients_against_fp64_oracle(weights, n):
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _model(weights)
    t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    images = cto.make_images(n, seed=40 + n, device=DEV).bfloat16()
    d_outs = _d_outs(n, 50 + n)
    _backward(t.hidden_states(images), d_outs)
    got = _grads(model)
    assert len(got) == 373 and all(v is not None for v in got.values())
    eg, lg = _oracle(weights, images, d_outs)
    errors = {}
    for key, name in zip(cte.EMBED_KEYS, EMBED_NAMES):
        errors[name] = _rel(got[name], eg[key])
        assert errors[name] < GATE, (name, errors[name])
    assert torch.equal(got[EMBED_NAMES[1]], got[EMBED_NAMES[2]][0])              # d class_embedding = d position_embedding[0], bitwise
    for i in range(23):
        keys = cto.layer_keys(i)
        for key in ctt.PARAM_KEYS:
            name = "vision_model." + keys[key]
            if key == "self_attn.k_proj.bias":                                     # exact gradient 0: measured against v_proj.bias's
                err = float((got[name].double() - lg[i][key]).norm() / lg[i]["self_attn.v_proj.bias"].norm())
            else:
                err = _rel(got[name], lg[i][key])
            errors[name] = err
            assert err < (GATE_QK if "q_proj" in key or "k_proj" in key else GATE), (name, err)
    print(f"N={n}: embedding stage rel-RMS " + ", ".join(f"{k.split('.')[-2]}.{k.split('.')[-1]} {errors[k]:.2e}" for k in EMBED_NAMES) +
          f"; worst layer gradient {max(v for k, v in errors.items() if k not in EMBED_NAMES):.2e}")


@pytest.mark.parametrize("n", [2, 29], ids=["N2", "N29-splitk"])
def test_bits_against_the_layers_only_step_checkpointing_repetition_accumulation(weights, n):
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _model(weights)
    full = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    layers_only = CLIPVisionTowerB200(model, trainable_layers=23)
    images = cto.make_images(n, seed=60 + n, device=DEV).bfloat16()
    with torch.no_grad():
        ref_outs = CLIPVisionTowerB200(model).hidden_states(images)
    d_outs = _d_outs(n, 70 + n)
    d_outs[16] = None                                                                 # an output the loss does not use

    def step(tower, checkpointing):
        _clear(model)
        model.gradient_checkpointing = checkpointing
        outs = tower.hidden_states(images)
        for a, b, j in zip(outs, ref_outs, cto.OUT_LAYERS):
            assert torch.equal(a, b) and a.requires_grad, j
        assert outs[3].grad_fn.checkpoint == checkpointing
        _backward(outs, d_outs)
        return _grads(model)

    plain = step(full, False)
    assert len(plain) == 373 and all(v is not None for v in plain.values())
    ckpt = step(full, True)
    again = step(full, True)
    base = step(layers_only, False)
    for name in plain:
        assert torch.equal(ckpt[name], plain[name]) and torch.equal(again[name], plain[name]), name
    for name, g in base.items():                                                     # the layers' gradients do not depend on the option
        assert (name in EMBED_NAMES) == (g is None), name
        if g is not None:
            assert torch.equal(g, plain[name]), name
    step(full, True)
    outs = full.hidden_states(images)                                                 # accumulates like any autograd gradient
    _backward(outs, d_outs)
    for name, p in model.named_parameters():
        assert torch.equal(p.grad, 2 * plain[name]), name


def test_frozen_layers_and_frozen_embedding_parameters(weights):
    """Every layer frozen, the embeddings trainable: the embedding gradients have the bits of the all-trainable step and no layer gets
    a gradient.  Then one embedding parameter frozen as well: it gets None, the others keep their bits."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    n = 3
    images = cto.make_images(n, seed=81, device=DEV).bfloat16()
    d_outs = _d_outs(n, 82)
    model = _model(weights)
    t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    _backward(t.hidden_states(images), d_outs)
    ref = _grads(model)
    model = _model(weights, layers=False)
    t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    outs = t.hidden_states(images)
    assert all(o.requires_grad for o in outs)
    _backward(outs, d_outs)
    for name, p in model.named_parameters():
        if name in EMBED_NAMES:
            assert torch.equal(p.grad, ref[name]), name
        else:
            assert p.grad is None, name
    _clear(model)
    named = dict(model.named_parameters())
    named[EMBED_NAMES[2]].requires_grad_(False)                                       # position_embedding frozen
    _backward(t.hidden_states(images), d_outs)
    assert named[EMBED_NAMES[2]].grad is None
    for name in EMBED_NAMES[:2] + EMBED_NAMES[3:]:
        assert torch.equal(named[name].grad, ref[name]), name
    # every trainable parameter frozen: the forward is the inference path again, with no graph
    for name in EMBED_NAMES:
        named[name].requires_grad_(False)
    assert not any(o.requires_grad for o in t.hidden_states(images))


def test_launches_and_memory(weights):
    """The whole-tower step launches exactly the 23-layer step's kernels plus five for the embedding stage (the saved copies are not
    kernels), and keeps exactly one more tensor, the embedding saved set, on top of the 23-layer step's saved sets or checkpoints, in
    both modes.
    Without the option nothing of it runs: same launches, same bytes."""
    from tokenpacker_b200 import CLIPVisionTowerB200, _lib
    lib = _lib.lib
    n = 4
    images = cto.make_images(n, seed=83, device=DEV).bfloat16()
    d_outs = _d_outs(n, 84)
    model = _model(weights)
    towers = {False: CLIPVisionTowerB200(model, trainable_layers=23), True: CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)}
    embed_bytes = lib.tp_clip_tower_embed_saved_bytes(n)
    out_bytes = 4 * n * 577 * 1024 * 2
    for checkpointing in (False, True):
        model.gradient_checkpointing = checkpointing
        saved_bytes = (lib.tp_clip_tower_ckpt_saved_bytes if checkpointing else lib.tp_clip_tower_train_saved_bytes)(n, 23)
        counts, kept = {}, {}
        for embed, t in towers.items():
            _clear(model)
            _backward(t.hidden_states(images), d_outs)                                # warm-up: derived cache and allocator
            _clear(model)
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            start = torch.cuda.memory_allocated()
            c0 = lib.tp_launch_count()
            outs = t.hidden_states(images)
            torch.cuda.synchronize()
            c1 = lib.tp_launch_count()
            kept[embed] = torch.cuda.memory_allocated() - start
            fn = outs[3].grad_fn
            assert fn.saved.numel() == saved_bytes
            assert (fn.embed_saved is not None) == embed and (not embed or fn.embed_saved.numel() == embed_bytes)
            _backward(outs, d_outs)
            counts[embed] = (c1 - c0, lib.tp_launch_count() - c1)
            del outs, fn
        assert counts[True][0] == counts[False][0], counts
        assert counts[True][1] == counts[False][1] + 5, counts
        assert saved_bytes + out_bytes <= kept[False] <= saved_bytes + out_bytes + MiB, kept
        # the allocator hands out large blocks in 2 MiB steps: the one extra tensor is embed_bytes, rounded up to the next step
        assert embed_bytes <= kept[True] - kept[False] < embed_bytes + 2 * MiB, (kept, embed_bytes)


def test_uint8_images_through_preprocessing_tower_and_projector(weights):
    """Decoded images -> hd_preprocess_batch -> the whole tower (checkpointing on, embeddings trainable) -> packed projector output with
    input_grad -> loss -> backward: the embedding stage's gradients agree with the fp64 oracle driven by the same four hidden-state
    gradients."""
    from tokenpacker_b200 import CLIPVisionTowerB200, TokenPackerB200, hd_preprocess_batch
    g = torch.Generator(device=DEV).manual_seed(91)
    images = [torch.randint(0, 256, (h_, w_, 3), generator=g, device=DEV, dtype=torch.uint8) for h_, w_ in ((336, 336), (400, 600))]
    torch.manual_seed(7)
    proj = TokenPackerB200(hidden_size=1024, scale_factor=2).to(DEV, torch.bfloat16).train()
    proj.input_grad = True
    sep, ret = torch.randn(1024, device=DEV).bfloat16(), torch.randn(1024, device=DEV).bfloat16()
    model = _model(weights)
    model.gradient_checkpointing = True
    t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    with torch.no_grad():
        crops, hb, wb = hd_preprocess_batch(images, patch_num=9, dtype=torch.bfloat16)
    hs = t.hidden_states(crops)
    assert hs[3].grad_fn.checkpoint
    for h in hs:
        h.retain_grad()
    proj.forward_hidden_states_packed(list(hs), hb, wb, sep, ret)[0].float().square().mean().backward()
    torch.cuda.synchronize()
    d_outs = {j: h.grad for j, h in zip(cto.OUT_LAYERS, hs)}
    assert all(d is not None for d in d_outs.values())
    eg, _ = _oracle(weights, crops, d_outs)
    named = dict(model.named_parameters())
    for key, name in zip(cte.EMBED_KEYS, EMBED_NAMES):
        err = _rel(named[name].grad, eg[key])
        assert err < GATE, (name, err)
