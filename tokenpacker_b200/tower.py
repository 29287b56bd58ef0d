"""The frozen CLIP-ViT-L/14-336 vision tower on the sm_90a kernels (include/tokenpacker_b200_clip_tower.h).

``CLIPVisionTowerB200(clip_vision_model).hidden_states(crops)`` returns hidden states 12, 16, 22 and 23 of transformers'
``CLIPVisionModel`` — exactly what ``TokenPackerB200.forward_hidden_states`` takes — without running layer 23 or post_layernorm
and without keeping the other 21 hidden states alive.  The reference's ``encode_images`` becomes

    proj.forward_hidden_states(tower.hidden_states(crops))          # or forward_hidden_states_packed for the HD 'slice' path

transformers is never imported: any module with CLIPVisionModel's parameter names (with or without the ``vision_model.`` prefix)
and a ``.config`` carrying its fields is accepted.

``CLIPVisionTowerB200(model, dtype=torch.float16)`` runs the tower in fp16, as the reference's evaluation and serving scripts do
(``vision_tower.to(dtype=torch.float16)``, llava/eval/model_vqa_loader.py): the hidden states come back fp16, and the caller casts them
to bf16 for the projector as clip_encoder.py does (``[h.to(torch.bfloat16) for h in hs]``).

``CLIPVisionTowerB200(model, trainable_layers=K)`` trains the last K encoder layers (include/tokenpacker_b200_clip_tower_train.h):
under ``torch.enable_grad()`` the four hidden states are attached to autograd, and their backward writes the gradients of the
parameters of layers 23 - K .. 22 that require grad.  With the projector's ``input_grad`` this closes the loop:

    tower = CLIPVisionTowerB200(vision_tower, trainable_layers=4)
    proj.input_grad = True
    proj.forward_hidden_states(tower.hidden_states(crops)).float().square().mean().backward()

When the wrapped model asks for gradient checkpointing (``vision_tower.gradient_checkpointing_enable()``, as the reference's recipes
do with ``--gradient_checkpointing True``), that training step keeps only each trainable layer's input and derived weights and
recomputes the rest in the backward (include/tokenpacker_b200_clip_tower_ckpt.h): less memory, more time, the same bits.

``CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)`` trains the whole tower: below the 23 layers, pre_layrnorm, the
class and position embeddings and the patch embedding get their gradients too (include/tokenpacker_b200_clip_tower_embed.h), with or
without gradient checkpointing.  That is what the recipes that unfreeze the vision tower (``vision_tower.requires_grad_(True)``) need.

``tower.input_grad = True`` backpropagates to the pixels: crops that require grad get their gradient (adversarial evaluation,
attribution of packed tokens to image regions, pixel-space perturbation learning); with ``hd_tile_batch`` the gradient reaches the
normalised images (INTEGRATION.md).
"""
from __future__ import annotations

import ctypes as C
import warnings

import torch
from torch import nn

from . import _lib
from ._lib import check, lib

_TOKENS = 577
_IMAGE = 336
_OUT_LAYERS = (12, 16, 22, 23)


_NUM_FN_INPUTS = 6                                      # _TowerTrainFunction's inputs before the parameters


def _train_step(checkpoint: bool, embed: bool, crop_grad: bool, n: int, k: int):
    """The entry points and buffer sizes of a training step over n crops that runs the top k layers: (forward, backward, saved bytes,
    forward workspace bytes, backward workspace bytes).  checkpoint: keep each layer's checkpoint (include/tokenpacker_b200_clip_tower_ckpt.h)
    instead of its full saved set; embed: the whole tower, k = 23 and the embedding stage (include/tokenpacker_b200_clip_tower_embed.h);
    crop_grad: the whole tower's backward gives the crops their gradient too (include/tokenpacker_b200_clip_tower_crop_grad.h)."""
    if checkpoint:
        names = ("tp_clip_tower_forward_ckpt", "tp_clip_tower_backward_ckpt")
        sizes = (lib.tp_clip_tower_ckpt_saved_bytes(n, k), lib.tp_clip_tower_workspace_bytes(n),
                 lib.tp_clip_tower_ckpt_backward_workspace_bytes(n, k))
    else:
        names = ("tp_clip_tower_forward_train", "tp_clip_tower_backward")
        sizes = (lib.tp_clip_tower_train_saved_bytes(n, k), lib.tp_clip_tower_train_workspace_bytes(n, k),
                 lib.tp_clip_tower_backward_workspace_bytes(n, k))
    if embed:
        names = ("tp_clip_tower_forward_train_embed", "tp_clip_tower_backward_crops" if crop_grad else "tp_clip_tower_backward_embed")
    return names + sizes


class _TowerTrainFunction(torch.autograd.Function):
    """hidden_states 12 / 16 / 22 / 23 under autograd, in every training mode of the tower.  Inputs after the first six are the 16 K
    parameters of the trainable layers, in _lib.CLIP_TOWER_LAYER_FIELDS order, layer 23 - K first; with ``tower.train_embeddings``
    (K = 23) the five embedding-stage parameters, in _lib.CLIP_TOWER_FIELDS order, come before them.  checkpoint: keep only each run
    layer's checkpoint instead of its full saved set; the backward follows the forward's mode.  crop_grad (``tower.input_grad``): all
    23 layers and the embedding stage run whatever K, every layer below the trainable ones only passes its input gradient on, and the
    crops get their gradient.  ``images`` are the caller's crops: they are cast to bf16 here, so that fp32 crops receive the fp32
    gradient the kernels accumulate."""

    @staticmethod
    def forward(ctx, tower, images, packed, w, checkpoint, crop_grad, *params):
        n, device = images.shape[0], images.device
        embed = crop_grad or tower.train_embeddings
        k = _lib.CLIP_TOWER_LAYERS if embed else tower.trainable_layers          # the layers the step runs and keeps
        x = images.to(torch.bfloat16)
        if not (x.stride(3) == 1 and x.stride(2) == _IMAGE and x.stride(1) == _IMAGE * _IMAGE and x.stride(0) >= 3 * _IMAGE * _IMAGE):
            x = x.contiguous()
        fwd_name, ctx.bwd_name, saved_bytes, ws_bytes, ctx.bwd_ws_bytes = _train_step(checkpoint, embed, crop_grad, n, k)
        outs = tuple(torch.empty((n, _TOKENS, 1024), dtype=torch.bfloat16, device=device) for _ in _OUT_LAYERS)
        saved = torch.empty(saved_bytes, dtype=torch.uint8, device=device)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        embed_saved = None
        ptrs = (C.c_void_p * 4)(*[o.data_ptr() for o in outs])
        args = (packed.data_ptr(), C.byref(w), x.data_ptr(), n, x.stride(0))
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            if embed:
                embed_bytes = lib.tp_clip_tower_embed_saved_bytes(n)
                embed_saved = torch.empty(embed_bytes, dtype=torch.uint8, device=device)
                status = getattr(lib, fwd_name)(*args, int(checkpoint), ptrs, saved.data_ptr(), saved_bytes, embed_saved.data_ptr(), embed_bytes,
                                                ws.data_ptr(), ws_bytes, stream)
            else:
                status = getattr(lib, fwd_name)(*args, k, ptrs, saved.data_ptr(), saved_bytes, ws.data_ptr(), ws_bytes, stream)
            check(status, fwd_name)
        ctx.w, ctx.saved, ctx.embed_saved, ctx.k, ctx.n, ctx.checkpoint, ctx.crop_grad = w, saved, embed_saved, k, n, checkpoint, crop_grad
        ctx.trainable_layers, ctx.train_embeddings, ctx.params = tower.trainable_layers, tower.train_embeddings, params
        ctx.crops_dtype = images.dtype
        ctx.set_materialize_grads(False)                # an output nobody used arrives as None, not as a tensor of zeros
        # hidden_states[j] is the output of layer j - 1: below the first layer run (23 - k) nothing of it depends on a trainable parameter
        frozen = [o for o, j in zip(outs, _OUT_LAYERS) if j - 1 < _lib.CLIP_TOWER_LAYERS - k]
        ctx.mark_non_differentiable(*frozen)
        return outs

    @staticmethod
    def backward(ctx, *d_outs):
        k, n, device = ctx.k, ctx.n, ctx.saved.device
        d_outs = [None if g is None else g.to(torch.bfloat16).contiguous() for g in d_outs]
        d_ptrs = (C.c_void_p * 4)(*[None if g is None else g.data_ptr() for g in d_outs])
        grads = [torch.empty_like(p) if ctx.needs_input_grad[_NUM_FN_INPUTS + i] else None for i, p in enumerate(ctx.params)]
        ptr = [None if g is None else g.data_ptr() for g in grads]
        n_top = len(_lib.CLIP_TOWER_FIELDS) if ctx.train_embeddings else 0
        per, first = len(_lib.CLIP_TOWER_LAYER_FIELDS), k - ctx.trainable_layers
        g_structs = (_lib.TpClipTowerLayerGrads * k)()
        for t in range(ctx.trainable_layers):
            g_structs[first + t] = _lib.TpClipTowerLayerGrads(*ptr[n_top + t * per:n_top + (t + 1) * per])
        f32 = ctx.crops_dtype == torch.float32
        d_crops = None
        if ctx.crop_grad:
            d_crops = torch.empty((n, 3, _IMAGE, _IMAGE), dtype=torch.float32 if f32 else torch.bfloat16, device=device)
        bwd_name, ws_bytes = ctx.bwd_name, ctx.bwd_ws_bytes
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            if ctx.embed_saved is None:
                status = getattr(lib, bwd_name)(C.byref(ctx.w), ctx.saved.data_ptr(), n, k, d_ptrs, g_structs, ws.data_ptr(), ws_bytes, stream)
            else:
                e_struct = _lib.TpClipTowerEmbedGrads(*ptr[:n_top])
                args = (C.byref(ctx.w), ctx.saved.data_ptr(), ctx.embed_saved.data_ptr(), n, int(ctx.checkpoint), d_ptrs, g_structs,
                        C.byref(e_struct))
                if d_crops is not None:
                    args += (d_crops.data_ptr(), _lib.TP_CROP_GRAD_F32 if f32 else _lib.TP_CROP_GRAD_BF16, d_crops.stride(0))
                status = getattr(lib, bwd_name)(*args, ws.data_ptr(), ws_bytes, stream)
            check(status, bwd_name)
        if d_crops is not None and not f32 and ctx.crops_dtype != torch.bfloat16:
            d_crops = d_crops.to(ctx.crops_dtype)
        return (None, d_crops) + (None,) * (_NUM_FN_INPUTS - 2) + tuple(grads)


def wants_gradient_checkpointing(vision_model: nn.Module) -> bool:
    """Whether the wrapped model asks for gradient checkpointing: some submodule has ``gradient_checkpointing`` truthy and is in
    training mode.  That is the condition under which transformers' own CLIPEncoder recomputes its layers
    (``CLIPVisionModel.gradient_checkpointing_enable()`` sets ``encoder.gradient_checkpointing``), and
    ``PreTrainedModel.is_gradient_checkpointing`` is the same test over ``modules()``."""
    return any(bool(getattr(m, "gradient_checkpointing", False)) and m.training for m in vision_model.modules())


def _check_crops(images):
    if not isinstance(images, torch.Tensor) or images.dim() != 4 or tuple(images.shape[1:]) != (3, _IMAGE, _IMAGE):
        shape = tuple(images.shape) if isinstance(images, torch.Tensor) else type(images).__name__
        raise ValueError(f"expected crops [N,3,336,336], got {shape}")


def _check_config(cfg):
    want = {"hidden_size": 1024, "intermediate_size": 4096, "num_attention_heads": 16, "patch_size": 14, "image_size": 336,
            "hidden_act": "quick_gelu", "num_channels": 3}
    if cfg is None:
        raise NotImplementedError("the vision model has no .config: CLIP-ViT-L/14-336 (CLIPVisionConfig) is required")
    for key, value in want.items():
        got = getattr(cfg, key, None)
        if got != value:
            raise NotImplementedError(f"CLIPVisionTowerB200 runs CLIP-ViT-L/14-336 only: config.{key} = {got!r}, expected {value!r}")
    layers = getattr(cfg, "num_hidden_layers", 0)
    if not isinstance(layers, int) or layers < _lib.CLIP_TOWER_LAYERS:
        raise NotImplementedError(f"config.num_hidden_layers = {layers!r}: hidden_states[23] needs at least 23 layers")
    eps = getattr(cfg, "layer_norm_eps", None)
    if not isinstance(eps, float) or abs(eps - 1e-5) > 1e-12:
        raise NotImplementedError(f"config.layer_norm_eps = {eps!r}, expected 1e-5")


class CLIPVisionTowerB200(nn.Module):
    """Forward-only CLIPVisionModel (openai/clip-vit-large-patch14-336) up to hidden_states[23].

    dtype: the precision the tower computes in.  None (the default) or torch.bfloat16: bf16 storage, and fp16 / fp32 towers are cast
    to bf16 once, with a warning.  torch.float16: fp16 storage (fp16 parameters read in place, others cast to fp16 once), fp16 outputs.
    The wrapped model stays the owner of the parameters (``self.vision_model``).  A derived cache (about 147 MB: per layer the q/k/v
    concatenation — with q scaled by 1/8 in bf16 —, and the biases in fp32) is keyed on the compute precision and every parameter's
    ``(data_ptr, _version, dtype)``, and dropped by ``load_state_dict``, ``.to()`` / ``.cuda()`` / ``.half()`` and
    ``invalidate_packed()``.

    trainable_layers: K in 0 .. 23, bf16 only.  0 (the default): forward only.  K > 0: encoder layers 23 - K .. 22 are trainable: see
    ``hidden_states``.  Layers 0 .. 22 - K stay frozen whatever their ``requires_grad`` says: they get no gradient; so do the
    embeddings and pre_layrnorm unless ``train_embeddings``.

    train_embeddings: False (the default) or True, which needs trainable_layers = 23.  True: the embedding stage below layer 0 is
    trainable as well: the patch embedding, ``class_embedding``, ``position_embedding`` and pre_layrnorm's weight and bias, each of
    which requires grad gets its gradient.  A step trains when any of these five or of the 23 layers' parameters requires grad, so the
    embeddings can train with every layer frozen.  To train the embeddings below some frozen layers, keep trainable_layers = 23 and
    set ``requires_grad=False`` on those layers' parameters: the backward still runs through them (their input gradients), and skips
    their weight gradients.

    input_grad: False (the default) or True; an attribute, like ``TokenPackerB200.input_grad``, not a constructor argument and not in
    the state_dict, and refused with dtype=torch.float16 (the fp16 tower is forward only).  True: crops that require grad get their
    gradient under grad mode (see ``hidden_states``).

    Gradient checkpointing has no switch of its own: the tower follows the wrapped model's (``gradient_checkpointing_enable()`` /
    ``_disable()``, see ``wants_gradient_checkpointing``).  Checkpointing trades time for memory and no property of the input decides
    between them, so the choice stays with the switch the model and the recipe that sets it already own; a second option here could
    only disagree with it."""

    def __init__(self, vision_model: nn.Module, dtype: torch.dtype | None = None, trainable_layers: int = 0, train_embeddings: bool = False):
        super().__init__()
        if dtype not in (None, torch.bfloat16, torch.float16):
            raise ValueError(f"CLIPVisionTowerB200 computes in torch.bfloat16 (dtype=None) or torch.float16, not {dtype!r}")
        if not isinstance(trainable_layers, int) or isinstance(trainable_layers, bool) or not 0 <= trainable_layers <= _lib.CLIP_TOWER_LAYERS:
            raise ValueError(f"trainable_layers = {trainable_layers!r}: expected an int in 0 .. {_lib.CLIP_TOWER_LAYERS}")
        if not isinstance(train_embeddings, bool):
            raise ValueError(f"train_embeddings = {train_embeddings!r}: expected True or False")
        if train_embeddings and trainable_layers != _lib.CLIP_TOWER_LAYERS:
            raise ValueError(f"train_embeddings=True needs trainable_layers={_lib.CLIP_TOWER_LAYERS} (got {trainable_layers}): the embedding stage "
                             "sits below every layer; freeze layers with requires_grad=False instead")
        if trainable_layers > 0 and dtype == torch.float16:
            raise ValueError("trainable_layers > 0 needs the bf16 tower: no released recipe trains CLIP in fp16 (its gradients underflow "
                             "without loss scaling), so the fp16 tower is forward only")
        _check_config(getattr(vision_model, "config", None))
        named = dict(vision_model.named_parameters())
        prefix = "vision_model." if "vision_model.embeddings.class_embedding" in named else ""
        names = [prefix + key for _, key in _lib.CLIP_TOWER_FIELDS]
        for i in range(_lib.CLIP_TOWER_LAYERS):
            names += [f"{prefix}encoder.layers.{i}.{key}" for _, key in _lib.CLIP_TOWER_LAYER_FIELDS]
        missing = [n for n in names if n not in named]
        if missing:
            raise NotImplementedError(f"not a CLIPVisionModel: parameters {missing[:3]} are missing")
        self.vision_model = vision_model
        self.dtype = torch.float16 if dtype == torch.float16 else torch.bfloat16
        self.trainable_layers = trainable_layers
        self.train_embeddings = train_embeddings
        self._names = names
        self._packed = None
        self._packed_key = None
        self._weights = None
        self._warned_dtype = False
        self._input_grad = False
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packed())

    @property
    def input_grad(self) -> bool:
        return self._input_grad

    @input_grad.setter
    def input_grad(self, value: bool):
        if not isinstance(value, bool):
            raise ValueError(f"input_grad = {value!r}: expected True or False")
        if value and self.dtype == torch.float16:
            raise ValueError("input_grad needs the bf16 tower: the fp16 tower is forward only")
        self._input_grad = value

    def invalidate_packed(self):
        """Drop the derived weight cache (call it after writing parameters through a ``.data`` alias: such writes change neither
        ``data_ptr`` nor ``_version``)."""
        self._packed = None
        self._packed_key = None
        self._weights = None

    def _apply(self, fn, *args, **kwargs):
        self.invalidate_packed()
        return super()._apply(fn, *args, **kwargs)

    def _params(self):
        named = dict(self.vision_model.named_parameters())
        return [named[n] for n in self._names]

    def _trainable_params(self):
        """The 16 K parameters of layers 23 - K .. 22, layer by layer in _lib.CLIP_TOWER_LAYER_FIELDS order; with train_embeddings, the
        five embedding-stage parameters (_lib.CLIP_TOWER_FIELDS order) before them."""
        if self.train_embeddings:
            return self._params()
        per = len(_lib.CLIP_TOWER_LAYER_FIELDS)
        first = len(_lib.CLIP_TOWER_FIELDS) + (_lib.CLIP_TOWER_LAYERS - self.trainable_layers) * per
        return self._params()[first:] if self.trainable_layers > 0 else []

    def _live_weights(self, w, train_params, device):
        """A copy of the weight struct whose trainable layers (and with train_embeddings, embedding stage) point at the live parameters."""
        for p in train_params:
            if p.dtype != torch.bfloat16 or p.device != device or not p.is_contiguous() or p.data_ptr() % 16 != 0:
                raise ValueError("the trainable layers' parameters are read in place: they must be contiguous, 16-byte aligned bf16 tensors "
                                 "on the crops' device")
        live = _lib.TpClipTowerWeights.from_buffer_copy(w)
        if self.train_embeddings:
            n_top = len(_lib.CLIP_TOWER_FIELDS)
            for (field, _), p in zip(_lib.CLIP_TOWER_FIELDS, train_params[:n_top]):
                setattr(live, field, p.data_ptr())
            train_params = train_params[n_top:]
        per = len(_lib.CLIP_TOWER_LAYER_FIELDS)
        first = _lib.CLIP_TOWER_LAYERS - self.trainable_layers
        for t in range(self.trainable_layers):
            live.layers[first + t] = _lib.TpClipTowerLayer(*[p.data_ptr() for p in train_params[t * per:(t + 1) * per]])
        return live

    def _packed_weights(self, device):
        params = self._params()
        key = (str(device), self.dtype) + tuple((p.data_ptr(), p._version, p.dtype) for p in params)
        if self._packed is not None and self._packed_key == key:
            return self._packed, self._weights
        f16 = self.dtype == torch.float16
        if not f16 and any(p.dtype != torch.bfloat16 for p in params) and not self._warned_dtype:
            self._warned_dtype = True
            warnings.warn("CLIPVisionTowerB200 computes with bf16 storage and fp32 accumulation: the tower's fp16 / fp32 parameters are "
                          "cast to bf16 once into the derived cache", UserWarning, stacklevel=3)
        # parameters of the compute dtype are read in place; anything else (other dtype, non-contiguous, not 16-byte aligned) through a
        # copy in it (in fp16 that cast is the reference's own vision_tower.to(dtype=torch.float16): no warning)
        bf = [p.detach().to(device=device, dtype=self.dtype).contiguous() for p in params]
        bf = [t if t.data_ptr() % 16 == 0 else t.clone() for t in bf]
        n_top = len(_lib.CLIP_TOWER_FIELDS)
        w = _lib.TpClipTowerWeights(*[t.data_ptr() for t in bf[:n_top]])
        per = len(_lib.CLIP_TOWER_LAYER_FIELDS)
        for i in range(_lib.CLIP_TOWER_LAYERS):
            w.layers[i] = _lib.TpClipTowerLayer(*[t.data_ptr() for t in bf[n_top + i * per: n_top + (i + 1) * per]])
        nbytes = lib.tp_clip_tower_packed_bytes()
        packed = torch.empty(nbytes, dtype=torch.uint8, device=device)
        stream = torch.cuda.current_stream(device).cuda_stream
        if f16:
            check(lib.tp_clip_tower_pack_weights_f16(C.byref(w), packed.data_ptr(), nbytes, stream), "tp_clip_tower_pack_weights_f16")
        else:
            check(lib.tp_clip_tower_pack_weights(C.byref(w), packed.data_ptr(), nbytes, stream), "tp_clip_tower_pack_weights")
        # parameters of the compute dtype are read in place by every forward; the cast copies of others are kept alive with the cache
        self._packed, self._packed_key, self._weights = packed, key, (w, bf)
        return packed, self._weights

    def hidden_states(self, images: torch.Tensor):
        """images: [N, 3, 336, 336] CUDA crops (bf16 read in place, any crop stride; other dtypes cast to bf16).  Returns the tuple
        (hidden_states[12], [16], [22], [23]), each bf16 [N, 577, 1024] with the CLS row.
        With dtype=torch.float16: bf16 and fp16 crops are read in place (bf16 ones converted as ``images.to(torch.float16)`` rounds
        them), other dtypes cast to fp16, and the four hidden states are fp16.
        With trainable_layers = K > 0, under ``torch.enable_grad()`` and when a parameter of layers 23 - K .. 22 requires grad: the same
        four tensors with the same bits, attached to autograd (those at or below the first trainable layer's input detached); their
        backward takes up to four gradients (None allowed) and gives every such parameter that requires grad its gradient.  The trainable
        layers' parameters must be bf16 CUDA tensors, contiguous and 16-byte aligned: they are read in place, and what is derived from
        them is rebuilt by every call.  The crops get no gradient.
        When, in addition, the wrapped model asks for gradient checkpointing (``wants_gradient_checkpointing``, read at every call),
        the step keeps per trainable layer only its input and its derived weights (1.2 MB per crop plus 6.3 MB, against 20.1 MB per
        crop), and the backward recomputes each layer's intermediates before its gradients: the outputs and every gradient have the same
        bits as without it.  A graph keeps the mode it was built with.
        With train_embeddings (trainable_layers = 23), the embedding stage's five parameters count among the trainable ones above: read
        in place under the same conditions, each that requires grad gets its gradient, and the step keeps in addition the crops' patch
        rows and the patch embedding's output (1.9 MB per crop), in both modes.
        With ``input_grad`` (bf16 tower), under grad mode and when the crops require grad: the step runs the whole-tower training pair
        (all 23 layers and the embedding stage, include/tokenpacker_b200_clip_tower_crop_grad.h), the four hidden states are attached to
        autograd, and the backward gives the crops their gradient (fp32 crops an fp32 gradient straight from the kernels' fp32 sums,
        other crops a bf16 one in their dtype; crop views of any crop stride are read in place).  Parameters get gradients exactly as
        above (those of the trainable layers and, with train_embeddings, of the embedding stage that require grad, with the bits the
        step without input_grad gives); every other layer only passes its input gradient on, whatever its requires_grad says.  The
        step keeps the saved sets of all 23 layers: about 23 x 20.1 MB per crop plus 1.86 MB per crop for the embedding stage, or with
        gradient checkpointing 23 x 1.2 MB per crop plus 23 x 6.3 MB (and the 1.86 MB per crop).  Checkpointing follows
        ``wants_gradient_checkpointing``, which needs the wrapped model in training mode: an attribution run on an eval-mode model keeps
        the full saved sets."""
        _check_crops(images)
        train_params = self._trainable_params() if torch.is_grad_enabled() else []
        train = any(p.requires_grad for p in train_params)
        crop_grad = self._input_grad and torch.is_grad_enabled() and images.requires_grad
        if not crop_grad and torch.is_grad_enabled() and (
                images.requires_grad or (self.trainable_layers == 0 and any(p.requires_grad for p in self._params()))):
            raise NotImplementedError("CLIPVisionTowerB200 is forward only (the tower is frozen in every TokenPacker recipe): run it under "
                                      "torch.no_grad(), or detach the crops and freeze the tower's parameters")
        if not images.is_cuda:
            raise RuntimeError("tokenpacker_b200 has no CPU path: crops must be CUDA tensors on an H100")
        n = images.shape[0]
        if crop_grad and n == 0:
            raise ValueError("input_grad needs at least one crop")
        device = images.device
        if n > 0 and (crop_grad or train):
            with torch.cuda.device(device):
                packed, (w, _) = self._packed_weights(device)
                return _TowerTrainFunction.apply(self, images, packed, self._live_weights(w, train_params, device),
                                                 wants_gradient_checkpointing(self.vision_model), crop_grad, *train_params)
        outs = tuple(torch.empty((n, _TOKENS, 1024), dtype=self.dtype, device=device) for _ in _OUT_LAYERS)
        if n > 0:
            with torch.cuda.device(device):
                packed, (w, _) = self._packed_weights(device)
                self._forward(images, packed, w, (C.c_void_p * 4)(*[o.data_ptr() for o in outs]), interleaved=False)
        return outs

    def interleaved_hidden_states(self, images: torch.Tensor) -> torch.Tensor:
        """images as for ``hidden_states``.  Returns hidden_states 12, 16, 22 and 23 side by side in one [N, 577, 4096] tensor of the
        tower's dtype (include/tokenpacker_b200_clip_tower_interleaved.h): columns 1024 j .. 1024 j + 1023 hold hidden_states[(12, 16,
        22, 23)[j]] with the bits ``hidden_states`` gives.  That is ``torch.cat(tower.hidden_states(images), dim=2)``, LLaVA's
        ``feature_select`` concatenation, written by the tower in place: one buffer instead of two, and no copy.
        Inference only: under grad mode, crops or tower parameters that require grad are refused (``hidden_states`` trains)."""
        _check_crops(images)
        if torch.is_grad_enabled() and (images.requires_grad or any(p.requires_grad for p in self._params())):
            raise NotImplementedError("interleaved_hidden_states is inference only: run it under torch.no_grad() (as LLaVA's "
                                      "CLIPVisionTower.forward does), or train through hidden_states")
        if not images.is_cuda:
            raise RuntimeError("tokenpacker_b200 has no CPU path: crops must be CUDA tensors on an H100")
        n, device = images.shape[0], images.device
        out = torch.empty((n, _TOKENS, len(_OUT_LAYERS) * 1024), dtype=self.dtype, device=device)
        if n > 0:
            with torch.cuda.device(device):
                packed, (w, _) = self._packed_weights(device)
                self._forward(images, packed, w, out.data_ptr(), interleaved=True)
        return out

    def _forward(self, images, packed, w, dest, interleaved: bool):
        """The inference forward over n > 0 crops into dest: the four outputs' pointers, or the interleaved output's."""
        f16 = self.dtype == torch.float16
        n, device = images.shape[0], images.device
        x = images if f16 and images.dtype in (torch.bfloat16, torch.float16) else images.to(self.dtype)
        if not (x.stride(3) == 1 and x.stride(2) == _IMAGE and x.stride(1) == _IMAGE * _IMAGE and x.stride(0) >= 3 * _IMAGE * _IMAGE):
            x = x.contiguous()
        ws_bytes = lib.tp_clip_tower_workspace_bytes(n)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        stream = torch.cuda.current_stream(device).cuda_stream
        name = "tp_clip_tower_forward" + ("_interleaved" if interleaved else "") + ("_f16" if f16 else "")
        crops = (x.data_ptr(),)
        if f16:
            crops += (_lib.TP_CLIP_CROPS_F16 if x.dtype == torch.float16 else _lib.TP_CLIP_CROPS_BF16,)
        check(getattr(lib, name)(packed.data_ptr(), C.byref(w), *crops, n, x.stride(0), dest, ws.data_ptr(), ws_bytes, stream), name)
