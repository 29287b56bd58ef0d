"""LLaVA's vision-tower seam on the sm_90a CLIP tower: ``build_vision_tower`` and ``CLIPVisionTower``.

A drop-in for ``llava/model/multimodal_encoder/builder.py`` and ``clip_encoder.CLIPVisionTower``: the same constructor, the same
``load_model`` / ``is_loaded`` / ``image_processor`` / ``config`` / ``hidden_size`` / ``num_patches`` / ``dummy_feature`` / ``dtype`` /
``device``, the same state_dict keys (``vision_tower.vision_model.…``) and the same ``forward(images) -> (feat, feat_multi)``, so
``llava_arch.py``, ``train.py`` and the evaluation scripts run unchanged once the builder is swapped:

    from tokenpacker_b200 import build_vision_tower          # in llava/model/multimodal_encoder/builder.py

``forward`` runs ``CLIPVisionTowerB200.interleaved_hidden_states``: the tower stores hidden states 12, 16, 22 and 23 straight into the
four 1024-column blocks of one [N, 577, 4096] buffer, so ``feat_multi`` is the reference's ``torch.cat`` without the copy and ``feat``
is a column slice of the same buffer.  The compute precision follows the wrapped model's parameters at every call: fp16 parameters
(``vision_tower.to(dtype=torch.float16)``, as the evaluation scripts do) run the fp16 tower, anything else the bf16 one.
"""
from __future__ import annotations

import os

import torch
from torch import nn

from .tower import CLIPVisionTowerB200, _OUT_LAYERS, _check_config

_SELECT_FEATURES = ("patch", "cls_patch")


def build_vision_tower(vision_tower_cfg, **kwargs):
    """``multimodal_encoder/builder.py``'s builder: a CLIPVisionTower for a local path or an ``openai/…`` / ``laion/…`` name (the
    config's ``mm_vision_tower``, else ``vision_tower``); kwargs (``delay_load``) go to the constructor."""
    name = getattr(vision_tower_cfg, "mm_vision_tower", getattr(vision_tower_cfg, "vision_tower", None))
    if isinstance(name, str) and (os.path.exists(name) or name.startswith("openai") or name.startswith("laion")):
        return CLIPVisionTower(name, args=vision_tower_cfg, **kwargs)
    raise ValueError(f"Unknown vision tower: {name}")


def _feature_block(select_layer, num_hidden_layers: int) -> int:
    """The column block (0 .. 3) of the interleaved buffer that holds ``hidden_states[select_layer]`` of a tower with
    num_hidden_layers layers (num_hidden_layers + 1 hidden states, negative indices from the end as in Python)."""
    states = num_hidden_layers + 1
    layer = None
    if isinstance(select_layer, int) and not isinstance(select_layer, bool) and -states <= select_layer < states:
        layer = select_layer % states
    if layer not in _OUT_LAYERS:
        raise NotImplementedError(f"mm_vision_select_layer = {select_layer!r}: the tower computes hidden states {list(_OUT_LAYERS)} only "
                                  f"(of {states}; e.g. -2 or 23 for hidden_states[23])")
    return _OUT_LAYERS.index(layer)


class CLIPVisionTower(nn.Module):
    """``clip_encoder.CLIPVisionTower`` on the sm_90a kernels.

    vision_tower: a path or hub name, as in the reference (loaded with transformers by ``load_model``); or an already loaded
    ``CLIPVisionModel`` (any module ``CLIPVisionTowerB200`` accepts), which is wrapped as it is, with no image processor.
    args: ``mm_vision_select_layer`` (any index naming hidden state 12, 16, 22 or 23: others raise ``NotImplementedError`` here) and
    ``mm_vision_select_feature`` (``'patch'``, the default, or ``'cls_patch'``; others raise ``ValueError`` in ``forward``, as the
    reference does).  delay_load: keep only the config until ``load_model()``.

    The wrapped ``CLIPVisionModel`` stays the owner of the parameters (``self.vision_tower``); the derived weight cache of
    ``CLIPVisionTowerB200`` is built on the first forward of each precision, kept while the parameters stay as they are, and dropped by
    ``load_state_dict``, ``.to()`` / ``.cuda()`` / ``.half()``, ``invalidate_packed()`` and a switch of precision."""

    def __init__(self, vision_tower, args, delay_load: bool = False):
        super().__init__()
        self.is_loaded = False
        self.select_layer = args.mm_vision_select_layer
        self.select_feature = getattr(args, "mm_vision_select_feature", "patch")
        self._towers = {}                      # compute dtype -> CLIPVisionTowerB200 (a plain dict: not submodules, not in the state_dict)
        if isinstance(vision_tower, nn.Module):
            self.vision_tower_name = getattr(getattr(vision_tower, "config", None), "_name_or_path", None)
            self._wrap(vision_tower, None)
        elif not delay_load:
            self.vision_tower_name = vision_tower
            self.load_model()
        else:
            from transformers import CLIPVisionConfig
            self.vision_tower_name = vision_tower
            self.cfg_only = CLIPVisionConfig.from_pretrained(vision_tower)
            _check_config(self.cfg_only)
        self._block = _feature_block(self.select_layer, self.config.num_hidden_layers)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packed())

    def load_model(self):
        """Load ``CLIPImageProcessor`` and ``CLIPVisionModel`` from ``vision_tower_name`` and freeze the model, as the reference does."""
        from transformers import CLIPImageProcessor, CLIPVisionModel
        processor = CLIPImageProcessor.from_pretrained(self.vision_tower_name)
        model = CLIPVisionModel.from_pretrained(self.vision_tower_name)
        model.requires_grad_(False)
        self._wrap(model, processor)

    def _wrap(self, model: nn.Module, processor):
        towers = {torch.bfloat16: CLIPVisionTowerB200(model), torch.float16: CLIPVisionTowerB200(model, dtype=torch.float16)}
        self.image_processor = processor
        self.vision_tower = model
        self._towers = towers
        self.is_loaded = True

    def invalidate_packed(self):
        """Drop the derived weight caches (see ``CLIPVisionTowerB200.invalidate_packed``)."""
        for tower in self._towers.values():
            tower.invalidate_packed()

    def _apply(self, fn, *args, **kwargs):
        self.invalidate_packed()
        return super()._apply(fn, *args, **kwargs)

    @torch.no_grad()
    def forward(self, images):
        """images: [N, 3, 336, 336] crops (on the tower's device, or moved there).  Returns (feat, feat_multi), the reference's
        (``hidden_states[select_layer]``, ``torch.cat(hidden_states[12, 16, 22, 23], dim=2)``), rows 1.. with 'patch' and all 577 with
        'cls_patch', in ``images.dtype``: views of one [N, 577 or 576, 4096] buffer (feat its 1024 columns of the selected layer), cast
        once when the tower's dtype is not the crops'.  Values are those of ``CLIPVisionTowerB200.hidden_states`` of that precision."""
        if isinstance(images, list):
            raise TypeError("CLIPVisionTower.forward takes one [N,3,336,336] tensor: stack the crops (the reference's list branch "
                            "cannot run, it appends to an undefined list)")
        if self.select_feature not in _SELECT_FEATURES:
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        if not self.is_loaded:
            raise RuntimeError("CLIPVisionTower: call load_model() first (built with delay_load=True)")
        dtype = torch.float16 if self.dtype == torch.float16 else torch.bfloat16
        for other, tower in self._towers.items():
            if other != dtype:
                tower.invalidate_packed()          # one precision's cache alive at a time
        buf = self._towers[dtype].interleaved_hidden_states(images.to(device=self.device))
        rows = buf[:, 1:] if self.select_feature == "patch" else buf
        if rows.dtype != images.dtype:
            rows = rows.to(images.dtype)
        return rows[:, :, 1024 * self._block:1024 * (self._block + 1)], rows

    @property
    def dummy_feature(self):
        return torch.zeros(1, self.hidden_size, device=self.device, dtype=self.dtype)

    @property
    def dtype(self):
        return next(self.vision_tower.parameters()).dtype

    @property
    def device(self):
        return next(self.vision_tower.parameters()).device

    @property
    def config(self):
        return self.vision_tower.config if self.is_loaded else self.cfg_only

    @property
    def hidden_size(self):
        return self.config.hidden_size

    @property
    def num_patches(self):
        return (self.config.image_size // self.config.patch_size) ** 2
