"""tokenpacker_b200 — H100 (sm_90a) implementation of the TokenPacker visual projector hot path.

Drop-in for ``llava/model/multimodal_projector/builder.py`` of CircleRadon/TokenPacker:
``build_vision_projector(config)`` / ``TokenPackerB200.forward((feat, feat_multi))`` keep the reference's
constructor, parameter names and output layout; the arithmetic runs in hand-written wgmma/TMA CUDA kernels behind
the C ABI declared in ``include/tokenpacker_b200.h``.  There is no CPU fallback.  ``build_vision_tower`` / ``CLIPVisionTower`` do the
same for ``llava/model/multimodal_encoder/builder.py``: the CLIP tower on the same kernels, returning ``(feat, feat_multi)``.
"""
from . import _lib  # noqa: F401  (fails loudly when the CUDA library is not built)
from .projector import TokenPackerB200, TokenPacker, build_vision_projector, IdentityMap
from .hd import Image_Patch, hd_grid, hd_tile, hd_tile_batch, hd_preprocess_batch, hd_plan, hd_assemble, hd_seq_len
from .clip import clip_preprocess_batch
from .jpeg import decode_jpeg_batch, jpeg_unsupported
from .png import decode_png_batch, png_unsupported
from .splice import splice_multimodal, splice_plan
from .tower import CLIPVisionTowerB200
from .vision_tower import CLIPVisionTower, build_vision_tower

__all__ = ["TokenPackerB200", "TokenPacker", "build_vision_projector", "IdentityMap", "Image_Patch", "hd_grid", "hd_tile", "hd_tile_batch",
           "hd_preprocess_batch", "hd_plan", "hd_assemble", "hd_seq_len", "clip_preprocess_batch", "decode_jpeg_batch", "jpeg_unsupported",
           "decode_png_batch", "png_unsupported", "splice_multimodal", "splice_plan", "CLIPVisionTowerB200",
           "CLIPVisionTower", "build_vision_tower"]
