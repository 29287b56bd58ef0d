"""tokenpacker_b200 — H100 (sm_90a) implementation of the TokenPacker visual projector hot path.

Drop-in for ``llava/model/multimodal_projector/builder.py`` of CircleRadon/TokenPacker:
``build_vision_projector(config)`` / ``TokenPackerB200.forward((feat, feat_multi))`` keep the reference's
constructor, parameter names and output layout; the arithmetic runs in hand-written wgmma/TMA CUDA kernels behind
the C ABI declared in ``include/tokenpacker_b200.h``.  There is no CPU fallback.
"""
from . import _lib  # noqa: F401  (fails loudly when the CUDA library is not built)
from .projector import TokenPackerB200, TokenPacker, build_vision_projector, IdentityMap
from .hd import Image_Patch, hd_grid, hd_tile, hd_tile_batch, hd_preprocess_batch, hd_plan, hd_assemble, hd_seq_len
from .clip import clip_preprocess_batch
from .splice import splice_multimodal, splice_plan

__all__ = ["TokenPackerB200", "TokenPacker", "build_vision_projector", "IdentityMap", "Image_Patch", "hd_grid", "hd_tile", "hd_tile_batch",
           "hd_preprocess_batch", "hd_plan", "hd_assemble", "hd_seq_len", "clip_preprocess_batch", "splice_multimodal", "splice_plan"]
