"""Non-HD CLIP input on the GPU: what the released 144-, 64- and 36-token recipes do to a decoded image before the vision tower.

Mirrors the reference seams:
  * ``expand2square(image, tuple(int(x * 255) for x in image_mean))``  llava/mm_utils.py:14-25, llava/train/train.py:679-694
    (``image_aspect_ratio == 'pad'``: finetuning and every eval script through ``process_images``)
  * ``CLIPImageProcessor.preprocess(image)['pixel_values']``           llava/train/train.py:693,732-734 (``'square'``: pretraining)
    with the openai/clip-vit-large-patch14-336 configuration of the slow (PIL) processor of transformers 4.31: shortest edge 336
    with PIL's 8-bit BICUBIC resample, center crop 336 x 336, rescale 1/255, normalise by the CLIP mean and std

The result is the processor's float32 output bit for bit (PIL's resample is fixed-point integer arithmetic, restated exactly by
the kernels).  That is the slow processor's: the default ``CLIPImageProcessor`` of transformers >= 5 is a torchvision-based "fast"
processor whose bits differ; ``CLIPImageProcessorPil`` is the slow one there.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import lib, check
from .hd import BLOCK, _norm_table_on, _staging, _u8_sources

ASPECT_RATIOS = {"square": _lib.TP_CLIP_SQUARE, "pad": _lib.TP_CLIP_PAD}


def clip_preprocess_plan(sizes, aspect_ratio: str = "pad"):
    """tp_clip_preprocess_plan on the host: (tp_clip_image rows, int32 coefficient tables, workspace bytes) for (h, w) sizes."""
    b = len(sizes)
    hs = (C.c_int64 * max(b, 1))(*[int(h) for h, _ in sizes])
    ws = (C.c_int64 * max(b, 1))(*[int(w) for _, w in sizes])
    nco, wsb = C.c_int64(0), C.c_size_t(0)
    mode = _mode(aspect_ratio)
    check(lib.tp_clip_preprocess_plan(hs, ws, b, mode, None, None, C.byref(nco), C.byref(wsb)), "tp_clip_preprocess_plan")
    images = (_lib.TpClipImage * max(b, 1))()
    coeffs = (C.c_int32 * max(nco.value, 1))()
    check(lib.tp_clip_preprocess_plan(hs, ws, b, mode, images, coeffs, C.byref(nco), C.byref(wsb)), "tp_clip_preprocess_plan")
    return images[:b], coeffs[:nco.value], wsb.value


def _mode(aspect_ratio):
    if aspect_ratio not in ASPECT_RATIOS:
        raise ValueError(f'aspect_ratio must be "pad" or "square", not {aspect_ratio!r}')
    return ASPECT_RATIOS[aspect_ratio]


def clip_preprocess_batch(images, aspect_ratio: str = "pad", dtype=torch.float32, layout: str = "HWC", _return_launch: bool = False):
    """expand2square (``aspect_ratio="pad"`` only) and the CLIP-336 image processor for a batch of DECODED 8-bit images, in two launches.

    images: sequence of uint8 CUDA tensors, [h, w, 3] for layout "HWC" (np.array(pil_image), what the reference decodes) or [3, h, w]
    for "CHW" (torchvision.io.decode_image); sizes may differ, and views are read through their strides, not copied.
    aspect_ratio: "pad" (``image_aspect_ratio == 'pad'``) or "square" (the default ``'square'``: the processor alone).
    dtype: torch.float32, or torch.bfloat16 (the tower's dtype; equal to the float32 output .to(torch.bfloat16), bit for bit).
    Returns [B, 3, 336, 336] in dtype, in the order of the images: the processor's ``pixel_values``, bit for bit in float32.  Not
    differentiable: the inputs are integer pixels and the resize is PIL's integer arithmetic; gradients to the pixels start at these
    crops (``crops.requires_grad_()`` with ``CLIPVisionTowerB200.input_grad``)."""
    mode = _mode(aspect_ratio)
    images, device, sizes, sources = _u8_sources(images, dtype, layout)
    b = len(images)
    hs = (C.c_int64 * b)(*[h for h, _ in sizes])
    ws = (C.c_int64 * b)(*[w for _, w in sizes])
    nco, wsb = C.c_int64(0), C.c_size_t(0)
    check(lib.tp_clip_preprocess_plan(hs, ws, b, mode, None, None, C.byref(nco), C.byref(wsb)), "tp_clip_preprocess_plan")
    # one pinned buffer, one asynchronous copy: [plan rows | sources | coefficient tables]
    src_off = (C.sizeof(_lib.TpClipImage) * b + 15) // 16 * 16
    co_off = (src_off + C.sizeof(_lib.TpHdU8Source) * b + 15) // 16 * 16
    total_bytes = co_off + max(nco.value, 1) * 4
    st = _staging(device, total_bytes)
    st["event"].synchronize()                     # the previous call's copy has left the pinned buffer
    host = st["host"]
    desc = (_lib.TpClipImage * b).from_address(host.data_ptr())
    check(lib.tp_clip_preprocess_plan(hs, ws, b, mode, desc, C.cast(host.data_ptr() + co_off, C.POINTER(C.c_int32)), C.byref(nco),
                                      C.byref(wsb)), "tp_clip_preprocess_plan")
    rows = (_lib.TpHdU8Source * b).from_address(host.data_ptr() + src_off)
    for i, s in enumerate(sources):
        rows[i] = _lib.TpHdU8Source(*s)
    table = _norm_table_on(device)
    out_dtype = 0 if dtype == torch.float32 else 1
    with torch.cuda.device(device):
        dev = st["dev"]
        dev[:total_bytes].copy_(host[:total_bytes], non_blocking=True)
        stream = torch.cuda.current_stream(device)
        st["event"].record(stream)
        out = torch.empty((b, 3, BLOCK, BLOCK), dtype=dtype, device=device)
        workspace = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device=device)
        check(lib.tp_clip_preprocess_batch(host.data_ptr(), dev.data_ptr(), dev.data_ptr() + src_off, dev.data_ptr() + co_off, b,
                                           table.data_ptr(), out_dtype, out.data_ptr(), workspace.data_ptr(), wsb.value,
                                           stream.cuda_stream), "tp_clip_preprocess_batch")
        # the source images and the workspace must outlive the asynchronous launches: tie them to the stream
        for t in images:
            t.record_stream(stream)
        workspace.record_stream(stream)
    if _return_launch:
        # benchmark hook: (device tables, sources offset, coefficients offset, a host copy of the plan rows, workspace, norm table)
        plan = (_lib.TpClipImage * b)()
        C.memmove(plan, desc, C.sizeof(plan))
        return out, (dev, src_off, co_off, plan, workspace, table)
    return out
