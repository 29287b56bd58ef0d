"""PNG files decoded on the GPU, byte for byte as PIL decodes them, into the uint8 images the GPU front ends read.

Replaces ``np.array(Image.open(path).convert('RGB'))`` in front of ``hd_preprocess_batch`` / ``clip_preprocess_batch`` for the PNG
files of a dataset (documents, charts and diagrams mostly are): the compressed bytes are uploaded instead of the decoded pixels.
Supported are non-interlaced files at bit depth <= 8 in every colour type; ``png_unsupported`` says which files are not, so that a
caller can send those to PIL.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import lib, check
from .hd import _staging
from .jpeg import _buffers

STATUS_TEXT = {_lib.TP_PNG_STATUS_BLOCK_TYPE: "invalid deflate block type",
               _lib.TP_PNG_STATUS_CODE_LENGTHS: "invalid code lengths set",
               _lib.TP_PNG_STATUS_SYMBOL: "invalid literal/length or distance code",
               _lib.TP_PNG_STATUS_DISTANCE: "invalid distance too far back",
               _lib.TP_PNG_STATUS_STORED: "invalid stored block lengths",
               _lib.TP_PNG_STATUS_TRUNCATED: "truncated image data",
               _lib.TP_PNG_STATUS_DATA_SIZE: "image data of the wrong size",
               _lib.TP_PNG_STATUS_ADLER: "incorrect data check",
               _lib.TP_PNG_STATUS_FILTER: "invalid row filter type"}


def _reason(code: int) -> str:
    return lib.tp_png_reason_string(code).decode()


def png_unsupported(data) -> list:
    """The host plan alone: per file None when decode_png_batch decodes it, else the reason it is refused ("16-bit samples",
    "interlaced PNG", "not a PNG file", "malformed or truncated chunks", ...)."""
    ptrs, sizes, keep = _buffers(data)
    b = len(ptrs)
    images = (_lib.TpPngImage * max(b, 1))()
    totals = _lib.TpPngTotals()
    check(lib.tp_png_plan((C.c_void_p * max(b, 1))(*ptrs), (C.c_int64 * max(b, 1))(*sizes), b, images, None, None, C.byref(totals)),
          "tp_png_plan")
    del keep
    return [None if images[i].reason == _lib.TP_PNG_SUPPORTED else _reason(images[i].reason) for i in range(len(data))]


def decode_png_batch(data, device="cuda", *, return_status: bool = False):
    """Decode PNG files on the GPU: a list of uint8 CUDA tensors [h, w, 3], each equal to
    ``np.array(Image.open(io.BytesIO(f)).convert('RGB'))`` byte for byte.  The outputs are views into one device buffer.

    data: a sequence of files as bytes, 1-D uint8 numpy arrays or 1-D uint8 CPU tensors.
    One host plan, one upload of the zlib streams and palettes, and a number of launches that follows from the files' sizes alone.
    A file the plan refuses raises ValueError naming its index and the reason before anything runs (``png_unsupported`` checks
    first).  return_status: False (default) synchronises the stream and raises ValueError naming every file whose image data was
    corrupt or truncated.  True returns ``(images, status)`` without synchronising: status is an int32 CUDA tensor [n, 4] of
    (status, deflate blocks, blocks the chain decoded itself, candidate block starts) per file, status 0 meaning the image is valid."""
    def launch(out, workspace, args, stream):
        check(lib.tp_png_decode_batch(*args, stream), "tp_png_decode_batch")

    rows, out, workspace, status = _plan_upload_launch(data, device, launch)
    views = [out[im.out_offset:im.out_offset + im.h * im.w * 3].view(im.h, im.w, 3) for im in rows]
    if return_status:
        return views, status
    bad = [(i, int(s)) for i, s in enumerate(status[:, 0].tolist()) if s != 0]
    if bad:
        raise ValueError("; ".join(f"file {i}: {STATUS_TEXT.get(s, f'status {s}')}" for i, s in bad))
    return views


def _plan_upload_launch(data, device, launch):
    """The plan, the upload and launch(out, workspace, args, stream), where args are tp_png_decode_batch's arguments before the
    stream (the stage tests launch their own stages here).  Returns (plan rows, output bytes, workspace, status)."""
    data = list(data)
    if not data:
        raise ValueError("decode_png_batch needs at least one file")
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("decode_png_batch runs on a CUDA device; there is no CPU path")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    ptrs, sizes, keep = _buffers(data)
    b = len(ptrs)
    # one pinned buffer, one asynchronous copy: [plan rows | palettes | staged zlib streams]; the streams need at most the files' bytes
    pal_off = (C.sizeof(_lib.TpPngImage) * b + 15) // 16 * 16
    stg_off = pal_off + _lib.TP_PNG_PALETTE_BYTES * b
    total_bytes = stg_off + sum((n + 15) // 16 * 16 for n in sizes) + 16
    st = _staging(device, total_bytes)
    st["event"].synchronize()                     # the previous call's copy has left the pinned buffer
    host = st["host"]
    images = (_lib.TpPngImage * b).from_address(host.data_ptr())
    totals = _lib.TpPngTotals()
    check(lib.tp_png_plan((C.c_void_p * b)(*ptrs), (C.c_int64 * b)(*sizes), b, images, host.data_ptr() + pal_off,
                          host.data_ptr() + stg_off, C.byref(totals)), "tp_png_plan")
    del keep
    for i in range(b):
        if images[i].reason != _lib.TP_PNG_SUPPORTED:
            raise ValueError(f"file {i}: {_reason(images[i].reason)} (decode it with PIL)")
    rows = (_lib.TpPngImage * b)()
    C.memmove(rows, images, C.sizeof(rows))
    copy_bytes = stg_off + totals.staged_bytes
    with torch.cuda.device(device):
        dev = st["dev"]
        dev[:copy_bytes].copy_(host[:copy_bytes], non_blocking=True)
        stream = torch.cuda.current_stream(device)
        st["event"].record(stream)
        out = torch.empty(max(totals.output_bytes, 1), dtype=torch.uint8, device=device)
        workspace = torch.empty(max(totals.workspace_bytes, 16), dtype=torch.uint8, device=device)
        status = torch.empty((b, 4), dtype=torch.int32, device=device)
        launch(out, workspace, (C.addressof(rows), dev.data_ptr(), dev.data_ptr() + pal_off, dev.data_ptr() + stg_off, b, out.data_ptr(),
                workspace.data_ptr(), workspace.numel(), status.data_ptr()), stream.cuda_stream)
        workspace.record_stream(stream)
    return rows, out, workspace, status
