"""Baseline JPEG files decoded on the GPU, bit for bit as PIL decodes them, into the uint8 images the GPU front ends read.

Replaces ``np.array(Image.open(path).convert('RGB'))`` in front of ``hd_preprocess_batch`` / ``clip_preprocess_batch``
(llava/train/train.py:679-734 and the eval loaders): the compressed bytes are uploaded instead of the decoded pixels.  Supported are
the files most JPEG writers produce (baseline or extended sequential Huffman, 8-bit, grayscale or YCbCr at 4:4:4 / 4:2:2 / 4:2:0);
``jpeg_unsupported`` says which files are not, so that a caller can send those to PIL.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check
from .hd import _staging

STATUS_TEXT = {_lib.TP_JPEG_STATUS_ENTROPY: "corrupt or truncated entropy-coded data",
               _lib.TP_JPEG_STATUS_RESTART: "restart markers do not match the restart interval"}


def _buffers(data):
    """(pointers, sizes, keep-alive) of the files: bytes-like objects, 1-D uint8 numpy arrays or 1-D uint8 CPU tensors."""
    ptrs, sizes, keep = [], [], []
    for i, d in enumerate(data):
        if isinstance(d, torch.Tensor):
            if d.device.type != "cpu" or d.dtype != torch.uint8 or d.dim() != 1:
                raise TypeError(f"file {i}: a tensor must be a 1-D uint8 CPU tensor")
            d = d.contiguous()
            keep.append(d)
            ptrs.append(d.data_ptr())
            sizes.append(d.numel())
            continue
        if isinstance(d, np.ndarray):
            if d.dtype != np.uint8 or d.ndim != 1:
                raise TypeError(f"file {i}: an array must be 1-D uint8")
            d = np.ascontiguousarray(d)
            keep.append(d)
            ptrs.append(d.ctypes.data)
            sizes.append(d.size)
            continue
        if isinstance(d, (bytearray, memoryview)):
            d = bytes(d)
        if not isinstance(d, bytes):
            raise TypeError(f"file {i}: expected bytes, a uint8 numpy array or a uint8 CPU tensor, not {type(d).__name__}")
        buf = C.c_char_p(d)
        keep.append((d, buf))
        ptrs.append(C.cast(buf, C.c_void_p).value or 0)
        sizes.append(len(d))
    return ptrs, sizes, keep


def _reason(code: int) -> str:
    return lib.tp_jpeg_reason_string(code).decode()


def jpeg_unsupported(data) -> list:
    """The host plan alone: per file None when decode_jpeg_batch decodes it, else the reason it is refused ("progressive JPEG",
    "CMYK, YCCK or RGB colour", "malformed or truncated header", "not a JPEG file", ...)."""
    ptrs, sizes, keep = _buffers(data)
    b = len(ptrs)
    images = (_lib.TpJpegImage * max(b, 1))()
    totals = _lib.TpJpegTotals()
    check(lib.tp_jpeg_plan((C.c_void_p * max(b, 1))(*ptrs), (C.c_int64 * max(b, 1))(*sizes), b, images, None, None, C.byref(totals)),
          "tp_jpeg_plan")
    del keep
    return [None if images[i].reason == _lib.TP_JPEG_SUPPORTED else _reason(images[i].reason) for i in range(len(data))]


def decode_jpeg_batch(data, device="cuda", *, return_status: bool = False):
    """Decode JPEG files on the GPU: a list of uint8 CUDA tensors [h, w, 3], each equal to
    ``np.array(Image.open(io.BytesIO(f)).convert('RGB'))`` bit for bit.  The outputs are views into one device buffer.

    data: a sequence of files as bytes, 1-D uint8 numpy arrays or 1-D uint8 CPU tensors.
    One host plan, one upload of the scan bytes and tables, four launches for the whole batch.  A file the plan refuses raises
    ValueError naming its index and the reason before anything runs (``jpeg_unsupported`` checks first).
    return_status: False (default) synchronises the stream and raises ValueError naming every file whose entropy-coded data was
    corrupt or truncated.  True returns ``(images, status)`` without synchronising: status is an int32 CUDA tensor [n, 4] of
    (status, sync rounds, subsequences, 0) per file, status 0 meaning the image is valid."""
    def launch(out, workspace, args, stream):
        check(lib.tp_jpeg_decode_batch(*args, stream), "tp_jpeg_decode_batch")

    rows, out, workspace, status = _plan_upload_launch(data, device, launch)
    views = [out[im.out_offset:im.out_offset + im.h * im.w * 3].view(im.h, im.w, 3) for im in rows]
    if return_status:
        return views, status
    bad = [(i, int(s)) for i, s in enumerate(status[:, 0].tolist()) if s != 0]
    if bad:
        raise ValueError("; ".join(f"file {i}: {STATUS_TEXT.get(s, f'status {s}')}" for i, s in bad))
    return views


def _plan_upload_launch(data, device, launch):
    """The plan, the upload and launch(out, workspace, args, stream), where args are tp_jpeg_decode_batch's arguments before the
    stream (the stage tests launch their own stages here).  Returns (plan rows, output bytes, workspace, status)."""
    data = list(data)
    if not data:
        raise ValueError("decode_jpeg_batch needs at least one file")
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("decode_jpeg_batch runs on a CUDA device; there is no CPU path")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    ptrs, sizes, keep = _buffers(data)
    b = len(ptrs)
    # one pinned buffer, one asynchronous copy: [plan rows | tables | staged scan bytes]; the scans need at most the files' bytes
    tab_off = (C.sizeof(_lib.TpJpegImage) * b + 15) // 16 * 16
    stg_off = tab_off + C.sizeof(_lib.TpJpegTables) * b
    total_bytes = stg_off + sum((n + 15) // 16 * 16 for n in sizes) + 16
    st = _staging(device, total_bytes)
    st["event"].synchronize()                     # the previous call's copy has left the pinned buffer
    host = st["host"]
    images = (_lib.TpJpegImage * b).from_address(host.data_ptr())
    totals = _lib.TpJpegTotals()
    check(lib.tp_jpeg_plan((C.c_void_p * b)(*ptrs), (C.c_int64 * b)(*sizes), b, images, host.data_ptr() + tab_off,
                           host.data_ptr() + stg_off, C.byref(totals)), "tp_jpeg_plan")
    del keep
    for i in range(b):
        if images[i].reason != _lib.TP_JPEG_SUPPORTED:
            raise ValueError(f"file {i}: {_reason(images[i].reason)} (decode it with PIL)")
    rows = (_lib.TpJpegImage * b)()
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
        launch(out, workspace, (C.addressof(rows), dev.data_ptr(), dev.data_ptr() + tab_off, dev.data_ptr() + stg_off, b, out.data_ptr(),
                workspace.data_ptr(), workspace.numel(), status.data_ptr()), stream.cuda_stream)
        workspace.record_stream(stream)
    return rows, out, workspace, status
