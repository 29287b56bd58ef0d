"""TokenPacker-HD front end: grid selection, crop tiling and slice assembly, host side of the C ABI.

Mirrors the reference seams:
  * ``Compose([ToTensor(), Normalize(CLIP mean, std)])`` on the decoded image  llava/train/train.py:645 (folded into the tiling launch)
  * ``Image_Patch(image_size=336, patch_num).calculate(h, w)``        llava/patch_divide.py:71-105
  * the inline resize -> pad -> split -> thumbnail block              llava/train/train.py:695-731 (9 pasted copies)
  * the per-image interleaving of crop tokens with ',' / '\\n' rows   llava/model/llava_arch.py:139-155
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib
from ._lib import lib, check

BLOCK = 336


def hd_grid(h: int, w: int, patch_num: int = 9, image_size: int = BLOCK):
    hb, wb = C.c_int(0), C.c_int(0)
    check(lib.tp_hd_grid(int(h), int(w), int(patch_num), int(image_size), C.byref(hb), C.byref(wb)), "tp_hd_grid")
    return hb.value, wb.value


class Image_Patch:
    """Same constructor and ``calculate`` contract as patch_divide.py:71-105 (returns the (h_block, w_block) tuple)."""

    def __init__(self, image_size=336, patch_num=9):
        if patch_num not in (9, 16, 25):
            raise NotImplementedError                                    # patch_divide.py:79-80
        if isinstance(image_size, (tuple, list)):
            if image_size[0] != image_size[1]:
                raise NotImplementedError("square crops only (the reference always passes 336)")
            image_size = image_size[0]
        self.image_size = (image_size, image_size)
        self.patch_num = patch_num

    def calculate(self, h, w):
        return hd_grid(h, w, self.patch_num, self.image_size[0])


def hd_fit(h: int, w: int, hb: int, wb: int):
    a, b, c, d = C.c_int(0), C.c_int(0), C.c_int(0), C.c_int(0)
    check(lib.tp_hd_fit(int(h), int(w), hb, wb, C.byref(a), C.byref(b), C.byref(c), C.byref(d)), "tp_hd_fit")
    return (a.value, b.value), (c.value, d.value)


def n_crops(hb: int, wb: int) -> int:
    return hb * wb + (1 if hb * wb > 1 else 0)


def hd_tile(image: torch.Tensor, patch_num: int = 9):
    """train.py:695-731 on the GPU.  image: float32 CUDA tensor [1,3,h,w] (or [3,h,w]), already normalised.
    Returns (crops [hb*wb(+1), 3, 336, 336] float32, h_block, w_block)."""
    if image.dim() == 4:
        if image.shape[0] != 1:
            raise ValueError("one image per call: [1,3,h,w]")
        image = image[0]
    if image.dim() != 3 or image.shape[0] != 3:
        raise ValueError("image must be [1,3,h,w] or [3,h,w]")
    if not image.is_cuda:
        raise RuntimeError("tokenpacker_b200 has no CPU path: image must be a CUDA tensor")
    image = image.to(torch.float32).contiguous()
    h, w = int(image.shape[1]), int(image.shape[2])
    hb, wb = hd_grid(h, w, patch_num)
    with torch.cuda.device(image.device):
        crops = torch.empty((n_crops(hb, wb), 3, BLOCK, BLOCK), dtype=torch.float32, device=image.device)
        stream = torch.cuda.current_stream(image.device).cuda_stream
        check(lib.tp_hd_tile(image.data_ptr(), h, w, hb, wb, crops.data_ptr(), stream), "tp_hd_tile")
    return crops, hb, wb


_STAGING: dict = {}


def _staging(device, nbytes: int):
    """Pinned host + device byte buffers for the batched tiling plan, one pair per device, grown on demand.  (Calls on one device
    are expected from one stream at a time, like every other entry point of the package.)"""
    key = str(device)
    st = _STAGING.get(key)
    if st is None or st["host"].numel() < nbytes:
        cap = max(1 << 16, 1 << (nbytes - 1).bit_length())
        with torch.cuda.device(device):
            st = {"host": torch.empty(cap, dtype=torch.uint8).pin_memory(), "dev": torch.empty(cap, dtype=torch.uint8, device=device),
                  "event": torch.cuda.Event()}
            st["event"].record(torch.cuda.current_stream(device))
        _STAGING[key] = st
    return st


def hd_tile_batch(images, patch_num: int = 9, _return_launch: bool = False):
    """The tiling block for a whole batch in ONE launch (the collator cats the crops of a batch, train.py:797-800).

    images: sequence of float32 CUDA tensors [3,h,w] or [1,3,h,w] (already normalised), sizes may differ.
    Returns (crops [sum_i n_crops_i, 3, 336, 336] float32 in the reference's order — image by image, grid row-major, thumbnail
    last —, h_block list, w_block list)."""
    imgs = []
    for im in images:
        if im.dim() == 4:
            if im.shape[0] != 1:
                raise ValueError("each image is [3,h,w] or [1,3,h,w]")
            im = im[0]
        if im.dim() != 3 or im.shape[0] != 3:
            raise ValueError("each image is [3,h,w] or [1,3,h,w]")
        if not im.is_cuda:
            raise RuntimeError("tokenpacker_b200 has no CPU path: images must be CUDA tensors")
        imgs.append(im.to(torch.float32).contiguous())
    if not imgs:
        raise ValueError("empty batch")

    def launch(tables, _sources, crop_table, n, crops, stream):
        check(lib.tp_hd_tile_batch(tables, crop_table, n, crops.data_ptr(), stream), "tp_hd_tile_batch")

    crops, hb, wb, (dev, _, table_off, n) = _run_tile_batch(imgs[0].device, [(int(im.shape[1]), int(im.shape[2])) for im in imgs],
                                                             [im.data_ptr() for im in imgs], None, patch_num, torch.float32, imgs, launch)
    if _return_launch:
        # benchmark hook: (device tables, table offset, crop count) so that the kernel can be re-launched and timed on its own
        return crops, hb, wb, (dev, table_off, n)
    return crops, hb, wb


def _run_tile_batch(device, sizes, image_ptrs, sources, patch_num, out_dtype, keep_alive, launch):
    """Host side shared by the batched tiling launches: the plan (tp_hd_tile_batch_plan), its tables staged through ONE pinned buffer
    and ONE asynchronous copy, the crops, and the stream bookkeeping that keeps the source images alive until the kernel has read them.

    sizes: (h, w) per image.  image_ptrs: the float32 images of tp_hd_image, or None.  sources: per image (pixels, stride_c, stride_y,
    stride_x) of tp_hd_u8_source, staged between the image descriptors and the crop table, or None.  launch(tables, sources, crop_table,
    n_crops, crops, stream) issues the kernel (device addresses).  Returns (crops, h_block list, w_block list,
    (device tables, sources offset, crop-table offset, n_crops))."""
    b = len(sizes)
    hs = (C.c_int64 * b)(*[h for h, _ in sizes])
    ws = (C.c_int64 * b)(*[w for _, w in sizes])
    ptrs = (C.c_void_p * b)(*image_ptrs) if image_ptrs is not None else None
    hb, wb = (C.c_int * b)(), (C.c_int * b)()
    nc = C.c_int64(0)
    check(lib.tp_hd_tile_batch_plan(hs, ws, ptrs, b, int(patch_num), None, None, hb, wb, C.byref(nc)), "tp_hd_tile_batch_plan")
    desc_bytes = C.sizeof(_lib.TpHdImage) * b
    src_off = (desc_bytes + 15) // 16 * 16
    table_off = (src_off + (C.sizeof(_lib.TpHdU8Source) * b if sources is not None else 0) + 15) // 16 * 16
    total_bytes = table_off + max(nc.value, 1) * 12
    st = _staging(device, total_bytes)
    st["event"].synchronize()                     # the previous call's copy has left the pinned buffer
    host = st["host"]
    desc = (_lib.TpHdImage * b).from_address(host.data_ptr())
    check(lib.tp_hd_tile_batch_plan(hs, ws, ptrs, b, int(patch_num), desc, C.cast(host.data_ptr() + table_off, C.POINTER(C.c_int32)), hb, wb,
                                    C.byref(nc)), "tp_hd_tile_batch_plan")
    if sources is not None:
        rows = (_lib.TpHdU8Source * b).from_address(host.data_ptr() + src_off)
        for i, s in enumerate(sources):
            rows[i] = _lib.TpHdU8Source(*s)
    with torch.cuda.device(device):
        dev = st["dev"]
        dev[:total_bytes].copy_(host[:total_bytes], non_blocking=True)
        st["event"].record(torch.cuda.current_stream(device))
        crops = torch.empty((nc.value, 3, BLOCK, BLOCK), dtype=out_dtype, device=device)
        stream = torch.cuda.current_stream(device)
        launch(dev.data_ptr(), dev.data_ptr() + src_off, dev.data_ptr() + table_off, nc.value, crops, stream.cuda_stream)
        # the source images must outlive the asynchronous launch: tie them to the stream
        for t in keep_alive:
            t.record_stream(stream)
    return crops, list(hb), list(wb), (dev, src_off, table_off, nc.value)


# ToTensor() + Normalize(mean, std) of every HD recipe (train.py:645; model_vqa.py:62): the CLIP image statistics
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)

_NORM_TABLE: dict = {}


def norm_table() -> torch.Tensor:
    """float32 [3, 256] on the CPU: entry (c, u) is what ToTensor + Normalize make of byte u in channel c.

    Computed with the CPU ops torchvision runs (uint8 -> float, div(255), then sub(mean) and div(std) per channel), so every entry
    has torchvision's bits.  Not computed on the device: ATen's CUDA kernels may divide by a scalar as a multiplication by its
    reciprocal, which can differ in the last bit."""
    u = torch.arange(256, dtype=torch.uint8)
    mean = torch.tensor(CLIP_MEAN, dtype=torch.float32)
    std = torch.tensor(CLIP_STD, dtype=torch.float32)
    return (u.float().div(255) - mean[:, None]) / std[:, None]


def _norm_table_on(device) -> torch.Tensor:
    key = str(device)
    t = _NORM_TABLE.get(key)
    if t is None:
        t = _NORM_TABLE[key] = norm_table().to(device)
    return t


def hd_preprocess_batch(images, patch_num: int = 9, dtype=torch.float32, layout: str = "HWC", _return_launch: bool = False):
    """ToTensor + Normalize (train.py:645) and the tiling block (train.py:695-731) for a batch of DECODED 8-bit images, in one launch.

    images: sequence of uint8 CUDA tensors, [h, w, 3] for layout "HWC" (np.array(pil_image), what the reference decodes) or [3, h, w]
    for "CHW" (torchvision.io.decode_image); sizes may differ, and views are read through their strides, not copied.
    dtype: torch.float32, or torch.bfloat16 (the tower's dtype; equal to the float32 crops .to(torch.bfloat16), bit for bit).
    Returns (crops [sum_i n_crops_i, 3, 336, 336] in dtype, h_block list, w_block list) in the reference's crop order.  The float32
    crops have exactly the bits hd_tile_batch gives for the same images normalised on the host (norm_table)."""
    if dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"dtype must be torch.float32 or torch.bfloat16, not {dtype}")
    if layout not in ("HWC", "CHW"):
        raise ValueError(f'layout must be "HWC" or "CHW", not {layout!r}')
    images = list(images)
    if not images:
        raise ValueError("empty batch")
    cdim = 2 if layout == "HWC" else 0
    for im in images:
        if im.dtype != torch.uint8:
            raise TypeError(f"images must be uint8 (decoded pixels), not {im.dtype}")
        if im.dim() != 3 or im.shape[cdim] != 3:
            raise ValueError(f"each image is {'[h,w,3]' if layout == 'HWC' else '[3,h,w]'} for layout {layout!r}, got {tuple(im.shape)}")
        if not im.is_cuda:
            raise RuntimeError("tokenpacker_b200 has no CPU path: images must be CUDA tensors (move pinned uint8 images with .cuda(non_blocking=True))")
    device = images[0].device
    if any(im.device != device for im in images):
        raise ValueError("all images must be on one device")
    if layout == "HWC":
        sizes = [(int(im.shape[0]), int(im.shape[1])) for im in images]
        sources = [(im.data_ptr(), im.stride(2), im.stride(0), im.stride(1)) for im in images]
    else:
        sizes = [(int(im.shape[1]), int(im.shape[2])) for im in images]
        sources = [(im.data_ptr(), im.stride(0), im.stride(1), im.stride(2)) for im in images]
    table = _norm_table_on(device)
    out_dtype = 0 if dtype == torch.float32 else 1

    def launch(tables, srcs, crop_table, n, crops, stream):
        check(lib.tp_hd_preprocess_batch(tables, srcs, crop_table, n, table.data_ptr(), out_dtype, crops.data_ptr(), stream), "tp_hd_preprocess_batch")

    crops, hb, wb, plan = _run_tile_batch(device, sizes, None, sources, patch_num, dtype, images, launch)
    if _return_launch:
        # benchmark hook: (device tables, sources offset, crop-table offset, crop count, device norm table)
        return crops, hb, wb, plan + (table,)
    return crops, hb, wb


def hd_seq_len(hb: int, wb: int, m: int) -> int:
    return hb * wb * m + hb * (wb - 1) + hb + ((m + 1) if hb * wb > 1 else 0)


@dataclass
class HdPlan:
    n_crops: int
    seg_row_offset: torch.Tensor   # int64 [n_crops]   destination row of each crop's first token
    sep_rows: torch.Tensor         # int64 [n_sep]     rows holding the ',' embedding
    ret_rows: torch.Tensor         # int64 [n_ret]     rows holding the '\n' embedding
    cu_seqlens: torch.Tensor       # int64 [B+1]


def hd_plan(h_block, w_block, tokens_per_crop: int) -> HdPlan:
    hb = [int(v) for v in h_block]
    wb = [int(v) for v in w_block]
    if len(hb) != len(wb):
        raise ValueError("h_block and w_block must have the same length")
    b = len(hb)
    arr = C.c_int * max(b, 1)
    hb_c, wb_c = arr(*hb), arr(*wb)
    nc, ns, nr = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    check(lib.tp_hd_plan(hb_c, wb_c, b, tokens_per_crop, None, None, None, None, C.byref(nc), C.byref(ns), C.byref(nr)), "tp_hd_plan")
    seg = torch.empty(nc.value, dtype=torch.int64)
    sep = torch.empty(ns.value, dtype=torch.int64)
    ret = torch.empty(nr.value, dtype=torch.int64)
    cu = torch.empty(b + 1, dtype=torch.int64)
    p64 = C.POINTER(C.c_int64)
    check(lib.tp_hd_plan(hb_c, wb_c, b, tokens_per_crop, C.cast(seg.data_ptr(), p64), C.cast(sep.data_ptr(), p64),
                         C.cast(ret.data_ptr(), p64), C.cast(cu.data_ptr(), p64), C.byref(nc), C.byref(ns), C.byref(nr)), "tp_hd_plan")
    return HdPlan(nc.value, seg, sep, ret, cu)


_PLAN_CACHE: dict = {}


def hd_plan_device(h_block, w_block, tokens_per_crop: int, device):
    """hd_plan with its index tensors resident on ``device`` (cached per grid signature: serving loops reuse the same few
    grids, and the three small synchronous H2D copies would otherwise sit on the critical path of every call)."""
    key = (tuple(int(v) for v in h_block), tuple(int(v) for v in w_block), int(tokens_per_crop), str(device))
    hit = _PLAN_CACHE.get(key)
    if hit is None:
        plan = hd_plan(h_block, w_block, tokens_per_crop)
        hit = (plan, plan.seg_row_offset.to(device), plan.sep_rows.to(device), plan.ret_rows.to(device))
        if len(_PLAN_CACHE) > 256:
            _PLAN_CACHE.clear()
        _PLAN_CACHE[key] = hit
    return hit


def hd_assemble(feats: torch.Tensor, h_block, w_block, sep_row: torch.Tensor, ret_row: torch.Tensor):
    """llava_arch.py:139-155 for already-projected crop features [sum(crops), M, H] (bf16, CUDA).

    Standalone form of the assembly (used after the multi-GPU all-gather); ``TokenPackerB200.forward_packed`` fuses
    the same scatter into the projector's last GEMM instead.  Returns (packed [sum(L_i), H], cu_seqlens)."""
    if not feats.is_cuda:
        raise RuntimeError("tokenpacker_b200 has no CPU path: feats must be a CUDA tensor")
    m, hdim = int(feats.shape[1]), int(feats.shape[2])
    device = feats.device
    plan, seg, sep_rows, ret_rows = hd_plan_device(h_block, w_block, m, device)
    if plan.n_crops != feats.shape[0]:
        raise ValueError(f"grids describe {plan.n_crops} crops but {feats.shape[0]} were given")
    if torch.is_grad_enabled() and (feats.requires_grad or sep_row.requires_grad or ret_row.requires_grad):
        from .projector import _PackedScatterFunction      # training: differentiable scatter (gradient = one row gather)
        with torch.cuda.device(device):
            out = _PackedScatterFunction.apply(feats.to(torch.bfloat16), sep_row, ret_row, seg, sep_rows, ret_rows, int(plan.cu_seqlens[-1]))
        return (out if feats.dtype == torch.bfloat16 else out.to(feats.dtype)), plan.cu_seqlens
    fb = feats.to(torch.bfloat16).contiguous()
    with torch.cuda.device(device):
        out = torch.empty((int(plan.cu_seqlens[-1]), hdim), dtype=torch.bfloat16, device=device)
        stream = torch.cuda.current_stream(device).cuda_stream
        check(lib.tp_hd_scatter_crops(fb.data_ptr(), plan.n_crops, m, hdim, seg.data_ptr(), out.data_ptr(), stream), "tp_hd_scatter_crops")
        sep_b = sep_row.to(device=device, dtype=torch.bfloat16).contiguous()
        ret_b = ret_row.to(device=device, dtype=torch.bfloat16).contiguous()
        check(lib.tp_hd_fill_separators(out.data_ptr(), hdim, sep_rows.data_ptr(), sep_rows.numel(), sep_b.data_ptr(),
                                        ret_rows.data_ptr(), ret_rows.numel(), ret_b.data_ptr(), stream), "tp_hd_fill_separators")
    return (out if feats.dtype == torch.bfloat16 else out.to(feats.dtype)), plan.cu_seqlens
