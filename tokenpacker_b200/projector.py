"""Host-side mirror of the reference projector interface (llava/model/multimodal_projector/builder.py).

``TokenPackerB200`` keeps the reference module's constructor arguments (builder.py:40-49), its parameter names and
shapes (so ``mm_projector.bin`` checkpoints load unchanged, llava_arch.py:78-83), its ``forward(x, attn_mask=None)``
signature with ``x = (feat[N,576,1024], feat_multi[N,576,4096])`` as handed over by ``CLIPVisionTower.forward``
(clip_encoder.py:62) and its ``[N, (24/s)^2, hidden]`` contiguous output (builder.py:136-137).  All arithmetic is
done by libtokenpacker_b200.so; the ``nn.Linear`` / ``nn.LayerNorm`` / ``nn.MultiheadAttention`` children below are
parameter containers only — their ``forward`` is never called.
"""
from __future__ import annotations

import ctypes as C
import warnings
from functools import partial

import torch
import torch.nn as nn
from torch.nn.init import trunc_normal_

from . import _lib
from ._lib import lib, check

_CLIP_LAYERS = 4          # builder.py:61,67: the multi-level stack is 4 CLIP layers x 1024 = 4096 (hard-coded upstream)


class IdentityMap(nn.Module):
    """builder.py:11-20 (unused upstream; kept so `from ... import IdentityMap` keeps working)."""

    def forward(self, x, *args, **kwargs):
        return x

    @property
    def config(self):
        return {"mm_projector_type": "identity"}


def _two_layer(in_dim: int, mid: int, out: int) -> nn.Sequential:
    # index 0 and 2 carry parameters, index 1 is the GELU: gives the state_dict keys "<name>.0.*" / "<name>.2.*"
    return nn.Sequential(nn.Linear(in_dim, mid), nn.GELU(), nn.Linear(mid, out))


class _ProjectorFunction(torch.autograd.Function):
    """autograd bridge: forward = tp_forward_train (keeps intermediates), backward = tp_backward (parameter gradients), or
    tp_backward_inputs when x0b / xmb need a gradient too (``TokenPackerB200.input_grad``)."""

    @staticmethod
    def forward(ctx, module, x0b, s0, xmb, sm, *params):
        device = x0b.device
        n = x0b.shape[0]
        # training: ALWAYS repack from the live parameters.  Optimizers that update through a ``.data`` alias (DeepSpeed ZeRO-2's
        # bit16 flat buffer: every reference recipe, scripts/v1_5/*.sh) change neither data_ptr nor _version, so no key can tell
        # that the weights moved; they change every step anyway and the pack is small next to forward + backward.
        # The matrices that need no transformation are read from the (bf16) parameters in place; only the fp32 biases, the
        # LayerNorm-folded in-projections and the k/v_proj.0 concatenation are rebuilt (tp_pack_weights_train).
        bf = [p.detach().to(device=device, dtype=torch.bfloat16).contiguous() for p in params]
        w_struct = _lib.TpWeights(*[t.data_ptr() for t in bf])
        stream = torch.cuda.current_stream(device).cuda_stream
        pbytes = lib.tp_packed_bytes(module.hidden_size)
        packed = torch.empty(pbytes, dtype=torch.uint8, device=device)
        check(lib.tp_pack_weights_train(C.byref(w_struct), module.hidden_size, packed.data_ptr(), pbytes, stream), "tp_pack_weights_train")
        module._packed = module._packed_key = None           # whatever the inference path cached predates this step's weights
        out = torch.empty((n, module.num_queries, module.hidden_size), dtype=torch.bfloat16, device=device)
        nbytes = lib.tp_train_saved_bytes(n, module.scale_factor, module.hidden_size)
        saved = torch.empty(nbytes, dtype=torch.uint8, device=device)
        check(lib.tp_forward_train(C.byref(w_struct), packed.data_ptr(), x0b.data_ptr(), xmb.data_ptr(), n, s0, sm, module.scale_factor,
                                   module.hidden_size, out.data_ptr(), saved.data_ptr(), nbytes, stream), "tp_forward_train")
        ctx.module = module
        ctx.saved = saved
        ctx.packed = packed if ctx.needs_input_grad[3] else None     # dxm reads [W_k0; W_v0] from it; ~80 MB at hidden 4096, else dropped
        ctx.xm = xmb if xmb.is_contiguous() else xmb.contiguous()
        ctx.weights_bf16 = bf                                # the parameters this forward read (bf16; aliases of the live ones when they are bf16)
        ctx.param_meta = [(p.dtype, p.requires_grad) for p in params]
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        module = ctx.module
        device = grad_out.device
        n = ctx.xm.shape[0]
        g = grad_out.to(torch.bfloat16).contiguous()
        grads = [torch.empty_like(w) for w in ctx.weights_bf16]
        w_struct = _lib.TpWeights(*[t.data_ptr() for t in ctx.weights_bf16])
        g_struct = _lib.TpWeights(*[t.data_ptr() for t in grads])
        need_x0, need_xm = ctx.needs_input_grad[1], ctx.needs_input_grad[3]
        d_x0 = d_xm = None
        with torch.cuda.device(device):
            ws_bytes = lib.tp_backward_workspace_bytes(n, module.scale_factor, module.hidden_size)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream
            if need_x0 or need_xm:
                d_x0 = torch.empty((n, 576, 1024), dtype=torch.bfloat16, device=device) if need_x0 else None     # every element written
                d_xm = torch.empty((n, 576, 4096), dtype=torch.bfloat16, device=device) if need_xm else None
                check(lib.tp_backward_inputs(C.byref(w_struct), ctx.packed.data_ptr() if need_xm else None, ctx.xm.data_ptr(),
                                             ctx.xm.stride(0), n, module.scale_factor, module.hidden_size, g.data_ptr(), ctx.saved.data_ptr(),
                                             C.byref(g_struct), d_x0.data_ptr() if need_x0 else None,
                                             d_xm.data_ptr() if need_xm else None, ws.data_ptr(), ws_bytes, stream), "tp_backward_inputs")
            else:
                check(lib.tp_backward(C.byref(w_struct), ctx.xm.data_ptr(), ctx.xm.stride(0), n, module.scale_factor, module.hidden_size,
                                      g.data_ptr(), ctx.saved.data_ptr(), C.byref(g_struct), ws.data_ptr(), ws_bytes, stream), "tp_backward")
        out = [gr.to(dt) if need else None for gr, (dt, need) in zip(grads, ctx.param_meta)]
        return (None, d_x0, None, d_xm, None) + tuple(out)


class _PackedScatterFunction(torch.autograd.Function):
    """Differentiable slice assembly (llava_arch.py:139-155) for the training path: crop blocks [N,M,H] -> packed rows, with the
    ',' / '\\n' rows filled in.  Forward = tp_hd_scatter_crops + tp_hd_fill_separators; backward = one row gather
    (tp_gather_rows with the forward's destination rows as source index) plus the column sums of the separator rows' gradients."""

    @staticmethod
    def forward(ctx, feats, sep_row, ret_row, seg, sep_rows, ret_rows, total_rows):
        n, m, h = feats.shape
        fb = feats.contiguous()
        out = torch.empty((total_rows, h), dtype=torch.bfloat16, device=feats.device)
        sep_b = sep_row.detach().to(device=feats.device, dtype=torch.bfloat16).contiguous()
        ret_b = ret_row.detach().to(device=feats.device, dtype=torch.bfloat16).contiguous()
        stream = torch.cuda.current_stream(feats.device).cuda_stream
        check(lib.tp_hd_scatter_crops(fb.data_ptr(), n, m, h, seg.data_ptr(), out.data_ptr(), stream), "tp_hd_scatter_crops")
        check(lib.tp_hd_fill_separators(out.data_ptr(), h, sep_rows.data_ptr(), sep_rows.numel(), sep_b.data_ptr(),
                                        ret_rows.data_ptr(), ret_rows.numel(), ret_b.data_ptr(), stream), "tp_hd_fill_separators")
        ctx.shape = (n, m, h)
        ctx.meta = (sep_row.dtype, ret_row.dtype)
        ctx.save_for_backward(seg, sep_rows, ret_rows)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        seg, sep_rows, ret_rows = ctx.saved_tensors
        n, m, h = ctx.shape
        g = g.to(torch.bfloat16).contiguous()
        src = (seg.view(n, 1) + torch.arange(m, device=g.device, dtype=torch.int64).view(1, m)).reshape(-1).contiguous()
        gf = torch.empty((n * m, h), dtype=torch.bfloat16, device=g.device)
        stream = torch.cuda.current_stream(g.device).cuda_stream
        check(lib.tp_gather_rows(g.data_ptr(), g.data_ptr(), h, src.data_ptr(), n * m, gf.data_ptr(), stream), "tp_gather_rows")
        g_sep = g.index_select(0, sep_rows).float().sum(0).to(ctx.meta[0]) if ctx.needs_input_grad[1] else None
        g_ret = g.index_select(0, ret_rows).float().sum(0).to(ctx.meta[1]) if ctx.needs_input_grad[2] else None
        return gf.view(n, m, h), g_sep, g_ret, None, None, None, None


class TokenPackerB200(nn.Module):
    def __init__(self, raw_grid=24, embed_dim=1024, num_heads=1024 // 128, kv_dim=1024, hidden_size=4096, scale_factor=2,
                 norm_layer=partial(nn.LayerNorm, eps=1e-6)):
        super().__init__()
        if raw_grid % scale_factor != 0:
            raise ValueError("scale_factor must be divisible by grid size")      # builder.py:51-52, same message
        if (raw_grid, embed_dim, num_heads, kv_dim) != (24, 1024, 8, 1024):
            raise NotImplementedError("the sm_90a kernels are specialised for CLIP-ViT-L/14-336: raw_grid=24, "
                                      "embed_dim=kv_dim=1024, num_heads=8 (the only configuration the reference builds)")
        if hidden_size % 32 != 0:
            raise NotImplementedError("hidden_size must be a multiple of 32")
        self.raw_grid = raw_grid
        self.grid_size = raw_grid // scale_factor
        self.num_queries = self.grid_size ** 2
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.scale_factor = scale_factor
        self.hidden_size = hidden_size

        self.q_proj_1 = nn.Linear(kv_dim, embed_dim, bias=False)
        self.k_proj_1 = _two_layer(_CLIP_LAYERS * 1024, 1024, 1024)
        self.v_proj_1 = _two_layer(_CLIP_LAYERS * 1024, 1024, 1024)
        self.ln_q_1 = norm_layer(embed_dim)
        self.ln_k_1 = norm_layer(embed_dim)
        self.ln_v_1 = norm_layer(embed_dim)
        self.clip_attn = nn.MultiheadAttention(embed_dim, num_heads)
        self.mlp = _two_layer(1024, hidden_size, hidden_size)
        for ln in (self.ln_q_1, self.ln_k_1, self.ln_v_1):
            if abs(ln.eps - 1e-6) > 1e-12 or not ln.elementwise_affine:
                raise NotImplementedError("norm_layer must be LayerNorm(eps=1e-6) with affine parameters")
        self.apply(self._init_weights)
        self._packed = None
        self._packed_key = None
        self._keepalive = None
        self._param_list = None
        self._warned_dtype = False
        # Gradients w.r.t. the CLIP features (unfrozen vision tower, LoRA / adapters on CLIP, attribution on the image features):
        # off by default, so that features left with requires_grad by accident keep failing loudly instead of silently costing the
        # xm gradient (a GEMM as large as the forward's largest, and [N,576,4096] bf16 of memory).  Set to True to have forward()
        # and forward_packed() carry gradients to feat / feat_multi.  Not a constructor argument and not in the state_dict.
        self.input_grad = False
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packed())

    @staticmethod
    def _init_weights(m):
        # builder.py:87-94: trunc_normal(std=.02) Linear weights, zero biases, LayerNorm (1, 0).  Like upstream this
        # leaves clip_attn.in_proj_weight at nn.MultiheadAttention's own xavier init (it is not an nn.Linear).
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    # ------------------------------------------------------------------------------------------------------------
    # derived weight cache
    # ------------------------------------------------------------------------------------------------------------
    def _raw_params(self):
        # the 23 nn.Parameter objects in tp_weights order; looked up once (walking named_parameters() costs more host time than
        # a single-image forward takes on the GPU) and again after anything that may have replaced them (invalidate_packed)
        params = self._param_list
        if params is None:
            sd = dict(self.named_parameters())
            params = self._param_list = [sd[key] for _, key in _lib.WEIGHT_FIELDS]
        return params

    def invalidate_packed(self):
        """Drop the derived weight cache.  Called automatically by load_state_dict, .to() / .cuda() / .half() (``_apply``),
        ``train()`` / ``eval()`` switches and after every training forward; call it yourself after writing parameters through a
        ``.data`` alias outside of training (such writes change neither ``data_ptr`` nor ``_version``, so no cache key sees them)."""
        self._packed = None
        self._packed_key = None
        self._param_list = None

    def _apply(self, fn, *args, **kwargs):
        self.invalidate_packed()
        return super()._apply(fn, *args, **kwargs)

    def train(self, mode: bool = True):
        self.invalidate_packed()
        return super().train(mode)

    def _packed_weights(self, device, fresh: bool = False):
        params = self._raw_params()
        key = (str(device),) + tuple((p.data_ptr(), p._version, p.dtype) for p in params)
        if not fresh and self._packed is not None and self._packed_key == key:
            return self._packed
        bf = [p.detach().to(device=device, dtype=torch.bfloat16).contiguous() for p in params]
        w = _lib.TpWeights(*[t.data_ptr() for t in bf])
        nbytes = lib.tp_packed_bytes(self.hidden_size)
        packed = torch.empty(nbytes, dtype=torch.uint8, device=device)
        stream = torch.cuda.current_stream(device).cuda_stream
        check(lib.tp_pack_weights(C.byref(w), self.hidden_size, packed.data_ptr(), nbytes, stream), "tp_pack_weights")
        self._keepalive = bf     # sources must outlive the asynchronous packing kernels
        # a pack made for a training forward is never reused (see _ProjectorFunction.forward): the next call repacks
        self._packed, self._packed_key = packed, (None if fresh else key)
        return packed

    # ------------------------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _as_crop_strided(t: torch.Tensor, width: int):
        """Return (tensor, crop_stride) with unit channel stride and dense rows; [:,1:] CLIP views pass through."""
        if t.stride(2) == 1 and t.stride(1) == width and t.stride(0) >= 576 * width and t.stride(0) % 8 == 0 \
                and t.data_ptr() % 16 == 0:
            return t, t.stride(0)
        t = t.contiguous()
        return t, t.stride(0)

    def _check_inputs(self, x, attn_mask, differentiable: bool = True):
        if attn_mask is not None:
            raise NotImplementedError("attn_mask must be None (the reference's sole caller passes none, llava_arch.py:97)")
        if not isinstance(x, (tuple, list)) or len(x) != 2:
            raise TypeError("x must be the (feat, feat_multi) pair returned by CLIPVisionTower.forward")
        x0, xm = x[0], x[1]
        if x0.dim() != 3 or xm.dim() != 3 or x0.shape[1:] != (576, 1024) or xm.shape[1:] != (576, 4096) \
                or x0.shape[0] != xm.shape[0]:
            raise ValueError(f"expected feat [N,576,1024] and feat_multi [N,576,4096], got {tuple(x0.shape)} {tuple(xm.shape)}")
        if not (x0.is_cuda and xm.is_cuda):
            raise RuntimeError("tokenpacker_b200 has no CPU path: inputs must be CUDA tensors on an H100")
        if not self._warned_dtype and (x0.dtype != torch.bfloat16 or self._raw_params()[0].dtype != torch.bfloat16):
            self._warned_dtype = True
            warnings.warn("tokenpacker_b200 computes with bf16 storage and fp32 accumulation: fp16 / fp32 inputs and parameters are cast to "
                          "bf16 at the boundary and the result is cast back (every released TokenPacker recipe runs bf16; an fp16 or "
                          "fp32 module gets bf16-precision results)", stacklevel=3)
        if torch.is_grad_enabled() and (x0.requires_grad or xm.requires_grad) and not (self.input_grad and differentiable):
            raise NotImplementedError("gradients w.r.t. the CLIP features are off by default (the vision tower is frozen in every "
                                      "released TokenPacker recipe): set `projector.input_grad = True` to have forward() / forward_packed() "
                                      "produce them, or detach the features or run under torch.no_grad()")
        return x0, xm

    def _inputs_need_grad(self, x0, xm) -> bool:
        return self.input_grad and torch.is_grad_enabled() and (x0.requires_grad or xm.requires_grad)

    def forward(self, x, attn_mask=None):
        x0, xm = self._check_inputs(x, attn_mask)
        out_dtype = x0.dtype
        n = x0.shape[0]
        device = x0.device
        if n == 0:
            return x0.new_empty((0, self.num_queries, self.hidden_size))
        with torch.cuda.device(device):
            x0b, s0 = self._as_crop_strided(x0.to(torch.bfloat16), 1024)
            xmb, sm = self._as_crop_strided(xm.to(torch.bfloat16), 4096)
            if (torch.is_grad_enabled() and any(p.requires_grad for p in self._raw_params())) or self._inputs_need_grad(x0, xm):
                # training: same output, intermediates kept, gradients for every parameter (tp_forward_train / tp_backward) and, with
                # input_grad, for the features that require one (tp_backward_inputs)
                out = _ProjectorFunction.apply(self, x0b, s0, xmb, sm, *self._raw_params())
            else:
                out = torch.empty((n, self.num_queries, self.hidden_size), dtype=torch.bfloat16, device=device)
                self._launch(x0b, s0, xmb, sm, out, None)
        return out if out_dtype == torch.bfloat16 else out.to(out_dtype)

    def _launch(self, x0b, s0, xmb, sm, out, seg_row_offset, out_crop_rows: int = 0):
        device = x0b.device
        n = x0b.shape[0]
        packed = self._packed_weights(device)
        ws_bytes = lib.tp_workspace_bytes(n, self.scale_factor, self.hidden_size)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        stream = torch.cuda.current_stream(device).cuda_stream
        if out_crop_rows:
            check(lib.tp_forward_packed(packed.data_ptr(), x0b.data_ptr(), xmb.data_ptr(), n, s0, sm, self.scale_factor,
                                        self.hidden_size, out.data_ptr(), int(out_crop_rows), ws.data_ptr(), ws_bytes, stream),
                  "tp_forward_packed")
            return
        seg_ptr = seg_row_offset.data_ptr() if seg_row_offset is not None else None
        check(lib.tp_forward(packed.data_ptr(), x0b.data_ptr(), xmb.data_ptr(), n, s0, sm, self.scale_factor,
                             self.hidden_size, out.data_ptr(), seg_ptr, ws.data_ptr(), ws_bytes, stream), "tp_forward")

    def forward_layers(self, layers):
        """Forward from the four CLIP hidden states (layers 12, 16, 22, 23; each [N,577,1024] with the CLS token, or [N,576,1024])
        WITHOUT materialising their concatenation: replaces ``feature_select`` + ``torch.cat`` (clip_encoder.py:28-44) followed by
        ``forward``; the last layer doubles as the single-level feature (select_layer = -2).  Inference only."""
        self._require_inference("forward_layers")
        if len(layers) != 4:
            raise ValueError("expected the 4 hidden states (12, 16, 22, 23)")
        views = []
        for t in layers:
            if t.dim() != 3 or t.shape[2] != 1024 or t.shape[1] not in (576, 577) or not t.is_cuda:
                raise ValueError("each layer must be a CUDA tensor [N,577,1024] or [N,576,1024]")
            t = t.to(torch.bfloat16)
            views.append(t[:, 1:] if t.shape[1] == 577 else t)
        n = views[0].shape[0]
        stride = views[0].stride(0)
        for i, v in enumerate(views):
            if v.shape[0] != n or v.stride(2) != 1 or v.stride(1) != 1024 or v.stride(0) != stride or v.data_ptr() % 16 != 0:
                views[i] = None
        if any(v is None for v in views) or stride % 8 != 0:
            views = [(t[:, 1:] if t.shape[1] == 577 else t).to(torch.bfloat16).contiguous() for t in layers]
            stride = views[0].stride(0)
        device = views[0].device
        with torch.no_grad(), torch.cuda.device(device):
            packed = self._packed_weights(device)
            out = torch.empty((n, self.num_queries, self.hidden_size), dtype=torch.bfloat16, device=device)
            ws_bytes = lib.tp_workspace_bytes(n, self.scale_factor, self.hidden_size)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            arr = (C.c_void_p * 4)(*[v.data_ptr() for v in views])
            stream = torch.cuda.current_stream(device).cuda_stream
            check(lib.tp_forward_layers(packed.data_ptr(), arr, n, stride, self.scale_factor, self.hidden_size, out.data_ptr(), None,
                                        ws.data_ptr(), ws_bytes, stream), "tp_forward_layers")
        return out

    def _require_inference(self, what: str):
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError(f"{what} is an inference path (its kernels keep no intermediates): call it under torch.no_grad(), "
                                      "or use forward() / forward_packed(), which are differentiable")

    def forward_into_peers(self, x, peer_ptrs, crop_offset: int, out_crop_rows: int = 0):
        """Fused projector + all-gather: this rank's crops are written by the last GEMM's TMA stores into the output buffer of
        every peer GPU (``peer_ptrs``: device pointers of the bf16 buffers, one per rank, mapped into this process — e.g.
        ``torch.distributed._symmetric_memory`` ``buffer_ptrs``).  ``out_crop_rows`` = 0: dense gathered [total_crops, M, H];
        = M + 1: the packed HD rows of llava_arch.py:139-155 directly (separator rows are the caller's).  Asynchronous; a cross-rank
        barrier must follow.  Inference only."""
        self._require_inference("forward_into_peers")
        x0, xm = self._check_inputs(x, None, differentiable=False)
        device = x0.device
        with torch.cuda.device(device):
            x0b, s0 = self._as_crop_strided(x0.to(torch.bfloat16), 1024)
            xmb, sm = self._as_crop_strided(xm.to(torch.bfloat16), 4096)
            n = x0b.shape[0]
            packed = self._packed_weights(device)
            ws_bytes = lib.tp_workspace_bytes(n, self.scale_factor, self.hidden_size)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream
            arr = (C.c_void_p * len(peer_ptrs))(*[int(p) for p in peer_ptrs])
            check(lib.tp_forward_allgather(packed.data_ptr(), x0b.data_ptr(), xmb.data_ptr(), n, s0, sm, self.scale_factor,
                                           self.hidden_size, arr, len(peer_ptrs), int(crop_offset), int(out_crop_rows), ws.data_ptr(),
                                           ws_bytes, stream),
                  "tp_forward_allgather")

    def forward_host(self, x, out: torch.Tensor | None = None, chunk_crops: int = 8, device=None):
        """End-to-end call with HOST tensors (pinned recommended): (feat, feat_multi) bf16 CPU tensors in, [N,M,H] bf16 CPU
        tensor out.  Host->device copies, the kernels and the device->host copy are pipelined over chunks of crops inside
        tp_forward_host; the call returns when ``out`` is complete."""
        x0, xm = x[0], x[1]
        if x0.is_cuda or xm.is_cuda or x0.dtype != torch.bfloat16 or xm.dtype != torch.bfloat16:
            raise TypeError("forward_host takes bf16 CPU tensors")
        if x0.shape[1:] != (576, 1024) or xm.shape[1:] != (576, 4096) or x0.shape[0] != xm.shape[0]:
            raise ValueError("expected feat [N,576,1024] and feat_multi [N,576,4096]")
        x0, xm = x0.contiguous(), xm.contiguous()
        n = x0.shape[0]
        device = torch.device(device if device is not None else next(self.parameters()).device)
        if device.type != "cuda":
            raise RuntimeError("tokenpacker_b200 has no CPU path: move the module to an H100 first")
        if out is None:
            out = torch.empty((n, self.num_queries, self.hidden_size), dtype=torch.bfloat16).pin_memory()
        with torch.cuda.device(device):
            packed = self._packed_weights(device)
            chunk = max(1, min(int(chunk_crops), n))
            d_x0 = torch.empty((n, 576, 1024), dtype=torch.bfloat16, device=device)
            d_xm = torch.empty((n, 576, 4096), dtype=torch.bfloat16, device=device)
            d_out = torch.empty((n, self.num_queries, self.hidden_size), dtype=torch.bfloat16, device=device)
            ws_bytes = lib.tp_workspace_bytes(chunk, self.scale_factor, self.hidden_size)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream
            check(lib.tp_forward_host(packed.data_ptr(), x0.data_ptr(), xm.data_ptr(), n, self.scale_factor, self.hidden_size,
                                      out.data_ptr(), d_x0.data_ptr(), d_xm.data_ptr(), d_out.data_ptr(), ws.data_ptr(), ws_bytes,
                                      chunk, stream), "tp_forward_host")
        return out

    def forward_packed(self, x, h_block, w_block, sep_row, ret_row):
        """Projector + HD slice assembly (llava_arch.py:139-155) in one pass.

        x as in forward(), crops ordered image by image (grid row-major, then the thumbnail); h_block / w_block:
        per-image grids; sep_row / ret_row: the ',' and '\\n' embedding rows [hidden].  Every crop of the packed sequence is
        followed by exactly one separator row, so crop i's tokens start at row i*(M+1): the last GEMM's TMA stores write them
        there directly (tp_forward_packed); the separator rows are filled by a tiny kernel.  Under autograd (training,
        pretrain_hd.sh / finetune_hd.sh use mode='slice') the same result comes from the differentiable forward plus a
        differentiable scatter.  Returns (packed [sum(L_i), hidden], cu_seqlens int64 [B+1] on the host)."""
        from .hd import hd_plan_device
        x0, xm = self._check_inputs(x, None)
        device = x0.device
        plan, seg, sep_rows, ret_rows = hd_plan_device(h_block, w_block, self.num_queries, device)
        if plan.n_crops != x0.shape[0]:
            raise ValueError(f"grids describe {plan.n_crops} crops but {x0.shape[0]} were given")
        total = int(plan.cu_seqlens[-1])
        crop_rows = self.num_queries + 1
        assert total == plan.n_crops * crop_rows      # one separator row per crop: the uniform stride the kernel relies on
        training = torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or sep_row.requires_grad
                                                or ret_row.requires_grad or self._inputs_need_grad(x0, xm))
        with torch.cuda.device(device):
            if training:
                feats = self.forward((x0, xm)).to(torch.bfloat16)
                out = _PackedScatterFunction.apply(feats, sep_row, ret_row, seg, sep_rows, ret_rows, total)
            else:
                x0b, s0 = self._as_crop_strided(x0.to(torch.bfloat16), 1024)
                xmb, sm = self._as_crop_strided(xm.to(torch.bfloat16), 4096)
                out = torch.empty((total, self.hidden_size), dtype=torch.bfloat16, device=device)
                self._launch(x0b, s0, xmb, sm, out, None, out_crop_rows=crop_rows)
                sep_b = sep_row.to(device=device, dtype=torch.bfloat16).contiguous()
                ret_b = ret_row.to(device=device, dtype=torch.bfloat16).contiguous()
                stream = torch.cuda.current_stream(device).cuda_stream
                check(lib.tp_hd_fill_separators(out.data_ptr(), self.hidden_size, sep_rows.data_ptr(), sep_rows.numel(),
                                                sep_b.data_ptr(), ret_rows.data_ptr(), ret_rows.numel(), ret_b.data_ptr(), stream),
                      "tp_hd_fill_separators")
        return (out if x0.dtype == torch.bfloat16 else out.to(x0.dtype)), plan.cu_seqlens

    def extra_repr(self):
        return f"scale_factor={self.scale_factor}, num_queries={self.num_queries}, hidden_size={self.hidden_size}, backend=sm_90a"


# the reference's class name, so `from ...builder import TokenPacker` style imports can be redirected unchanged
TokenPacker = TokenPackerB200


def build_vision_projector(config):
    """builder.py:144-145 — ignores mm_projector_type exactly like upstream."""
    return TokenPackerB200(hidden_size=config.hidden_size, scale_factor=config.scale_factor)
