"""Direct Python handles on individual kernels of the path (unit tests and microbenchmarks)."""
from __future__ import annotations

import torch

from ._lib import lib, check


def gemm_bf16(a: torch.Tensor, b: torch.Tensor, bias: torch.Tensor | None = None, gelu: bool = False, alpha: float = 1.0,
              out: torch.Tensor | None = None) -> torch.Tensor:
    """C[M,N] = alpha * act(A[M,K] @ B[N,K]^T + bias): the wgmma GEMM every nn.Linear of the path runs on.
    a, b: bf16 CUDA, unit inner stride; bias: fp32 [N] or None."""
    if not (a.is_cuda and b.is_cuda) or a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16:
        raise TypeError("gemm_bf16 needs bf16 CUDA tensors (no CPU path)")
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != b.shape[1] or a.stride(1) != 1 or b.stride(1) != 1:
        raise ValueError("a: [M,K], b: [N,K], unit inner stride")
    m, k = a.shape
    n = b.shape[0]
    if out is None:
        out = torch.empty((m, n), dtype=torch.bfloat16, device=a.device)
    if bias is not None:
        bias = bias.to(device=a.device, dtype=torch.float32).contiguous()
    with torch.cuda.device(a.device):
        stream = torch.cuda.current_stream(a.device).cuda_stream
        check(lib.tp_gemm_bf16(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0), m, n, k,
                               bias.data_ptr() if bias is not None else None, int(gelu), float(alpha), stream), "tp_gemm_bf16")
    return out


def gemm_tn_bf16(a: torch.Tensor, b: torch.Tensor, alpha: float = 1.0, out: torch.Tensor | None = None) -> torch.Tensor:
    """C[M,N] = alpha * A^T @ B with A: [K,M], B: [K,N] row-major bf16 (the wgrad form: contraction over rows, no transposes)."""
    if not (a.is_cuda and b.is_cuda) or a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16:
        raise TypeError("gemm_tn_bf16 needs bf16 CUDA tensors (no CPU path)")
    if a.dim() != 2 or b.dim() != 2 or a.shape[0] != b.shape[0] or a.stride(1) != 1 or b.stride(1) != 1:
        raise ValueError("a: [K,M], b: [K,N], unit inner stride")
    k, m = a.shape
    n = b.shape[1]
    if out is None:
        out = torch.empty((m, n), dtype=torch.bfloat16, device=a.device)
    with torch.cuda.device(a.device):
        stream = torch.cuda.current_stream(a.device).cuda_stream
        check(lib.tp_gemm_tn_bf16(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0), m, n, k,
                                  float(alpha), stream), "tp_gemm_tn_bf16")
    return out


def gemm_nn_bf16(a: torch.Tensor, b: torch.Tensor, alpha: float = 1.0, out: torch.Tensor | None = None) -> torch.Tensor:
    """C[M,N] = alpha * A @ B with A: [M,K], B: [K,N] row-major bf16 (the dgrad form: B is a weight as stored, no transposed copy)."""
    if not (a.is_cuda and b.is_cuda) or a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16:
        raise TypeError("gemm_nn_bf16 needs bf16 CUDA tensors (no CPU path)")
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != b.shape[0] or a.stride(1) != 1 or b.stride(1) != 1:
        raise ValueError("a: [M,K], b: [K,N], unit inner stride")
    m, k = a.shape
    n = b.shape[1]
    if out is None:
        out = torch.empty((m, n), dtype=torch.bfloat16, device=a.device)
    with torch.cuda.device(a.device):
        stream = torch.cuda.current_stream(a.device).cuda_stream
        check(lib.tp_gemm_nn_bf16(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0), m, n, k,
                                  float(alpha), stream), "tp_gemm_nn_bf16")
    return out
