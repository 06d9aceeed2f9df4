"""Grouped linear layers on the hand-written wgmma/TMA GEMM (csrc/gemm_wgmma.cu).

``grouped_linear(x[G,M,K], w[G,N,K], bias[G,N]) -> [G,M,N]`` computes ``x @ w^T + bias`` per group (per local expert).
Forward and both backward GEMMs run on the same TN kernel (operands are brought into K-contiguous form with a transpose
copy, which costs a few µs next to a multi-GFLOP GEMM).  Shapes the kernel does not cover (CPU tensors, non-bf16,
M/N not multiples of 128, K not a multiple of 64) fall back to ``torch.baddbmm``.
"""
from __future__ import annotations

from typing import Optional

import torch

from ..core import native

__all__ = ["grouped_linear", "grouped_gemm_tn", "tcgen05_supported"]


def tcgen05_supported(x: torch.Tensor, M: int, N: int, K: int) -> bool:
    """Whether the wgmma grouped GEMM handles this problem (the name is historical): bf16 CUDA operands, ``M % 128 == 0``, ``N % 128 == 0``, ``K % 64 == 0``."""
    return x.is_cuda and x.dtype == torch.bfloat16 and native().grouped_gemm_supported(M, N, K)


def grouped_gemm_tn(a: torch.Tensor, b: torch.Tensor, bias: Optional[torch.Tensor] = None, act: str = "none") -> torch.Tensor:
    """``out[g] = act(a[g] @ b[g]^T + bias[g])`` with a [G,M,K], b [G,N,K] contiguous bf16 CUDA tensors (wgmma kernel)."""
    G, M, K = a.shape
    N = b.shape[1]
    assert b.shape[0] == G and b.shape[2] == K and a.is_contiguous() and b.is_contiguous()
    out = torch.empty(G, M, N, dtype=torch.bfloat16, device=a.device)
    bias32 = bias.float().contiguous() if bias is not None else None
    native().grouped_gemm_tn(a.data_ptr(), b.data_ptr(), out.data_ptr(), bias32.data_ptr() if bias32 is not None else 0, G, M, N, K,
                             {"none": 0, "gelu": 1}[act], torch.cuda.current_stream().cuda_stream)
    return out


class _GroupedLinear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias):
        ctx.save_for_backward(x, w)
        ctx.has_bias = bias is not None
        return grouped_gemm_tn(x.contiguous(), w.contiguous(), bias)

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        gy = gy.contiguous()
        G, M, K = x.shape
        N = w.shape[1]
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            # dX[M,K] = dY[M,N] @ W[N,K]  →  TN form with B = W^T [K,N]
            gx = grouped_gemm_tn(gy, w.transpose(1, 2).contiguous()) if tcgen05_supported(gy, M, K, N) else torch.bmm(gy, w)
        if ctx.needs_input_grad[1]:
            # dW[N,K] = dY^T[N,M] @ X[M,K]  →  TN form with A = dY^T [N,M], B = X^T [K,M]
            if tcgen05_supported(gy, N, K, M):
                gw = grouped_gemm_tn(gy.transpose(1, 2).contiguous(), x.transpose(1, 2).contiguous())
            else:
                gw = torch.bmm(gy.transpose(1, 2), x)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = gy.float().sum(dim=1).to(gy.dtype)
        return gx, gw, gb


def grouped_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Per-group linear layer: ``x[G,M,K] @ w[G,N,K]^T + bias[G,N]``."""
    G, M, K = x.shape
    N = w.shape[1]
    if tcgen05_supported(x, M, N, K) and w.dtype == torch.bfloat16:
        return _GroupedLinear.apply(x, w, bias)
    out = torch.bmm(x, w.transpose(1, 2))
    return out + bias.unsqueeze(1) if bias is not None else out
