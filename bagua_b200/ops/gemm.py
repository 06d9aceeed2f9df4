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


def _check_grouped_shapes(a: torch.Tensor, b: torch.Tensor, bias: Optional[torch.Tensor], names=("a", "b")):
    """a [G,M,K] and b [G,N,K] agree in G and K; ``bias`` is None or a floating [G,N] tensor (one row per group: the kernel reads
    ``bias[g * N + n]``, so a shared [N] bias would be read past its end)."""
    na, nb = names
    if a.dim() != 3 or b.dim() != 3:
        raise ValueError(f"{na} and {nb} must be 3-D [G, M, K] and [G, N, K], got {tuple(a.shape)} and {tuple(b.shape)}")
    G, _, K = a.shape
    if b.shape[0] != G or b.shape[2] != K:
        raise ValueError(f"{nb} must be [G={G}, N, K={K}] to match {na} {tuple(a.shape)}, got {tuple(b.shape)}")
    if bias is not None:
        if not bias.is_floating_point():
            raise TypeError(f"bias must be a floating-point tensor, got {bias.dtype}")
        if tuple(bias.shape) != (G, b.shape[1]):
            raise ValueError(f"bias must be [G={G}, N={b.shape[1]}] (one row per group), got {tuple(bias.shape)}")


def grouped_gemm_tn(a: torch.Tensor, b: torch.Tensor, bias: Optional[torch.Tensor] = None, act: str = "none") -> torch.Tensor:
    """``out[g] = act(a[g] @ b[g]^T + bias[g])`` with a [G,M,K], b [G,N,K] contiguous bf16 CUDA tensors (wgmma kernel), ``bias``
    a floating [G,N] tensor on the same device (read as fp32), ``act`` "none" or "gelu" (tanh form).  Anything else raises
    before the kernel is launched."""
    _check_grouped_shapes(a, b, bias)
    G, M, K = a.shape
    N = b.shape[1]
    if G < 1:
        raise ValueError(f"a must hold at least one group, got G={G}")
    for name, t in (("a", a), ("b", b)):
        if t.dtype != torch.bfloat16:
            raise TypeError(f"{name} must be bfloat16, got {t.dtype}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    if act not in ("none", "gelu"):
        raise ValueError(f"act must be 'none' or 'gelu', got {act!r}")
    for name, t in (("b", b), ("bias", bias)):
        if t is not None and t.device != a.device:
            raise ValueError(f"{name} is on {t.device}, a on {a.device}: all operands must be on one device")
    if not a.is_cuda:
        raise ValueError(f"a must be a CUDA tensor, got one on {a.device}")
    if not native().grouped_gemm_supported(M, N, K):
        raise ValueError(f"grouped_gemm_tn needs M % 128 == 0, N % 128 == 0 and K % 64 == 0, got M={M}, N={N}, K={K}")
    for name, t in (("a", a), ("b", b)):
        if t.data_ptr() % 16:
            raise ValueError(f"{name} must be 16-byte aligned")
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
        ctx.bias_dtype = bias.dtype if bias is not None else None
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
            gb = gy.float().sum(dim=1).to(ctx.bias_dtype)   # summed in fp32, returned in the bias's own dtype
        return gx, gw, gb


def grouped_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Per-group linear layer: ``x[G,M,K] @ w[G,N,K]^T + bias[G,N]`` (``bias`` must be [G,N] on both paths)."""
    _check_grouped_shapes(x, w, bias, names=("x", "w"))
    G, M, K = x.shape
    N = w.shape[1]
    if tcgen05_supported(x, M, N, K) and w.dtype == torch.bfloat16:
        return _GroupedLinear.apply(x, w, bias)
    out = torch.bmm(x, w.transpose(1, 2))
    return out + bias.unsqueeze(1) if bias is not None else out
