"""Fused channels_last conv-block epilogues (csrc/nhwc_fused.cu): ``bias + ReLU`` and ``bias + ReLU + maxpool2x2`` with
single-pass forward and backward (the backward also produces the bias gradient, so the convolution runs bias-free)."""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F

from ..core import dtype_code, native

__all__ = ["bias_relu", "bias_relu_maxpool2", "conv_bias_relu", "fused_supported"]


def _aligned(t: torch.Tensor) -> bool:
    """The kernels read and write every tensor with 16-byte vectors."""
    return t.data_ptr() % 16 == 0


def fused_supported(x: torch.Tensor, channels: int) -> bool:
    """Whether the fused NHWC epilogue kernels accept ``x``: channels_last f16/bf16 CUDA 4-D tensor, channels a multiple of 8 that
    maps onto a 256-thread block (``256 % (channels / 8) == 0``), at most 2048, data 16-byte aligned."""
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and x.dim() == 4 and channels % 8 == 0 and channels <= 2048
            and 256 % (channels // 8) == 0 and x.is_contiguous(memory_format=torch.channels_last) and _aligned(x))


def _kernel_bias(bias: torch.Tensor) -> torch.Tensor:
    """``bias`` as the kernels read it: contiguous and 16-byte aligned. A bias that lives in a flattened bucket right after a
    tensor whose size is not a multiple of 8 is a misaligned view; it is copied (at most 2048 elements), and the copy's gradient
    flows back into the view."""
    if bias.is_contiguous() and _aligned(bias):
        return bias
    return bias.clone(memory_format=torch.contiguous_format)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


_MAX_C = 2048
_workspaces = {}


def _finish_in_kernel() -> bool:
    """Opt-in (``BAGUA_NHWC_FINALIZE=1``): the backward kernels finish the bias-gradient reduction themselves (last CTA converts
    the fp32 sums and re-zeroes the workspace) instead of a ``zeros`` fill before and a dtype cast after every launch."""
    return os.environ.get("BAGUA_NHWC_FINALIZE", "0") == "1"


def _deterministic() -> bool:
    """Under ``torch.use_deterministic_algorithms(True)`` the bias gradient is torch's (fixed-order) sum of the masked gradient the
    kernel writes, not the kernel's own atomic reduction, whose summation order varies from run to run; the rest of the backward
    is the same kernel."""
    return torch.are_deterministic_algorithms_enabled()


def _workspace(device: torch.device, stream: int) -> torch.Tensor:
    """Zeroed fp32[2048] sums + one uint32 ticket, per (device, stream): kernels on one stream run back to back and each one
    hands the buffer back zeroed, so it is allocated and cleared exactly once."""
    key = (device.index, stream)
    ws = _workspaces.get(key)
    if ws is None:
        ws = torch.zeros(_MAX_C + 4, dtype=torch.float32, device=device)
        _workspaces[key] = ws
    return ws


class _BiasReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, bias):
        N, C, H, W = y.shape
        native().bias_relu_nhwc_fwd(y.data_ptr(), bias.data_ptr(), N * H * W, C, dtype_code(y.dtype), _stream())
        ctx.mark_dirty(y)
        ctx.save_for_backward(y)
        ctx.bias_dtype = bias.dtype
        return y

    @staticmethod
    def backward(ctx, g):
        (y,) = ctx.saved_tensors
        N, C, H, W = y.shape
        g = g.contiguous(memory_format=torch.channels_last)
        gout = torch.empty_like(g, memory_format=torch.channels_last)
        if _finish_in_kernel() and not _deterministic():
            stream = _stream()
            ws = _workspace(y.device, stream)
            bias_grad = torch.empty(C, dtype=ctx.bias_dtype, device=y.device)
            native().bias_relu_nhwc_bwd_fin(g.data_ptr(), y.data_ptr(), gout.data_ptr(), ws.data_ptr(), bias_grad.data_ptr(), ws.data_ptr() + 4 * _MAX_C,
                                            N * H * W, C, dtype_code(y.dtype), stream)
            return gout, bias_grad
        bg = torch.zeros(C, dtype=torch.float32, device=y.device)
        native().bias_relu_nhwc_bwd(g.data_ptr(), y.data_ptr(), gout.data_ptr(), bg.data_ptr(), N * H * W, C, dtype_code(y.dtype), _stream())
        if _deterministic():
            bg = torch.sum(gout, dim=(0, 2, 3), dtype=torch.float32)
        return gout, bg.to(ctx.bias_dtype)


class _BiasReLUMaxPool2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias):
        N, C, H, W = x.shape
        out = torch.empty((N, C, H // 2, W // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        idx = torch.empty((N, C, H // 2, W // 2), dtype=torch.uint8, device=x.device, memory_format=torch.channels_last)
        native().bias_relu_pool_nhwc_fwd(x.data_ptr(), bias.data_ptr(), out.data_ptr(), idx.data_ptr(), N, H, W, C, dtype_code(x.dtype), _stream())
        ctx.save_for_backward(out, idx)
        ctx.in_shape = (N, C, H, W)
        ctx.bias_dtype = bias.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        out, idx = ctx.saved_tensors
        N, C, H, W = ctx.in_shape
        g = g.contiguous(memory_format=torch.channels_last)
        gin = torch.empty((N, C, H, W), dtype=out.dtype, device=out.device, memory_format=torch.channels_last)
        if _finish_in_kernel() and not _deterministic():
            stream = _stream()
            ws = _workspace(out.device, stream)
            bias_grad = torch.empty(C, dtype=ctx.bias_dtype, device=out.device)
            native().bias_relu_pool_nhwc_bwd_fin(g.data_ptr(), out.data_ptr(), idx.data_ptr(), gin.data_ptr(), ws.data_ptr(), bias_grad.data_ptr(),
                                                 ws.data_ptr() + 4 * _MAX_C, N, H, W, C, dtype_code(out.dtype), stream)
            return gin, bias_grad
        bg = torch.zeros(C, dtype=torch.float32, device=out.device)
        native().bias_relu_pool_nhwc_bwd(g.data_ptr(), out.data_ptr(), idx.data_ptr(), gin.data_ptr(), bg.data_ptr(), N, H, W, C, dtype_code(out.dtype),
                                         _stream())
        if _deterministic():   # gin holds every masked gradient exactly once (zeros elsewhere): same sum as the kernel's
            bg = torch.sum(gin, dim=(0, 2, 3), dtype=torch.float32)
        return gin, bg.to(ctx.bias_dtype)


_native_fns = [False]


def _native_functions():
    """C++ autograd Functions of the optional torch extension (opt-in ``BAGUA_NATIVE_NHWC=1``), or ``None`` (also in deterministic
    mode, which only the Python Functions implement)."""
    if _deterministic():
        return None
    if _native_fns[0] is False:
        ext = None
        if os.environ.get("BAGUA_NATIVE_NHWC", "0") == "1":
            try:
                from .. import _C_torch as ext  # built by bagua_b200/_build.py:build_torch_hooks

                ext.nhwc_init(native().nhwc_api_ptr(), _finish_in_kernel())
            except Exception as e:  # noqa: BLE001 - not built / not loadable: the Python Functions below do the same work
                import logging

                logging.getLogger(__name__).warning("bagua_b200: BAGUA_NATIVE_NHWC=1 but the torch extension is unavailable (%s); using the Python Functions", e)
                ext = None
        _native_fns[0] = ext
    return _native_fns[0]


def bias_relu(y: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """``relu(y + bias[None, :, None, None])`` in place on a channels_last f16/bf16 CUDA tensor (torch ops otherwise)."""
    if fused_supported(y, y.shape[1]) and bias.dtype == y.dtype:
        bias = _kernel_bias(bias)
        ext = _native_functions()
        if ext is not None:
            return ext.bias_relu(y, bias)
        return _BiasReLU.apply(y, bias)
    return F.relu(y + bias.view(1, -1, 1, 1))


def bias_relu_maxpool2(x: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """``max_pool2d(relu(x + bias), 2, 2)`` in one pass."""
    if fused_supported(x, x.shape[1]) and bias.dtype == x.dtype and x.shape[2] % 2 == 0 and x.shape[3] % 2 == 0:
        bias = _kernel_bias(bias)
        ext = _native_functions()
        if ext is not None:
            return ext.bias_relu_maxpool2(x, bias)
        return _BiasReLUMaxPool2.apply(x, bias)
    return F.max_pool2d(F.relu(x + bias.view(1, -1, 1, 1)), 2, 2)


def _out_hw(x: torch.Tensor, conv: torch.nn.Conv2d):
    """Spatial size of ``conv(x)`` (integer padding only — the modules the fused path accepts)."""
    out = []
    for i in range(2):
        k, s, p, d = conv.kernel_size[i], conv.stride[i], conv.padding[i], conv.dilation[i]
        out.append((x.shape[2 + i] + 2 * p - d * (k - 1) - 1) // s + 1)
    return out


def conv_bias_relu(x: torch.Tensor, conv: torch.nn.Conv2d, pool: bool = False) -> torch.Tensor:
    """Conv2d (cuDNN, bias-free) followed by the fused epilogue; falls back to the plain module sequence when unsupported."""
    if conv.bias is not None and fused_supported(x, conv.out_channels) and conv.weight.dtype == x.dtype:
        ext = _native_functions()
        if ext is not None and conv.bias.dtype == x.dtype and (not pool or (_out_hw(x, conv)[0] % 2 == 0 and _out_hw(x, conv)[1] % 2 == 0)):
            return ext.conv_bias_relu(x, conv.weight, _kernel_bias(conv.bias), list(conv.stride), list(conv.padding), list(conv.dilation), conv.groups,
                                      pool)
        y = F.conv2d(x, conv.weight, None, conv.stride, conv.padding, conv.dilation, conv.groups)
        return bias_relu_maxpool2(y, conv.bias) if pool else bias_relu(y, conv.bias)
    y = F.relu(conv(x))
    return F.max_pool2d(y, 2, 2) if pool else y
