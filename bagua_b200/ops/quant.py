"""MinMaxUInt8 compression: kernel wrappers, a pure-torch implementation (oracle + CPU path) and the
``torch.distributed`` fallbacks of the two quantised collectives.

Wire format and rounding follow the reference (kernels/bagua_kernels.cu:456-501, tests/internal/compressor.py:4-33):
per chunk ``[min:T][max:T][pad → 32 B][u8 payload padded → 32 B]``; ``scale = 255/(max-min+1e-7)``,
``upper = rint(max*scale)``, ``lower = upper-255``, ``q = min(rint(x*scale), upper) - lower``, ``x' = (q+lower)/scale``.
"""
from __future__ import annotations

from typing import Tuple

import torch
import torch.distributed as dist

from ..core import dtype_code, native

EPS = 1e-7
LEVELS = 255.0


def _align32(x: int) -> int:
    return (x + 31) // 32 * 32


def chunk_bytes(chunk_elems: int) -> int:
    """Wire size of one MinMaxUInt8 chunk: 32-byte header (min, max) + payload padded to 32 bytes."""
    return _align32(chunk_elems) + 32


def compressed_size(numel: int, n_chunks: int) -> int:
    """Bytes of the compressed buffer (reference datatypes/mod.rs:703-739)."""
    return n_chunks * chunk_bytes(numel // n_chunks)


# ---- torch implementation (oracle / CPU) --------------------------------------------------------------------
def _scale(mn: torch.Tensor, mx: torch.Tensor) -> torch.Tensor:
    # a true fp32 division like the kernel's 255/(max-min+eps) — `255.0 / tensor` would be reciprocal()*255 (two roundings)
    return torch.div(torch.full_like(mx, LEVELS), (mx - mn) + torch.full_like(mx, EPS))


def torch_compress_chunk(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Returns (minmax[2] in x.dtype, uint8 levels) for one chunk."""
    xf = x.float()
    mn, mx = xf.min(), xf.max()
    scale = _scale(mn, mx)
    upper = torch.round(mx * scale)
    lower = upper - LEVELS
    level = torch.minimum(torch.round(xf * scale), upper)
    # round-half-even can put min·scale 256 levels below upper (both products end in .5): the GPU's float→uint8 conversion
    # saturates that −1 to 0; torch's CPU cast would wrap it to 255, so clamp explicitly
    return torch.stack([mn, mx]).to(x.dtype), (level - lower).clamp_(0, LEVELS).to(torch.uint8)


def torch_decompress_chunk(minmax: torch.Tensor, q: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Inverse of :func:`torch_compress_chunk`: ``(q + lower) / scale`` in ``dtype``."""
    mn, mx = minmax[0].float(), minmax[1].float()
    scale = _scale(mn, mx)
    upper = torch.round(mx * scale)
    lower = upper - LEVELS
    return ((q.float() + lower) / scale).to(dtype)


def torch_compress(x: torch.Tensor, n_chunks: int) -> torch.Tensor:
    """Whole wire buffer for ``x`` split in ``n_chunks`` (any device)."""
    assert x.numel() % n_chunks == 0
    c = x.numel() // n_chunks
    cb = chunk_bytes(c)
    out = torch.zeros(n_chunks * cb, dtype=torch.uint8, device=x.device)
    es = x.element_size()
    for j, chunk in enumerate(x.reshape(-1).chunk(n_chunks)):
        mm, q = torch_compress_chunk(chunk)
        out[j * cb : j * cb + 2 * es] = mm.view(torch.uint8)
        out[j * cb + 32 : j * cb + 32 + c] = q
    return out


def torch_decompress(buf: torch.Tensor, numel: int, n_chunks: int, dtype: torch.dtype) -> torch.Tensor:
    """Decode a whole wire buffer of ``n_chunks`` chunks back into ``numel`` elements of ``dtype`` (any device)."""
    c = numel // n_chunks
    cb = chunk_bytes(c)
    es = torch.empty(0, dtype=dtype).element_size()
    outs = []
    for j in range(n_chunks):
        mm = buf[j * cb : j * cb + 2 * es].clone().view(dtype)
        outs.append(torch_decompress_chunk(mm, buf[j * cb + 32 : j * cb + 32 + c], dtype))
    return torch.cat(outs)


# ---- kernel wrappers ------------------------------------------------------------------------------------------
def compress(x: torch.Tensor, n_chunks: int = 1, target_chunk: int = -1, out: torch.Tensor | None = None) -> torch.Tensor:
    """MinMaxUInt8-compress ``x`` (sm_90a kernel on CUDA tensors, torch elsewhere)."""
    assert x.is_contiguous() and x.numel() % n_chunks == 0
    if x.device.type != "cuda":
        full = torch_compress(x, n_chunks)
        if out is not None:
            out.copy_(full)
            return out
        return full
    C = native()
    if out is None:
        out = torch.zeros(compressed_size(x.numel(), n_chunks), dtype=torch.uint8, device=x.device)
    scratch = torch.empty(2 * n_chunks, dtype=torch.float32, device=x.device)
    C.minmax_uint8_compress(x.data_ptr(), x.numel(), dtype_code(x.dtype), n_chunks, target_chunk, out.data_ptr(), scratch.data_ptr(),
                            torch.cuda.current_stream().cuda_stream)
    return out


def decompress(buf: torch.Tensor, out: torch.Tensor, n_chunks: int = 1) -> torch.Tensor:
    """Inverse of :func:`compress` into ``out`` (its dtype/numel define the layout)."""
    assert out.is_contiguous() and out.numel() % n_chunks == 0
    if out.device.type != "cuda":
        out.copy_(torch_decompress(buf, out.numel(), n_chunks, out.dtype).view_as(out))
        return out
    native().minmax_uint8_decompress(buf.data_ptr(), out.numel(), dtype_code(out.dtype), n_chunks, out.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream)
    return out


# ---- torch.distributed fallbacks of the fused collectives ---------------------------------------------------
def bytegrad_allreduce_fallback(bucket, pg, average: bool):
    """The reference's 7-step ByteGrad pipeline (comm_ops/centralized_low_precision_synchronous.rs:22-73) on
    ``torch.distributed``: compress → alltoall → decompress → chunk-reduce → compress own chunk → allgather → decompress."""
    flat, scatter_back = bucket._flat_or_gather()
    n = pg.size()
    c = pg.get_global_communicator()
    r = c.rank()
    numel = flat.numel()
    assert numel % n == 0, "ByteGrad buckets are padded to a multiple of nranks"
    chunk = numel // n
    cb = chunk_bytes(chunk)
    with torch.no_grad():
        q = compress(flat, n)
        recv = torch.empty_like(q)
        c.alltoall(q, recv)
        tmp = torch.empty_like(flat)
        decompress(recv, tmp, n)  # tmp[j] = peer j's version of my chunk
        red = tmp.view(n, chunk).float().sum(dim=0)
        if average:
            red = red / n
        mine = red.to(flat.dtype).contiguous()
        q2 = compress(mine, 1)
        gathered = torch.empty(n * cb, dtype=torch.uint8, device=flat.device)
        c.allgather(q2, gathered)
        decompress(gathered, flat, n)
    if scatter_back is not None:
        scatter_back()


def low_precision_ring_fallback(bucket, pg, weight, left, right):
    """Ring step of low-precision decentralized SGD (comm_ops/decentralized_low_precision_synchronous.rs:28-153)."""
    x, scatter_back = bucket._flat_or_gather()
    n = pg.size()
    c = pg.get_global_communicator()
    r = c.rank()
    lp, rp = (r + n - 1) % n, (r + 1) % n
    with torch.no_grad():
        x.add_(left.view(-1), alpha=1.0 / 3.0)
        x.add_(right.view(-1), alpha=1.0 / 3.0)
        x.sub_(weight.view(-1), alpha=5.0 / 3.0)
        q = compress(x, 1)
        ql, qr = torch.empty_like(q), torch.empty_like(q)
        reqs = [
            dist.isend(q, c._global(lp), group=pg.torch_group),
            dist.isend(q, c._global(rp), group=pg.torch_group),
            dist.irecv(ql, c._global(lp), group=pg.torch_group),
            dist.irecv(qr, c._global(rp), group=pg.torch_group),
        ]
        for req in reqs:
            req.wait()
        tmp = torch.empty_like(x)
        left.view(-1).add_(decompress(ql, tmp, 1))
        right.view(-1).add_(decompress(qr, tmp, 1))
        decompress(q, x, 1)
        x.add_(weight.view(-1))
        weight.view(-1).copy_(x)
    if scatter_back is not None:
        scatter_back()
