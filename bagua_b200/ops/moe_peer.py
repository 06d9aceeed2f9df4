"""NVSwitch path of MoE dispatch/combine: autograd functions over the peer scatter/gather kernels (csrc/moe_kernels.cu).

Forward and backward each need one *scatter* (rows pushed into the owner GPU's capacity slots) and one *gather* (rows pulled
from the owners, weighted and summed):

=================  =============================================  ==========================================
                   forward                                        backward
=================  =============================================  ==========================================
dispatch           scatter(tokens)                                gather(grad_dispatched, w=1)
combine            gather(expert_out, w) (+ keeps fetched rows)   scatter(grad_out · w)  and  grad_w = <grad_out, fetched rows>
=================  =============================================  ==========================================

Two symmetric buffers per (group, shape) are shared by all MoE layers: results are copied out right away (a 16 MiB copy
is ~5 µs of HBM time) so the buffers can be recycled by the next layer.  The kernels run on the *current* (compute)
stream with the group's own signal pads, in the same order on every rank.
"""
from __future__ import annotations

import logging
import os
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist

from ..core import dtype_code, native

logger = logging.getLogger(__name__)
_contexts: Dict[int, Optional["MoEPeerContext"]] = {}


class MoEPeerContext:
    """Symmetric buffers + kernel wrappers of one process group's MoE exchange (scatter / gather / GEMM-push over peer memory)."""
    def __init__(self, engine):
        self.engine = engine
        self.comm = engine.comm
        self.world = engine.world
        self.rank = engine.rank
        self._buffers: Dict[int, tuple] = {}
        self.blocks = int(os.environ.get("BAGUA_MOE_BLOCKS", "64"))

    def _buf(self, nbytes: int, which: int, key=None):
        """Symmetric buffer for an exchange.  ``key is None``: the pair shared by every call site of this size (results must be
        copied out before the next exchange).  With a ``key`` (one per MoE layer and direction) the call site OWNS its buffer —
        16 MiB per layer for GPT-2-medium MoE-8, nothing next to 80 GB — so the received rows are used in place: no ``clone``
        behind the scatter.  Reuse is safe across iterations: a layer's next scatter opens with a cross-GPU barrier that every rank
        reaches only after (stream order) it has finished the previous iteration's backward, the last reader of the buffer."""
        pair = self._buffers.get((nbytes, key))
        if pair is None:
            if key is None:
                pair = (self.engine.alloc(nbytes), self.engine.alloc(nbytes))  # collective: identical call sequence on all ranks
            else:
                one = self.engine.alloc(nbytes)
                pair = (one, one)
            self._buffers[(nbytes, key)] = pair
        return pair[which]

    # -- raw kernels ------------------------------------------------------------------------------------------------------
    def scatter(self, rows: torch.Tensor, expert_idx, slot_idx, scale: Optional[torch.Tensor], E_local: int, C: int, key=None) -> torch.Tensor:
        """rows[S, M] → local view [world, E_local, C, M] of what every rank sent to my experts (``key``: see :meth:`_buf`)."""
        S, M = rows.shape
        K = expert_idx.shape[1]
        nbytes = self.world * E_local * C * M * rows.element_size()
        buf = self._buf(nbytes, 0, key)
        rows = rows.contiguous()
        native().moe_scatter(self.comm, buf.buf, buf.offset, rows.data_ptr(), expert_idx.data_ptr(), slot_idx.data_ptr(),
                             scale.data_ptr() if scale is not None else 0, S, K, M, E_local, C, dtype_code(rows.dtype), self.blocks,
                             torch.cuda.current_stream().cuda_stream)
        if key is None:
            return buf.view(rows.dtype, self.world * E_local * C * M).view(self.world, E_local, C, M).clone()
        # in-place use of the layer's own receive buffer: a tensor over the same bytes with its OWN autograd version counter (every
        # slice of a slab is a view of one base tensor, so an in-place torch op on any other slice would otherwise mark these rows,
        # which autograd saves for the expert GEMMs' backward, as "modified")
        raw = buf.tensor
        es = rows.element_size()
        return torch.empty(0, dtype=rows.dtype, device=rows.device).set_(raw.untyped_storage(), raw.storage_offset() // es, (self.world, E_local, C, M))

    def gather(self, owner_rows: torch.Tensor, expert_idx, slot_idx, weights: Optional[torch.Tensor], S: int, keep_rows: bool,
               E_local: int, C: int) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """owner_rows [world, E_local, C, M] (what my experts produced for every source rank) → out[S, M] on the source ranks."""
        M = owner_rows.shape[-1]
        K = expert_idx.shape[1]
        nbytes = owner_rows.numel() * owner_rows.element_size()
        buf = self._buf(nbytes, 1)
        buf.view(owner_rows.dtype, owner_rows.numel()).copy_(owner_rows.reshape(-1))
        out = torch.empty(S, M, dtype=owner_rows.dtype, device=owner_rows.device)
        picked = torch.empty(S, K, M, dtype=owner_rows.dtype, device=owner_rows.device) if keep_rows else None
        native().moe_gather(self.comm, buf.buf, buf.offset, out.data_ptr(), expert_idx.data_ptr(), slot_idx.data_ptr(),
                            weights.data_ptr() if weights is not None else 0, picked.data_ptr() if picked is not None else 0, S, K, M, E_local, C,
                            dtype_code(owner_rows.dtype), self.blocks, torch.cuda.current_stream().cuda_stream)
        return out, picked

    def linear_push_gather(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], expert_idx, slot_idx, weights: torch.Tensor, S: int,
                           C: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """``combine(linear(x))`` with the all-to-all inside the GEMM: x [E_local, world*C, K] (rows ordered [source rank][slot]),
        w [E_local, N, K].  The wgmma GEMM's epilogue stores every 128-row tile straight into the symmetric buffer of the
        rank the tokens came from; the local-layout gather (which opens with the peer barrier) then forms
        out[s] = Σ_k weights[s,k] · row.  Returns (out [S, N], picked [S, k, N])."""
        from .gemm import _check_grouped_shapes

        _check_grouped_shapes(x, w, bias, names=("x", "w"))
        E_local, _, Kdim = x.shape
        N = w.shape[1]
        K = expert_idx.shape[1]
        nbytes = self.world * E_local * C * N * x.element_size()
        buf = self._buf(nbytes, 1)
        bias32 = bias.float().contiguous() if bias is not None else None
        stream = torch.cuda.current_stream().cuda_stream
        native().grouped_gemm_tn_push(x.data_ptr(), w.data_ptr(), bias32.data_ptr() if bias32 is not None else 0, E_local, N, Kdim, 0, self.comm, buf.buf,
                                      buf.offset, C, stream)
        out = torch.empty(S, N, dtype=x.dtype, device=x.device)
        picked = torch.empty(S, K, N, dtype=x.dtype, device=x.device)
        native().moe_gather(self.comm, buf.buf, buf.offset, out.data_ptr(), expert_idx.data_ptr(), slot_idx.data_ptr(), weights.data_ptr(),
                            picked.data_ptr(), S, K, N, E_local, C, dtype_code(x.dtype), self.blocks, stream, True)
        return out, picked

    def fused_combine_supported(self, x: torch.Tensor, N: int, C: int) -> bool:
        Kdim = x.shape[-1]
        return (x.is_cuda and x.dtype == torch.bfloat16 and C % 128 == 0 and native().grouped_gemm_supported(self.world * C, N, Kdim)
                and os.environ.get("BAGUA_MOE_FUSED_COMBINE", "0") == "1")

    # -- autograd ------------------------------------------------------------------------------------------------------
    def dispatch(self, tokens, expert_idx, slot_idx, num_experts: int, capacity: int, num_local_experts: int, key=None):
        return _Dispatch.apply(tokens, expert_idx.contiguous(), slot_idx.contiguous(), self, num_local_experts, capacity, key)

    def combine(self, expert_out, expert_idx, slot_idx, weights, num_experts: int, capacity: int, num_local_experts: int, key=None):
        return _Combine.apply(expert_out, weights, expert_idx.contiguous(), slot_idx.contiguous(), self, num_local_experts, capacity, key)


class _Dispatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tokens, expert_idx, slot_idx, pctx: MoEPeerContext, E_local: int, C: int, key=None):
        ctx.pctx, ctx.E_local, ctx.C, ctx.S = pctx, E_local, C, tokens.shape[0]
        ctx.save_for_backward(expert_idx, slot_idx)
        return pctx.scatter(tokens, expert_idx, slot_idx, None, E_local, C, key=(key, "dispatch") if key is not None else None)

    @staticmethod
    def backward(ctx, grad_dispatched):
        expert_idx, slot_idx = ctx.saved_tensors
        g, _ = ctx.pctx.gather(grad_dispatched.contiguous(), expert_idx, slot_idx, None, ctx.S, False, ctx.E_local, ctx.C)
        return g, None, None, None, None, None, None


class _Combine(torch.autograd.Function):
    @staticmethod
    def forward(ctx, expert_out, weights, expert_idx, slot_idx, pctx: MoEPeerContext, E_local: int, C: int, key=None):
        S = expert_idx.shape[0]
        w32 = weights.float().contiguous()
        out, picked = pctx.gather(expert_out.contiguous(), expert_idx, slot_idx, w32, S, True, E_local, C)
        ctx.pctx, ctx.E_local, ctx.C = pctx, E_local, C
        ctx.key = key
        ctx.wdtype = weights.dtype
        ctx.save_for_backward(expert_idx, slot_idx, w32, picked)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        expert_idx, slot_idx, w32, picked = ctx.saved_tensors
        grad_out = grad_out.contiguous()
        valid = (slot_idx >= 0).to(torch.float32)
        grad_w = (picked.float() * grad_out.float().unsqueeze(1)).sum(-1) * valid
        grad_rows = ctx.pctx.scatter(grad_out, expert_idx, slot_idx, (w32 * valid).contiguous(), ctx.E_local, ctx.C,
                                     key=(ctx.key, "combine_bwd") if ctx.key is not None else None)
        return grad_rows, grad_w.to(ctx.wdtype), None, None, None, None, None, None


class _LinearCombine(torch.autograd.Function):
    """``combine(grouped_linear(x, w, b))`` with the combine all-to-all fused into the GEMM epilogue (forward).  Backward is
    the mirror image built from the existing pieces: scatter(grad_out · weight) to the owners, then the two backward GEMMs."""

    @staticmethod
    def forward(ctx, x, w, bias, weights, expert_idx, slot_idx, pctx: "MoEPeerContext", C: int):
        S = expert_idx.shape[0]
        x, w = x.contiguous(), w.contiguous()
        w32 = weights.float().contiguous()
        out, picked = pctx.linear_push_gather(x, w, bias, expert_idx, slot_idx, w32, S, C)
        ctx.pctx, ctx.C, ctx.wdtype, ctx.has_bias = pctx, C, weights.dtype, bias is not None
        ctx.bias_dtype = bias.dtype if bias is not None else None
        ctx.save_for_backward(x, w, expert_idx, slot_idx, w32, picked)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        from .gemm import grouped_gemm_tn, tcgen05_supported

        x, w, expert_idx, slot_idx, w32, picked = ctx.saved_tensors
        E_local, rows, Kdim = x.shape
        N = w.shape[1]
        grad_out = grad_out.contiguous()
        valid = (slot_idx >= 0).to(torch.float32)
        grad_w = (picked.float() * grad_out.float().unsqueeze(1)).sum(-1) * valid
        gy = ctx.pctx.scatter(grad_out, expert_idx, slot_idx, (w32 * valid).contiguous(), E_local, ctx.C)      # [world, E_local, C, N]
        gy = gy.permute(1, 0, 2, 3).reshape(E_local, rows, N)
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = grouped_gemm_tn(gy, w.transpose(1, 2).contiguous()) if tcgen05_supported(gy, rows, Kdim, N) else torch.bmm(gy, w)
        if ctx.needs_input_grad[1]:
            if tcgen05_supported(gy, N, Kdim, rows):
                gw = grouped_gemm_tn(gy.transpose(1, 2).contiguous(), x.transpose(1, 2).contiguous())
            else:
                gw = torch.bmm(gy.transpose(1, 2), x)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = gy.float().sum(dim=1).to(ctx.bias_dtype)   # summed in fp32, returned in the bias's own dtype
        return gx, gw, gb, grad_w.to(ctx.wdtype), None, None, None, None


def linear_combine(x, w, bias, weights, expert_idx, slot_idx, pctx: "MoEPeerContext", capacity: int):
    """See :class:`_LinearCombine`."""
    return _LinearCombine.apply(x, w, bias, weights, expert_idx.contiguous(), slot_idx.contiguous(), pctx, capacity)


def get_context(group, world: int) -> Optional[MoEPeerContext]:
    """The MoE peer context of a torch process group (``None`` → use all_to_all_single)."""
    if os.environ.get("BAGUA_MOE_PEER", "1") != "1" or not dist.is_initialized():
        return None
    key = id(group) if group is not None else 0
    if key in _contexts:
        return _contexts[key]
    ctx = None
    try:
        from .. import communication as comm_mod

        torch_group = group if group is not None else dist.group.WORLD
        # a dedicated BaguaProcessGroup → dedicated signal pads: these kernels run on the compute stream and must not share
        # epochs with the bucket kernels on the comm stream
        ranks = sorted(dist.get_process_group_ranks(torch_group))
        pg = comm_mod.BaguaProcessGroup(ranks, None, f"moe{key}", torch_group)
        eng = pg.peer_engine()
        if eng is not None:
            ctx = MoEPeerContext(eng)
            ctx._pg = pg
    except Exception as e:  # noqa: BLE001
        logger.warning("bagua_b200: MoE peer dispatch/combine unavailable (%s); using all_to_all_single", e)
        ctx = None
    _contexts[key] = ctx
    return ctx
