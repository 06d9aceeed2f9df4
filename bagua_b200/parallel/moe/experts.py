"""Container of a rank's local experts (reference: bagua/torch_api/model_parallel/moe/experts.py:1-41)."""
from __future__ import annotations

import copy
import os

import torch


class Experts(torch.nn.Module):
    def __init__(self, expert: torch.nn.Module, num_local_experts: int = 1):
        super().__init__()
        self.bagua_experts = torch.nn.ModuleList([copy.deepcopy(expert) for _ in range(num_local_experts)])
        self.num_local_experts = num_local_experts
        for e in self.bagua_experts:
            for _, p in e.named_parameters():
                p.expert = True  # skipped by the data-parallel engine (bagua_build_params)

    def _grouped_mlp(self):
        """(fc1, fc2, activation) lists when every local expert is a 2-layer MLP ``fc2(act(fc1(x)))`` — the shape the
        wgmma grouped GEMM accelerates; ``None`` otherwise."""
        cached = getattr(self, "_grouped_cache", None)
        if cached is not None:
            return cached or None
        ok = True
        for e in self.bagua_experts:
            fc1, fc2 = getattr(e, "fc1", None), getattr(e, "fc2", None)
            if not (isinstance(fc1, torch.nn.Linear) and isinstance(fc2, torch.nn.Linear) and getattr(e, "grouped_gemm_compatible", False)):
                ok = False
        self._grouped_cache = ok
        return ok or None

    def _forward_grouped(self, inputs: torch.Tensor) -> torch.Tensor:
        from ...ops.gemm import grouped_linear

        W, E, C, M = inputs.shape
        x = inputs.permute(1, 0, 2, 3).reshape(E, W * C, M)  # tokens of every source rank, per local expert
        w1, b1, w2, b2 = self._stacked()
        h = torch.nn.functional.gelu(grouped_linear(x, w1, b1), approximate="tanh")
        y = grouped_linear(h, w2, b2)
        return y.reshape(E, W, C, -1).permute(1, 0, 2, 3)

    def _stacked(self):
        w1 = torch.stack([e.fc1.weight for e in self.bagua_experts])
        b1 = torch.stack([e.fc1.bias for e in self.bagua_experts]) if self.bagua_experts[0].fc1.bias is not None else None
        w2 = torch.stack([e.fc2.weight for e in self.bagua_experts])
        b2 = torch.stack([e.fc2.bias for e in self.bagua_experts]) if self.bagua_experts[0].fc2.bias is not None else None
        return w1, b1, w2, b2

    def fused_combine_context(self, inputs: torch.Tensor, group, world: int):
        """The NVSwitch MoE context when the second expert GEMM can push its output tiles straight to the token owners
        (opt-in: ``BAGUA_MOE_FUSED_COMBINE=1``; grouped 2-layer MLP experts, bf16, capacity a multiple of 128)."""
        if os.environ.get("BAGUA_MOE_FUSED_COMBINE", "0") != "1":
            return None
        if not (inputs.is_cuda and inputs.dtype == torch.bfloat16 and world >= 1 and self._grouped_mlp()):
            return None
        from ...ops import moe as moe_ops

        pctx = moe_ops._peer_ctx(inputs, group, world)
        if pctx is None:
            return None
        C = inputs.shape[2]
        fc2 = self.bagua_experts[0].fc2
        hidden = torch.empty(0, fc2.in_features, dtype=inputs.dtype, device=inputs.device)
        return pctx if pctx.fused_combine_supported(hidden, fc2.out_features, C) else None

    def forward_combine(self, inputs: torch.Tensor, weights: torch.Tensor, expert_idx: torch.Tensor, slot_idx: torch.Tensor, pctx) -> torch.Tensor:
        """``combine(experts(inputs))`` → ``[S, model]``: fc1 + GELU as usual, then ONE kernel for fc2 and the combine all-to-all
        (the GEMM epilogue stores each output tile into the symmetric buffer of the rank that owns those tokens)."""
        from ...ops.gemm import grouped_linear
        from ...ops.moe_peer import linear_combine

        W, E, C, M = inputs.shape
        x = inputs.permute(1, 0, 2, 3).reshape(E, W * C, M)
        w1, b1, w2, b2 = self._stacked()
        h = torch.nn.functional.gelu(grouped_linear(x, w1, b1), approximate="tanh")
        return linear_combine(h, w2, b2, weights, expert_idx, slot_idx, pctx, C)

    def forward(self, inputs: torch.Tensor) -> torch.Tensor:
        """``inputs``: ``[world, num_local_experts, capacity, model]``; expert ``i`` processes ``inputs[:, i]``."""
        if inputs.is_cuda and inputs.dtype == torch.bfloat16 and self._grouped_mlp() and os.environ.get("BAGUA_DISABLE_GROUPED_GEMM") != "1":
            return self._forward_grouped(inputs)
        outs = []
        for chunk, expert in zip(inputs.chunk(self.num_local_experts, dim=1), self.bagua_experts):
            out = expert(chunk)
            if isinstance(out, tuple):
                out = out[0]
            outs.append(out)
        return torch.cat(outs, dim=1)
