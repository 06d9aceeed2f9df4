"""GShard-style top-1 / top-2 gated mixture of experts with expert parallelism
(reference: bagua/torch_api/model_parallel/moe/sharded_moe.py:1-375).

Semantics kept: fp32 gate, capacity = ceil(tokens/experts·factor) (≥ ``min_capacity`` for top-1), random token selection
under overflow for top-1, Gumbel-max second expert for top-2, the auxiliary load-balancing loss, ``exp_counts`` (kept on the device unless ``BAGUA_MOE_EXP_COUNTS_ON_CPU=1``).

H100-first formulation: gating produces *indices* — for every token and choice k: expert id, slot in that expert's
capacity buffer (or dropped) and combine weight — instead of the reference's dense one-hot ``[S, E, C]`` tensors, whose
``einsum("sec,sm->ecm")`` dispatch costs S·E·C·M MACs (sharded_moe.py:352-354).  Dispatch is then a row scatter and combine
a weighted row gather; on NVSwitch both are kernels that store/load token rows directly in the destination expert's
symmetric buffer on the peer GPU (``bagua_b200/ops/moe.py``), which *is* the all-to-all.  Elsewhere the rows go through
``torch.distributed.all_to_all_single``."""
from __future__ import annotations

import math
import os
from typing import Any, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import Tensor

from ...ops import moe as moe_ops

__all__ = ["TopKGate", "MOELayer", "top1gating", "top2gating", "top1gating_indices", "top2gating_indices", "GateOutput"]

_uniform_cache = {}
_gumbel_cache = {}


def _uniform(shape, device, low=0.0, high=1.0) -> Tensor:
    return torch.empty(shape, device=device, dtype=torch.float32).uniform_(low, high)


def multiplicative_jitter(x: Tensor, device: torch.device, epsilon: float = 1e-2) -> Tensor:
    """Multiply by U(1-ε, 1+ε) noise (makes the gate robust to bf16 rounding)."""
    if epsilon == 0:
        return x
    return x * _uniform(x.shape, device, 1.0 - epsilon, 1.0 + epsilon)


def gumbel_rsample(shape, device: torch.device) -> Tensor:
    u = _uniform(shape, device).clamp_(1e-20, 1.0)
    return -torch.log(-torch.log(u))


class GateOutput:
    """Index form of a gating decision for ``S`` tokens and ``K`` choices per token."""

    def __init__(self, l_aux, expert_idx, slot_idx, weights, capacity, num_experts, exp_counts):
        self.l_aux = l_aux                # scalar tensor
        self.expert_idx = expert_idx      # int64 [S, K]
        self.slot_idx = slot_idx          # int64 [S, K]; -1 = dropped
        self.weights = weights            # float32 [S, K] (0 for dropped); differentiable w.r.t. the gate
        self.capacity = capacity
        self.num_experts = num_experts
        self.exp_counts = exp_counts      # int tensor [E] (device of the logits; CPU on request)

    def dense(self) -> Tuple[Tensor, Tensor]:
        """(combine_weights[S,E,C], dispatch_mask[S,E,C]) exactly as the reference returns them."""
        S, K = self.expert_idx.shape
        cw = torch.zeros(S, self.num_experts, self.capacity, dtype=self.weights.dtype, device=self.weights.device)
        for k in range(K):
            valid = self.slot_idx[:, k] >= 0
            s = torch.nonzero(valid, as_tuple=True)[0]
            cw = cw.index_put((s, self.expert_idx[s, k], self.slot_idx[s, k]), self.weights[s, k], accumulate=True)
        return cw, cw.bool()


def _exp_counts(mask1: Tensor) -> Tensor:
    """Tokens routed to each expert (first choice).  The reference copies this to the CPU in every forward
    (sharded_moe.py:126,202) — one host synchronisation per MoE layer that drains the launch queue; here it stays where it was
    computed and is only a CPU tensor on request (``BAGUA_MOE_EXP_COUNTS_ON_CPU=1``, or ``.cpu()`` by whoever logs it)."""
    counts = torch.sum(mask1, dim=0).detach()
    return counts.to("cpu") if os.environ.get("BAGUA_MOE_EXP_COUNTS_ON_CPU", "0") == "1" else counts


def top1gating_indices(logits: Tensor, capacity_factor: float, min_capacity: int, used_token: Optional[Tensor] = None,
                       noisy_gate_policy: Optional[str] = None) -> GateOutput:
    if noisy_gate_policy == "RSample":
        logits_w_noise = logits + gumbel_rsample(logits.shape, device=logits.device)
    gates = F.softmax(logits, dim=1)  # everything is fp32 here
    S, E = gates.shape
    capacity = max(math.ceil((S / E) * capacity_factor), min_capacity)
    indices1_s = torch.argmax(logits_w_noise if noisy_gate_policy == "RSample" else gates, dim=1)
    mask1 = F.one_hot(indices1_s, num_classes=E)
    if used_token is not None:
        mask1 = mask1 * used_token.to(mask1.dtype).unsqueeze(1)
    exp_counts = _exp_counts(mask1)
    me = torch.mean(gates, dim=0)
    ce = torch.mean(mask1.float(), dim=0)
    l_aux = torch.sum(me * ce) * E
    assert S >= min_capacity, "No. of tokens (batch-size) should be greater than min_capacity. Either set min_capacity to 0 or inrease your batch size."
    # under overflow keep a uniformly random subset of `capacity` tokens per expert (reference :133-149)
    mask1_rand = mask1 * _uniform(mask1.shape, logits.device)
    _, top_idx = torch.topk(mask1_rand, k=min(capacity, S), dim=0)
    new_mask1 = mask1 * torch.zeros_like(mask1).scatter_(0, top_idx, 1)
    locations1 = torch.cumsum(new_mask1, dim=0) - 1
    kept = new_mask1.gather(1, indices1_s.unsqueeze(1)).squeeze(1) > 0
    slot = torch.where(kept, locations1.gather(1, indices1_s.unsqueeze(1)).squeeze(1), torch.full_like(indices1_s, -1))
    w = gates.gather(1, indices1_s.unsqueeze(1)).squeeze(1) * kept.to(gates.dtype)
    return GateOutput(l_aux, indices1_s.unsqueeze(1), slot.unsqueeze(1), w.unsqueeze(1), capacity, E, exp_counts)


def top2gating_indices(logits: Tensor, capacity_factor: float) -> GateOutput:
    gates = F.softmax(logits, dim=1)
    S, E = gates.shape
    capacity = math.ceil((2 * S / E) * capacity_factor)
    indices1_s = torch.argmax(gates, dim=1)
    mask1 = F.one_hot(indices1_s, num_classes=E)
    # second expert by the Gumbel-max trick, first one masked out
    logits_w_noise = logits + gumbel_rsample(logits.shape, device=logits.device)
    logits_except1 = logits_w_noise.masked_fill(mask1.bool(), float("-inf"))
    indices2_s = torch.argmax(logits_except1, dim=1)
    mask2 = F.one_hot(indices2_s, num_classes=E)
    locations1 = torch.cumsum(mask1, dim=0) - 1
    locations2 = torch.cumsum(mask2, dim=0) - 1 + torch.sum(mask1, dim=0, keepdim=True)
    exp_counts = _exp_counts(mask1)
    me = torch.mean(gates, dim=0)
    ce = torch.mean(mask1.float(), dim=0)
    l_aux = torch.mean(me * ce) * E * E
    loc1 = locations1.gather(1, indices1_s.unsqueeze(1)).squeeze(1)
    loc2 = locations2.gather(1, indices2_s.unsqueeze(1)).squeeze(1)
    keep1, keep2 = loc1 < capacity, loc2 < capacity
    g1 = gates.gather(1, indices1_s.unsqueeze(1)).squeeze(1) * keep1.to(gates.dtype)
    g2 = gates.gather(1, indices2_s.unsqueeze(1)).squeeze(1) * keep2.to(gates.dtype)
    denom = torch.clamp(g1 + g2, min=torch.finfo(gates.dtype).eps)
    w = torch.stack([g1 / denom, g2 / denom], dim=1)
    slot = torch.stack([torch.where(keep1, loc1, torch.full_like(loc1, -1)), torch.where(keep2, loc2, torch.full_like(loc2, -1))], dim=1)
    return GateOutput(l_aux, torch.stack([indices1_s, indices2_s], dim=1), slot, w, capacity, E, exp_counts)


def top1gating(logits, capacity_factor, min_capacity, used_token=None, noisy_gate_policy=None):
    """Reference-shaped result: ``(l_aux, combine_weights[S,E,C], dispatch_mask[S,E,C], exp_counts)``."""
    g = top1gating_indices(logits, capacity_factor, min_capacity, used_token, noisy_gate_policy)
    cw, mask = g.dense()
    return g.l_aux, cw, mask, g.exp_counts


def top2gating(logits, capacity_factor):
    g = top2gating_indices(logits, capacity_factor)
    cw, mask = g.dense()
    return g.l_aux, cw, mask, g.exp_counts


class TopKGate(torch.nn.Module):
    """Gate network (always fp32).  ``forward`` returns the reference's dense tuple; ``route`` the index form."""

    wg: torch.nn.Linear

    def __init__(self, model_dim: int, num_experts: int, k: int = 1, capacity_factor: float = 1.0, eval_capacity_factor: float = 1.0,
                 min_capacity: int = 4, noisy_gate_policy: Optional[str] = None) -> None:
        super().__init__()
        if k != 1 and k != 2:
            raise ValueError("Only top-1 and top-2 gatings are supported.")
        self.wg = torch.nn.Linear(model_dim, num_experts, bias=False).float()
        self.k = k
        self.capacity_factor = capacity_factor
        self.eval_capacity_factor = eval_capacity_factor
        self.min_capacity = min_capacity
        self.noisy_gate_policy = noisy_gate_policy

    def _apply(self, fn, *args, **kwargs):
        # The gate is always fp32 (reference sharded_moe.py:271-273 re-casts it inside forward). Doing it here instead keeps
        # ``model.to(torch.bfloat16)`` from ever producing a bf16 gate, so the parameter (and its bucketed gradient) is never
        # re-created after ``with_bagua`` has registered it.
        super()._apply(fn, *args, **kwargs)
        if self.wg.weight.is_floating_point() and self.wg.weight.dtype != torch.float32:
            self.wg.weight.data = self.wg.weight.data.float()
            if self.wg.weight.grad is not None:
                self.wg.weight.grad = self.wg.weight.grad.float()
        return self

    def route(self, input: Tensor, used_token: Optional[Tensor] = None) -> GateOutput:
        if self.wg.weight.dtype != torch.float32:
            raise RuntimeError("the MoE gate must stay fp32; do not cast `gate.wg` after wrapping the model with with_bagua")
        x = input.float()
        if self.noisy_gate_policy == "Jitter" and self.training:
            x = multiplicative_jitter(x, device=input.device)
        logits = self.wg(x)
        cf = self.capacity_factor if self.training else self.eval_capacity_factor
        if self.k == 1:
            return top1gating_indices(logits, cf, self.min_capacity, used_token, self.noisy_gate_policy if self.training else None)
        return top2gating_indices(logits, cf)

    def forward(self, input: Tensor, used_token: Optional[Tensor] = None):
        g = self.route(input, used_token)
        cw, mask = g.dense()
        return g.l_aux, cw, mask, g.exp_counts


class MOELayer(torch.nn.Module):
    """gate → dispatch (all-to-all) → local experts → combine (all-to-all)."""

    def __init__(self, gate: torch.nn.Module, experts: torch.nn.Module, num_local_experts: int, group: Optional[Any] = None) -> None:
        super().__init__()
        self.gate = gate
        self.experts = experts
        self.group = group
        self.world_size = dist.get_world_size(group) if dist.is_initialized() else 1
        self.num_local_experts = num_local_experts
        self.l_aux = None
        self.exp_counts = None

    def _recv_key(self):
        """Identity of this layer's private receive buffers (NVSwitch path): the dispatched rows are used in place, so ONE forward of
        this layer may be outstanding per backward — true of ordinary training loops, activation recomputation and gradient
        accumulation.  ``BAGUA_MOE_INPLACE_RECV=0`` restores the shared buffer + copy for exotic schedules (two forwards, then
        two backwards)."""
        import os

        return id(self) if os.environ.get("BAGUA_MOE_INPLACE_RECV", "1") == "1" else None

    def forward(self, *input: Tensor, **kwargs: Any) -> Tensor:
        x = input[0]
        used_token = input[1] if len(input) > 1 else None
        d_model = x.shape[-1]
        tokens = x.reshape(-1, d_model)
        g = self.gate.route(tokens, used_token)
        self.l_aux, self.exp_counts = g.l_aux, g.exp_counts
        # [E_total, C, M] rows land on the rank owning the expert: [world(src), E_local, C, M]
        dispatched = moe_ops.dispatch(tokens, g.expert_idx, g.slot_idx, g.num_experts, g.capacity, self.group, self.world_size,
                                      self.num_local_experts, key=self._recv_key())
        fused = self.experts.fused_combine_context(dispatched, self.group, self.world_size) if hasattr(self.experts, "fused_combine_context") else None
        if fused is not None:
            combined = self.experts.forward_combine(dispatched, g.weights.to(x.dtype), g.expert_idx, g.slot_idx, fused)
            return combined.reshape(x.shape)
        expert_out = self.experts(dispatched)
        combined = moe_ops.combine(expert_out, g.expert_idx, g.slot_idx, g.weights.to(x.dtype), g.num_experts, g.capacity, self.group,
                                   self.world_size, self.num_local_experts, key=self._recv_key())
        return combined.reshape(x.shape)
