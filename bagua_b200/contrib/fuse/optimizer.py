"""Generic fused optimizer (reference: bagua/torch_api/contrib/fuse/optimizer.py:1-574).

``fuse_optimizer(opt)`` returns an optimizer with ``fuse_step()``.  Two engines sit behind it:

* **kernel path** — for ``torch.optim.SGD / Adam / AdamW`` on CUDA the step of every parameter group is executed by the
  sm_90a multi-tensor / flat kernels (``bagua_b200.ops.optim``): one launch per group instead of one per op per tensor.
* **generic path** — for *any* other optimizer (and on CPU) the reference's idea is kept: tensors that are contiguous in
  memory simultaneously for weights, gradients and every state entry are viewed as ONE parameter, the optimizer's own
  ``step()`` runs on those few fused parameters, and the resulting state is sliced back (so it stays contiguous and fusable).
"""
from __future__ import annotations

import copy
import logging
from typing import Dict, List, Optional

import torch

from ...utils import check_contiguous

__all__ = ["fuse_optimizer", "is_fused_optimizer", "calculate_mutual_groups"]

logger = logging.getLogger(__name__)


def is_fused_optimizer(optimizer: torch.optim.Optimizer) -> bool:
    """``True`` for optimizers returned by :func:`fuse_optimizer`."""
    return hasattr(optimizer, "_bagua_fused_optimizer")


def _flatten_params_(params: List[torch.nn.Parameter], what: str):
    """Re-point the weights (``what='data'``) or gradients (``what='grad'``) of ``params`` into one fresh contiguous
    storage, in order, keeping each tensor's (dense) strides."""
    from ...tensor import dense_strides

    tensors = [p.data if what == "data" else p.grad for p in params]
    total = sum(t.numel() for t in tensors)
    flat = torch.zeros(total, dtype=tensors[0].dtype, device=tensors[0].device)
    off = 0
    with torch.no_grad():
        for p, t in zip(params, tensors):
            view = torch.as_strided(flat, t.shape, dense_strides(t), off)
            view.copy_(t)
            if what == "data":
                p.data = view
            else:
                p.grad = view
            off += t.numel()
    return flat


def flatten_params_and_grads_(optimizer: torch.optim.Optimizer):
    """Per (param group, dtype, device): make weights contiguous with each other and gradients contiguous with each other,
    in the same order (reference optimizer.py:39-81).  Parameters whose gradients are already bucket views (``with_bagua``)
    keep their gradient layout; only their weights are flattened to mirror it."""
    for group in optimizer.param_groups:
        by_key: Dict[tuple, List[torch.nn.Parameter]] = {}
        for p in group["params"]:
            if p.requires_grad:
                by_key.setdefault((p.dtype, p.device), []).append(p)
        for params in by_key.values():
            for p in params:
                if p.grad is None:
                    p.grad = torch.zeros_like(p.data)
            bucketed = all(getattr(p, "_bagua_bucket", None) is not None and getattr(p, "_bagua_getter_closure", None) is not None for p in params)
            if bucketed:
                params = sorted(params, key=lambda p: p.grad.data_ptr())
            weight_comm = any(getattr(p, "_bagua_bucket", None) is not None and getattr(p, "_bagua_getter_closure", None) is None for p in params)
            if not weight_comm and not check_contiguous([p.data for p in params]):
                _flatten_params_(params, "data")
            if not bucketed and not check_contiguous([p.grad for p in params]):
                _flatten_params_(params, "grad")


def calculate_mutual_groups(tensors_list: List[List[torch.Tensor]]) -> List[List[int]]:
    """Indices ``[[i0, i1, ...], ...]`` of maximal runs (length ≥ 2) such that for EVERY list in ``tensors_list`` the
    tensors at those indices are contiguous in memory in that order (reference optimizer.py:120-139)."""
    n = len(tensors_list[0])
    if n == 0:
        return []
    order = sorted(range(n), key=lambda i: tensors_list[0][i].data_ptr())
    groups: List[List[int]] = []
    cur = [order[0]]
    for a, b in zip(order, order[1:]):
        ok = True
        for tensors in tensors_list:
            ta, tb = tensors[a], tensors[b]
            if ta.dtype != tb.dtype or ta.device != tb.device or ta.data_ptr() + ta.numel() * ta.element_size() != tb.data_ptr() or ta.numel() == 0:
                ok = False
                break
        if ok:
            cur.append(b)
        else:
            if len(cur) > 1:
                groups.append(cur)
            cur = [b]
    if len(cur) > 1:
        groups.append(cur)
    return groups


def _view_over(tensors: List[torch.Tensor]) -> torch.Tensor:
    total = sum(t.numel() for t in tensors)
    first = tensors[0]
    return torch.empty(0, dtype=first.dtype, device=first.device).set_(first.untyped_storage(), first.storage_offset(), (total,))


def _kernel_kind(optimizer) -> Optional[str]:
    t = type(optimizer)
    if t is torch.optim.SGD:
        return "sgd"
    if t is torch.optim.AdamW:
        return "adamw"
    if t is torch.optim.Adam:
        return "adam"
    return None


def _kernel_step(opt, kind: str) -> bool:
    """Run one step of SGD/Adam/AdamW through the multi-tensor kernels; returns False if a group is not eligible."""
    from ...core import dtype_code, native
    from ...ops.optim import _cached_plan, _launch_groups

    C = native()
    plans = opt.__dict__.setdefault("_bagua_kernel_plans", {})
    launches = 0
    for gi, group in enumerate(opt.param_groups):
        if group.get("maximize") or group.get("amsgrad") or group.get("capturable") or group.get("differentiable"):
            return False
        params = [p for p in group["params"] if p.grad is not None]
        if not params:
            continue
        if any((not p.is_cuda) or p.grad.is_sparse or p.grad.dtype != p.dtype or not p.is_contiguous() or not p.grad.is_contiguous() for p in params):
            return False
        if any(p.dtype not in (torch.float32, torch.float16, torch.bfloat16) for p in params):
            return False
    stream = torch.cuda.current_stream().cuda_stream
    for gi, group in enumerate(opt.param_groups):
        params = [p for p in group["params"] if p.grad is not None]
        if kind == "sgd":
            mom = group["momentum"]
            groups = _launch_groups(params, lambda p: mom != 0 and opt.state[p].get("momentum_buffer") is not None)
        else:
            for p in params:
                st = opt.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0)
                    st["exp_avg"] = torch.zeros_like(p.data)
                    st["exp_avg_sq"] = torch.zeros_like(p.data)
                st["step"] = st["step"] + 1
            groups = _launch_groups(params, lambda p: int(opt.state[p]["step"]))
        for (dt, k), ps in groups:
            if kind == "sgd":
                first = mom != 0 and opt.state[ps[0]].get("momentum_buffer") is None
                lists = [[p.data for p in ps], [p.grad for p in ps]]
                if mom != 0:
                    for p in ps:
                        if opt.state[p].get("momentum_buffer") is None:
                            opt.state[p]["momentum_buffer"] = torch.zeros_like(p.data)
                    lists.append([opt.state[p]["momentum_buffer"] for p in ps])
            else:
                step = int(opt.state[ps[0]]["step"])
                lists = [[p.data for p in ps], [p.grad for p in ps], [opt.state[p]["exp_avg"] for p in ps], [opt.state[p]["exp_avg_sq"] for p in ps]]
            plan = _cached_plan(plans, (gi, dt, k), lists)
            if kind == "sgd":
                C.multi_tensor_sgd(*plan.args(), dtype_code(dt), mom != 0, float(group["lr"]), float(mom), float(group["dampening"]),
                                   float(group["weight_decay"]), bool(group["nesterov"]), bool(first), 1.0, stream)
            else:
                b1, b2 = group["betas"]
                C.multi_tensor_adam(*plan.args(), dtype_code(dt), float(group["lr"]), float(b1), float(b2), float(group["eps"]),
                                    float(group["weight_decay"]), step, kind == "adamw", 1.0, stream)
            launches += 1
    opt._bagua_fused_count = launches
    return True


def _generic_fuse_step(opt, closure=None):
    """Reference-style aliasing: run the optimizer's own step() on fused views."""
    shadow = opt._bagua_shadow
    fused_count = 0
    new_groups = []
    fused_records = []  # (fused_param, [member params])
    for group in opt.param_groups:
        params = [p for p in group["params"] if p.grad is not None]
        rest = [p for p in group["params"] if p.grad is None]
        state_keys = None
        for p in params:
            keys = tuple(sorted(k for k, v in opt.state.get(p, {}).items() if isinstance(v, torch.Tensor) and v.numel() == p.numel() and v.dim() > 0))
            state_keys = keys if state_keys is None else (state_keys if state_keys == keys else ())
        state_keys = state_keys or ()
        lists = [[p.data for p in params], [p.grad for p in params]] + [[opt.state[p][k] for p in params] for k in state_keys]
        uniform_scalars = True
        groups = calculate_mutual_groups(lists) if len(params) > 1 else []
        in_group = set(i for g in groups for i in g)
        g_params = []
        for g in groups:
            members = [params[i] for i in g]
            # scalar state (e.g. step) must agree inside a fused run
            scal = [{k: v for k, v in opt.state.get(p, {}).items() if k not in state_keys} for p in members]
            if any(str(s) != str(scal[0]) for s in scal[1:]):
                for i in g:
                    in_group.discard(i)
                continue
            fp = torch.nn.Parameter(_view_over([m.data for m in members]), requires_grad=True)
            fp.grad = _view_over([m.grad for m in members])
            st = {k: _view_over([opt.state[m][k] for m in members]) for k in state_keys}
            st.update(copy.copy(scal[0]))
            if st:
                shadow.state[fp] = st
            fused_records.append((fp, members))
            g_params.append(fp)
            fused_count += 1
        singles = [params[i] for i in range(len(params)) if i not in in_group]
        for p in singles:
            if p in opt.state:
                shadow.state[p] = opt.state[p]
        ng = {k: v for k, v in group.items() if k != "params"}
        ng["params"] = g_params + singles + rest
        new_groups.append(ng)
    shadow.param_groups = new_groups
    loss = shadow.step(closure) if closure is not None else shadow.step()
    # slice the (possibly newly created) fused state back to the members so it stays contiguous for the next step
    for fp, members in fused_records:
        st = shadow.state.pop(fp, {})
        off = 0
        for m in members:
            mst = opt.state[m]
            for k, v in st.items():
                if isinstance(v, torch.Tensor) and v.dim() > 0 and v.numel() == fp.numel():
                    mst[k] = v.view(-1)[off : off + m.numel()].view(m.shape)
                else:
                    mst[k] = copy.copy(v) if not isinstance(v, torch.Tensor) else v.clone()
            off += m.numel()
    for p in list(shadow.state.keys()):
        if p not in opt.state:
            opt.state[p] = shadow.state[p]
    shadow.state.clear()
    # hyper-parameters changed by the step (schedulers mutate opt.param_groups, not the shadow)
    opt._bagua_fused_count = fused_count
    return loss


def fuse_optimizer(optimizer: torch.optim.Optimizer, do_flatten: bool = True, check_flatten: bool = True) -> torch.optim.Optimizer:
    """Return ``optimizer`` extended with ``fuse_step(closure=None)`` (and ``step`` left untouched).

    Args:
        optimizer: any torch optimizer.
        do_flatten: flatten weights (and gradients, unless they already are bucket views) so that whole parameter groups
            fuse.  Do not combine a *fused* step with the plain ``step`` of the same optimizer after flattening.
        check_flatten: re-check contiguity at every ``fuse_step`` (cheap pointer comparison) instead of trusting the
            initial flattening.
    """
    if is_fused_optimizer(optimizer):
        raise RuntimeError("trying to fuse an optimizer twice!")
    optimizer._bagua_fused_optimizer = True
    optimizer._bagua_check_flatten = check_flatten
    optimizer._bagua_do_flatten = do_flatten
    optimizer._bagua_fused_count = 0
    shadow = copy.copy(optimizer)
    shadow.state = type(optimizer.state)() if not isinstance(optimizer.state, dict) else {}
    import collections

    shadow.state = collections.defaultdict(dict)
    shadow.param_groups = []
    # never run the algorithm hooks twice: the shadow executes the *original* step
    if hasattr(optimizer, "_bagua_original_step"):
        shadow.step = optimizer._bagua_original_step
    optimizer._bagua_shadow = shadow
    if do_flatten:
        flatten_params_and_grads_(optimizer)

    def fuse_step(self, closure=None):
        r"""Perform a single optimization step with fused kernels / fused parameters."""
        kind = _kernel_kind(self)
        done = False
        loss = None
        if kind is not None and closure is None:
            with torch.no_grad():
                done = _kernel_step(self, kind)
        if not done:
            loss = _generic_fuse_step(self, closure)
        post = getattr(self, "_bagua_post_step_hook", None)
        if post is not None:
            post(self)
        return loss

    from types import MethodType

    optimizer.fuse_step = MethodType(fuse_step, optimizer)
    return optimizer
