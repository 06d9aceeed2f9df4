"""Fused optimizers on the sm_90a multi-tensor / flat kernels (csrc/multi_tensor.cu).

Reference: ``bagua/torch_api/contrib/fuse/optimizer.py`` fuses by *aliasing* contiguous tensors and then runs the stock
torch ``step()`` (several element-wise kernels, several passes over HBM).  Here a step over a bucket-flattened model is
ONE kernel launch that reads grad + state once and writes param/state (and the low-precision model copy, and the
zeroed gradient) once.  Layout trick kept from the reference: parameters are re-pointed into a flat arena — but the
arena mirrors the *gradient bucket layout* produced by ``with_bagua`` so the same flat index addresses grad, master
weight, momentum and model weight.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from ..core import dtype_code, native
from ..tensor import dense_strides

__all__ = ["FusedSGD", "FusedAdam", "FusedLAMB", "FusedLARS", "FusedLion", "flat_sgd_", "flat_adam_", "multi_tensor_plan"]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _kernels_apply(params) -> bool:
    """The sm_90a kernels handle CUDA tensors; everything else takes the plain torch update (also the hook the CPU tests use to
    drive the kernel call sites with a host double)."""
    return params[0].device.type == "cuda"


def flat_sgd_(param, grad, momentum_buf, *, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, first_step=False,
              grad_scale=1.0, zero_grad=False, model: Optional[torch.Tensor] = None):
    """One fused SGD step over flat CUDA tensors (param: fp32 master or model dtype; optional low-precision ``model`` copy)."""
    n = param.numel()
    assert grad.numel() == n and (momentum_buf is None or momentum_buf.numel() == n)
    native().flat_sgd(param.data_ptr(), dtype_code(param.dtype), grad.data_ptr(), dtype_code(grad.dtype),
                      momentum_buf.data_ptr() if momentum_buf is not None else 0, model.data_ptr() if model is not None else 0,
                      dtype_code(model.dtype) if model is not None else 0, n, float(lr), float(momentum), float(dampening), float(weight_decay),
                      bool(nesterov), bool(first_step), float(grad_scale), bool(zero_grad), _stream())


def flat_adam_(param, grad, exp_avg, exp_avg_sq, *, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, step=1, adamw=False, grad_scale=1.0,
               zero_grad=False, model: Optional[torch.Tensor] = None):
    """One fused Adam/AdamW step over flat CUDA tensors; moments are fp32."""
    n = param.numel()
    native().flat_adam(param.data_ptr(), dtype_code(param.dtype), grad.data_ptr(), dtype_code(grad.dtype), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                       model.data_ptr() if model is not None else 0, dtype_code(model.dtype) if model is not None else 0, n, float(lr),
                       float(betas[0]), float(betas[1]), float(eps), float(weight_decay), int(step), bool(adamw), float(grad_scale), bool(zero_grad),
                       _stream())


class _MultiPlan:
    """Device tables for the chunked multi-tensor kernels: pointer lists [n_lists][n_tensors], sizes, block map."""

    CHUNK = 65536

    def __init__(self, lists: List[List[torch.Tensor]]):
        self.n_tensors = len(lists[0])
        dev = lists[0][0].device
        self.keep = lists
        ptrs = [t.data_ptr() for lst in lists for t in lst]
        sizes = [t.numel() for t in lists[0]]
        b2t, b2c = [], []
        for i, n in enumerate(sizes):
            for c in range((n + self.CHUNK - 1) // self.CHUNK):
                b2t.append(i)
                b2c.append(c)
        self.n_blocks = len(b2t)
        self.ptrs = torch.tensor(ptrs, dtype=torch.int64, device=dev)
        self.sizes = torch.tensor(sizes, dtype=torch.int64, device=dev)
        self.b2t = torch.tensor(b2t, dtype=torch.int32, device=dev)
        self.b2c = torch.tensor(b2c, dtype=torch.int32, device=dev)
        self.signature = tuple(ptrs)

    def args(self):
        return (self.ptrs.data_ptr(), self.sizes.data_ptr(), self.b2t.data_ptr(), self.b2c.data_ptr(), self.n_tensors, self.n_blocks, self.CHUNK)


def multi_tensor_plan(lists: List[List[torch.Tensor]]) -> _MultiPlan:
    """Device pointer / size / block tables for the chunked multi-tensor kernels over ``lists`` (``[list][tensor]``, equal lengths)."""
    return _MultiPlan(lists)


def _launch_groups(params, state_key) -> List[tuple]:
    """Split ``params`` into multi-tensor launches: one per (dtype, ``state_key(p)``), in order of first appearance.  One launch
    applies one set of scalars (first step, bias correction) to all its tensors, so parameters whose optimizer state differs —
    one whose gradient was ``None`` at earlier steps — must not share it.  Returns ``[((dtype, ordinal), params)]``; the ordinal
    counts the launches of that dtype, so the pair stays the same from step to step and keys the plan cache."""
    groups: Dict[tuple, List[torch.nn.Parameter]] = {}
    for p in params:
        groups.setdefault((p.dtype, state_key(p)), []).append(p)
    out, seen = [], {}
    for (dt, _), ps in groups.items():
        seen[dt] = seen.get(dt, -1) + 1
        out.append(((dt, seen[dt]), ps))
    return out


def _cached_plan(cache: dict, key, lists: List[List[torch.Tensor]]) -> _MultiPlan:
    plan = cache.get(key)
    if plan is None or plan.signature != tuple(t.data_ptr() for lst in lists for t in lst):
        plan = cache[key] = _MultiPlan(lists)
    return plan


def _grad_in_layout(p: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """``p.grad`` in ``dtype`` and in ``p``'s memory layout: the multi-tensor kernels address parameter, gradient and state
    with one flat index over raw memory (a channels_last parameter may well receive a contiguous gradient)."""
    g = p.grad
    if g.dtype == dtype and g.stride() == p.stride():
        return g
    return torch.empty_like(p.data, dtype=dtype).copy_(g)


class _Segment:
    """A span of the gradient arena owned by one param group: grads, params and state share flat indices."""

    def __init__(self, params: List[torch.nn.Parameter], master_weights: bool):
        grads = [p.grad for p in params]
        es = grads[0].element_size()
        order = sorted(range(len(params)), key=lambda i: grads[i].data_ptr())
        self.params = [params[i] for i in order]
        grads = [grads[i] for i in order]
        start = grads[0].data_ptr()
        end = grads[-1].data_ptr() + grads[-1].numel() * es
        self.numel = (end - start) // es
        self.grad_ptr = start
        self.grad_dtype = grads[0].dtype
        dev = grads[0].device
        pdtype = self.params[0].dtype
        self.offsets = [(g.data_ptr() - start) // es for g in grads]
        # flat view over the gradient span (keeps the arena alive through the first grad's storage)
        self.grad_flat = torch.empty(0, dtype=self.grad_dtype, device=dev).set_(
            grads[0].untyped_storage(), grads[0].storage_offset(), (self.numel,)
        )
        assert self.grad_flat.data_ptr() == start
        self.param_flat = torch.zeros(self.numel, dtype=pdtype, device=dev)
        with torch.no_grad():
            for p, off in zip(self.params, self.offsets):
                dst = torch.as_strided(self.param_flat, p.shape, p.stride(), off)
                dst.copy_(p.data)
                p.data = dst
        self.master = None
        if master_weights and pdtype in (torch.float16, torch.bfloat16):
            self.master = self.param_flat.float()
        self.state: Dict[str, torch.Tensor] = {}
        self.steps = 0
        self.bound = False  # per-parameter optimizer state aliased to the flat buffers (see _FusedBase._bind_state)

    def state_flat(self, key: str) -> torch.Tensor:
        t = self.state.get(key)
        if t is None:
            t = torch.zeros(self.numel, dtype=torch.float32, device=self.param_flat.device)
            self.state[key] = t
        return t

    def valid(self) -> bool:
        p0, p1 = self.params[0], self.params[-1]
        if p0.grad is None or p1.grad is None:
            return False
        es = p0.grad.element_size()
        return (p0.grad.data_ptr() == self.grad_ptr + self.offsets[0] * es and p1.grad.data_ptr() == self.grad_ptr + self.offsets[-1] * es
                and p0.data_ptr() == self.param_flat.data_ptr() + self.offsets[0] * self.param_flat.element_size())

    def view_of(self, flat: torch.Tensor, idx: int) -> torch.Tensor:
        p, off = self.params[idx], self.offsets[idx]
        return torch.as_strided(flat, p.shape, p.stride(), off)


def _can_flatten(group_params: List[torch.nn.Parameter], all_params: List[torch.nn.Parameter]) -> bool:
    if not group_params:
        return False
    g0 = group_params[0].grad
    if g0 is None or not _kernels_apply([g0]):
        return False
    mine = set(id(p) for p in group_params)
    for p in group_params:
        if p.grad is None or p.grad.dtype != g0.dtype or p.dtype != group_params[0].dtype:
            return False
        # flat index i must address the same logical element in grad and param: identical dense layouts
        if p.grad.stride() != p.stride() or dense_strides(p) != p.stride():
            return False
        if p.grad.untyped_storage().data_ptr() != g0.untyped_storage().data_ptr():
            return False
        # parameters that are themselves communicated in place (weight-averaging algorithms) must not be re-pointed
        if hasattr(p, "_bagua_backend_tensor") and getattr(p, "_bagua_getter_closure", None) is None:
            return False
    # the flat kernels update (and clear) the whole span: every tensor of the buckets involved must belong to this group —
    # a second optimizer's parameters interleaved in the same buckets would have their gradients cleared under its feet
    seen_buckets = set()
    for p in group_params:
        b = getattr(p, "_bagua_bucket", None)
        if b is None or id(b) in seen_buckets:
            continue
        seen_buckets.add(id(b))
        for t in b.tensors:
            if id(t) not in mine and not getattr(t, "bagua_tensor_name", "").startswith("bagua_padding_tensor"):
                return False
    es = g0.element_size()
    lo = min(p.grad.data_ptr() for p in group_params)
    hi = max(p.grad.data_ptr() + p.grad.numel() * es for p in group_params)
    payload = sum(p.grad.numel() * es for p in group_params)
    if hi - lo > payload + 4096 * len(group_params) + (1 << 20):
        return False
    for q in all_params:
        if id(q) in mine or q.grad is None:
            continue
        a, b = q.grad.data_ptr(), q.grad.data_ptr() + q.grad.numel() * q.grad.element_size()
        if a < hi and b > lo:
            return False
    return True


class _FusedBase(torch.optim.Optimizer):
    """Shared machinery: lazily builds one flat segment per param group when the group's gradients live in one bucket
    arena, otherwise drives the chunked multi-tensor kernel over pointer tables."""

    def __init__(self, params, defaults, master_weights: bool, zero_grad_in_step: bool):
        super().__init__(params, defaults)
        self.master_weights = master_weights
        self.zero_grad_in_step = zero_grad_in_step
        self._segments: Dict[int, Optional[_Segment]] = {}
        self._multi: Dict[tuple, _MultiPlan] = {}
        self._grads_zeroed = False
        self.kernel_launches = 0

    def _all_params(self):
        return [p for g in self.param_groups for p in g["params"]]

    def _segment_for(self, gi: int, group) -> Optional[_Segment]:
        seg = self._segments.get(gi, False)
        if seg is not False and (seg is None or seg.valid()):
            return seg
        params = [p for p in group["params"] if p.requires_grad]
        seg = None
        if params and all(p.grad is not None for p in params) and _can_flatten(params, self._all_params()):
            seg = _Segment(params, self.master_weights)
        self._segments[gi] = seg
        return seg

    def zero_grad(self, set_to_none: bool = False):
        """Gradients stay allocated (they are views of the bucket arena); when the previous ``step`` already cleared them
        inside the kernel this is free."""
        if self._grads_zeroed:
            self._grads_zeroed = False
            return
        for gi, group in enumerate(self.param_groups):
            seg = self._segments.get(gi)
            if seg:
                seg.grad_flat.zero_()
            else:
                for p in group["params"]:
                    if p.grad is not None:
                        p.grad.detach_()
                        p.grad.zero_()

    def flat_segments(self) -> List[_Segment]:
        return [s for s in self._segments.values() if s]

    def _bind_state(self, seg: _Segment, key: str, flat: Optional[torch.Tensor] = None) -> bool:
        """``self.state[p][key]`` of every parameter of the segment becomes its view of the segment's flat buffer.  Values
        that are already there — a loaded checkpoint, the buffers of a segment that was rebuilt — are copied in first, so
        ``state_dict()`` / ``load_state_dict()`` round-trip through the flat kernels.  Returns whether anything was adopted."""
        flat = seg.state_flat(key) if flat is None else flat
        adopted = False
        for i, p in enumerate(seg.params):
            view = seg.view_of(flat, i)
            cur = self.state[p].get(key)
            if isinstance(cur, torch.Tensor) and cur.data_ptr() != view.data_ptr() and cur.shape == view.shape:
                view.copy_(cur)
                adopted = True
            self.state[p][key] = view
        return adopted

    def state_dict(self):
        for seg in self.flat_segments():
            step = self.state[seg.params[0]].get("step") if seg.params else None
            if step is not None:
                for p in seg.params[1:]:
                    self.state[p]["step"] = step
        return super().state_dict()

    def load_state_dict(self, state_dict):
        """torch casts loaded state to the parameter dtype; moments and master weights of low-precision parameters are fp32
        here, so tensors are re-read from ``state_dict`` unchanged, and the flat segments re-adopt them at the next step."""
        super().load_state_dict(state_dict)
        ids = [i for g in state_dict["param_groups"] for i in g["params"]]
        params = [p for g in self.param_groups for p in g["params"]]
        for pid, p in zip(ids, params):
            for k, v in state_dict["state"].get(pid, {}).items():
                if isinstance(v, torch.Tensor):
                    self.state[p][k] = v.detach().clone().to(device=p.device)
        for seg in self.flat_segments():
            seg.bound = False

    @torch.no_grad()
    def clip_grad_norm_(self, max_norm: float, norm_type: float = 2.0) -> torch.Tensor:
        """Global gradient-norm clipping without a per-tensor pass: for parameter groups on the flat path the norm is one
        reduction over the group's span of the bucket arena and the scaling one in-place multiply (the gaps of the span are
        alignment padding that holds zeros); other parameters go through the usual per-tensor path.  No host synchronisation;
        returns the total norm (a device tensor) like ``torch.nn.utils.clip_grad_norm_``.  Call it after the gradients are
        complete (after ``backward()`` of the last micro-batch) and before ``step()``."""
        flat_ids, norms, loose = set(), [], []
        for gi, group in enumerate(self.param_groups):
            seg = self._segment_for(gi, group)
            if seg is not None:
                norms.append(torch.linalg.vector_norm(seg.grad_flat, norm_type, dtype=torch.float32))
                flat_ids.update(id(p) for p in seg.params)
        for group in self.param_groups:
            loose += [p for p in group["params"] if p.grad is not None and id(p) not in flat_ids]
        norms += [torch.linalg.vector_norm(p.grad, norm_type, dtype=torch.float32) for p in loose]
        if not norms:
            return torch.zeros(())
        dev = norms[0].device
        total = torch.linalg.vector_norm(torch.stack([n.to(dev) for n in norms]), norm_type)
        coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
        for seg in self.flat_segments():
            seg.grad_flat.mul_(coef.to(seg.grad_flat.device, seg.grad_flat.dtype))
        for p in loose:
            p.grad.mul_(coef.to(p.grad.device, p.grad.dtype))
        return total

    @torch.no_grad()
    def refresh_master_weights(self):
        """Re-read the fp32 master copies from the (low-precision) parameters.  Needed after the weights were loaded or
        edited behind the optimizer's back: the next step writes ``master − lr·update`` over the parameters."""
        for seg in self.flat_segments():
            if seg.master is not None:
                seg.master.copy_(seg.param_flat.float())
        for p, st in self.state.items():
            if isinstance(st, dict) and "master" in st:
                st["master"].copy_(p.data)


class FusedSGD(_FusedBase):
    """SGD (momentum / nesterov / weight decay) with the update of a whole bucket-flattened model in one kernel.

    ``master_weights=True`` keeps fp32 master weights and momentum for bf16/fp16 models and writes the low-precision
    model copy in the same pass.  ``zero_grad_in_step=True`` clears gradients in the kernel (saves the memset pass)."""

    def __init__(self, params, lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, master_weights=True,
                 zero_grad_in_step=True, grad_scale=1.0):
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov)
        super().__init__(params, defaults, master_weights, zero_grad_in_step)
        self.grad_scale = grad_scale

    @torch.no_grad()
    def step(self, closure=None, only: Optional[set] = None):
        """``only``: restrict the update to these parameter ids (chunked multi-tensor kernels; used by the in-bucket optimizers
        for parameters that are not part of any bucket — MoE experts, ignored parameters)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        C = native()
        for gi, group in enumerate(self.param_groups):
            seg = self._segment_for(gi, group) if only is None else None
            lr, mom, damp, wd, nest = group["lr"], group["momentum"], group["dampening"], group["weight_decay"], group["nesterov"]
            if seg is not None:
                if not seg.bound or (mom != 0 and "momentum_buffer" not in seg.state):
                    if mom != 0 and self._bind_state(seg, "momentum_buffer"):
                        seg.steps = max(seg.steps, 1)  # adopted momentum: this is not a first step
                    if seg.master is not None:
                        self._bind_state(seg, "master", seg.master)
                    seg.bound = True
                first = seg.steps == 0
                mbuf = seg.state_flat("momentum_buffer") if mom != 0 else None
                if seg.master is not None:
                    flat_sgd_(seg.master, seg.grad_flat, mbuf, lr=lr, momentum=mom, dampening=damp, weight_decay=wd, nesterov=nest,
                              first_step=first, grad_scale=self.grad_scale, zero_grad=self.zero_grad_in_step, model=seg.param_flat)
                else:
                    flat_sgd_(seg.param_flat, seg.grad_flat, mbuf, lr=lr, momentum=mom, dampening=damp, weight_decay=wd, nesterov=nest,
                              first_step=first, grad_scale=self.grad_scale, zero_grad=self.zero_grad_in_step)
                seg.steps += 1
                self.kernel_launches += 1
                continue
            # multi-tensor path (per dtype)
            params = [p for p in group["params"] if p.grad is not None and (only is None or id(p) in only)]
            if not params:
                continue
            if not _kernels_apply(params):
                self._torch_step(params, group)
                continue
            for (dt, k), ps in _launch_groups(params, lambda p: mom != 0 and "momentum_buffer" in self.state[p]):
                # low-precision parameters keep fp32 master weights and fp32 momentum (mixed-precision kernel)
                mixed = self.master_weights and dt in (torch.float16, torch.bfloat16)
                first = mom != 0 and "momentum_buffer" not in self.state[ps[0]]
                for p in ps:
                    st = self.state[p]
                    if mixed and "master" not in st:
                        st["master"] = torch.empty_like(p.data, dtype=torch.float32).copy_(p.data)
                    if mom != 0:
                        sdt = torch.float32 if mixed else p.dtype
                        buf = st.get("momentum_buffer")
                        if buf is None:
                            st["momentum_buffer"] = torch.zeros_like(p.data, dtype=sdt)
                        elif buf.dtype != sdt or buf.stride() != p.stride():  # e.g. a checkpoint written with another precision
                            st["momentum_buffer"] = torch.empty_like(p.data, dtype=sdt).copy_(buf)
                lists = [[p.data for p in ps], [_grad_in_layout(p, dt) for p in ps]]
                if mixed:
                    lists.append([self.state[p]["master"] for p in ps])
                if mom != 0:
                    lists.append([self.state[p]["momentum_buffer"] for p in ps])
                plan = _cached_plan(self._multi, (gi, dt, k), lists)
                fn = C.multi_tensor_sgd_mp if mixed else C.multi_tensor_sgd
                fn(*plan.args(), dtype_code(dt), mom != 0, float(lr), float(mom), float(damp), float(wd), bool(nest), bool(first),
                   float(self.grad_scale), _stream())
                self.kernel_launches += 1
        if only is None:
            self._grads_zeroed = self.zero_grad_in_step and all(s is not None for s in self._segments.values()) and len(self._segments) == len(self.param_groups)
        return loss

    def _torch_step(self, params, group):
        for p in params:
            d = p.grad * self.grad_scale
            if group["weight_decay"] != 0:
                d = d.add(p.data, alpha=group["weight_decay"])
            if group["momentum"] != 0:
                buf = self.state[p].get("momentum_buffer")
                if buf is None:
                    buf = self.state[p]["momentum_buffer"] = d.clone()
                else:
                    buf.mul_(group["momentum"]).add_(d, alpha=1 - group["dampening"])
                d = d.add(buf, alpha=group["momentum"]) if group["nesterov"] else buf
            p.data.add_(d, alpha=-group["lr"])


class FusedAdam(_FusedBase):
    """Adam / AdamW in one kernel per flat segment (fp32 moments, optional fp32 master weights)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, adamw=False, master_weights=True,
                 zero_grad_in_step=True, grad_scale=1.0):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, adamw=adamw)
        super().__init__(params, defaults, master_weights, zero_grad_in_step)
        self.grad_scale = grad_scale

    @torch.no_grad()
    def step(self, closure=None, only: Optional[set] = None):
        """``only``: see :meth:`FusedSGD.step`."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        C = native()
        for gi, group in enumerate(self.param_groups):
            seg = self._segment_for(gi, group) if only is None else None
            lr, betas, eps, wd, adamw = group["lr"], group["betas"], group["eps"], group["weight_decay"], group["adamw"]
            if seg is not None:
                if not seg.bound:
                    adopted = self._bind_state(seg, "exp_avg")
                    self._bind_state(seg, "exp_avg_sq")
                    if seg.master is not None:
                        self._bind_state(seg, "master", seg.master)
                    if adopted:  # loaded checkpoint / rebuilt segment: continue its step count (bias correction)
                        seg.steps = max(seg.steps, int(self.state[seg.params[0]].get("step", 0)))
                    seg.bound = True
                seg.steps += 1
                m1, m2 = seg.state_flat("exp_avg"), seg.state_flat("exp_avg_sq")
                self.state[seg.params[0]]["step"] = seg.steps  # the other parameters get it in state_dict() (hot path: one write)
                target = seg.master if seg.master is not None else seg.param_flat
                flat_adam_(target, seg.grad_flat, m1, m2, lr=lr, betas=betas, eps=eps, weight_decay=wd, step=seg.steps, adamw=adamw,
                           grad_scale=self.grad_scale, zero_grad=self.zero_grad_in_step, model=seg.param_flat if seg.master is not None else None)
                self.kernel_launches += 1
                continue
            params = [p for p in group["params"] if p.grad is not None and (only is None or id(p) in only)]
            if not params:
                continue
            if not _kernels_apply(params):
                self._torch_step(params, group)
                continue
            for p in params:
                st = self.state[p]
                if "exp_avg" not in st:
                    # low-precision parameters keep fp32 moments and fp32 master weights (mixed-precision kernel)
                    mixed = self.master_weights and p.dtype in (torch.float16, torch.bfloat16)
                    sdt = torch.float32 if mixed else p.dtype
                    # preserve_format: state shares the parameter's memory order (the kernel walks raw memory)
                    st["exp_avg"] = torch.zeros_like(p.data, dtype=sdt)
                    st["exp_avg_sq"] = torch.zeros_like(p.data, dtype=sdt)
                    st["step"] = 0
                    if mixed:
                        st["master"] = torch.empty_like(p.data, dtype=torch.float32).copy_(p.data)
                st["step"] += 1
            for (dt, k), ps in _launch_groups(params, lambda p: int(self.state[p]["step"])):
                mixed = self.master_weights and dt in (torch.float16, torch.bfloat16)
                step = int(self.state[ps[0]]["step"])
                lists = [[p.data for p in ps], [_grad_in_layout(p, dt) for p in ps], [self.state[p]["exp_avg"] for p in ps],
                         [self.state[p]["exp_avg_sq"] for p in ps]]
                if mixed:
                    lists.append([self.state[p]["master"] for p in ps])
                plan = _cached_plan(self._multi, (gi, dt, k), lists)
                fn = C.multi_tensor_adam_mp if mixed else C.multi_tensor_adam
                fn(*plan.args(), dtype_code(dt), float(lr), float(betas[0]), float(betas[1]), float(eps), float(wd), int(step), bool(adamw),
                   float(self.grad_scale), _stream())
                self.kernel_launches += 1
        if only is None:
            self._grads_zeroed = self.zero_grad_in_step and all(s is not None for s in self._segments.values()) and len(self._segments) == len(self.param_groups)
        return loss

    def _torch_step(self, params, group):
        b1, b2 = group["betas"]
        for p in params:
            st = self.state[p]
            if "exp_avg" not in st:
                st["exp_avg"], st["exp_avg_sq"], st["step"] = torch.zeros_like(p.data), torch.zeros_like(p.data), 0
            st["step"] += 1
            g = p.grad * self.grad_scale
            if group["adamw"]:
                p.data.mul_(1 - group["lr"] * group["weight_decay"])
            elif group["weight_decay"] != 0:
                g = g.add(p.data, alpha=group["weight_decay"])
            st["exp_avg"].mul_(b1).add_(g, alpha=1 - b1)
            st["exp_avg_sq"].mul_(b2).addcmul_(g, g, value=1 - b2)
            bc1, bc2 = 1 - b1 ** st["step"], 1 - b2 ** st["step"]
            denom = (st["exp_avg_sq"].sqrt() / (bc2 ** 0.5)).add_(group["eps"])
            p.data.addcdiv_(st["exp_avg"], denom, value=-group["lr"] / bc1)


class FusedLAMB(_FusedBase):
    """LAMB with layer-wise trust ratios, two multi-tensor kernels per (dtype, step count) and step.

    The rule is LAMB (You et al., 2019, "Large Batch Optimization for Deep Learning") with the semantics of apex ``FusedLAMB``
    at its defaults (bias correction, gradient averaging, decoupled weight decay inside the update, no NVLAMB):

    ``m ← β1·m + (1−β1)·g``, ``v ← β2·v + (1−β2)·g²``, ``u = (m/bc1) / (sqrt(v)/sqrt(bc2) + eps) + wd·w``,
    ``w ← w − lr·r·u`` with the trust ratio ``r = ‖w‖/‖u‖`` over each whole parameter when ``wd ≠ 0`` and both norms are
    positive, else 1 — so a no-decay group (biases, LayerNorm) gets no layer adaptation.

    On CUDA every step is two multi-tensor kernels per (dtype, step count): the moments with per-block fp64 ``Σw²``/``Σu²``,
    then the per-parameter ratio (a fixed-order sum of the parameter's block partials, rounded to fp32 once) and the update.
    Moments are fp32; ``master_weights=True`` keeps fp32 master weights for bf16/fp16 parameters and writes the parameter
    rounded once. ``zero_grad_in_step=True`` clears the gradients in the first kernel. CPU tensors take a torch implementation
    of the same rule."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01, master_weights=True, zero_grad_in_step=True):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults, master_weights, zero_grad_in_step)
        self._sums: Dict[tuple, torch.Tensor] = {}

    @torch.no_grad()
    def step(self, closure=None, only: Optional[set] = None):
        """``only``: see :meth:`FusedSGD.step`."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        C = native()
        for gi, group in enumerate(self.param_groups):
            lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
            params = [p for p in group["params"] if p.grad is not None and (only is None or id(p) in only)]
            if not params:
                continue
            if not _kernels_apply(params):
                self._torch_step(params, group)
                continue
            for p in params:
                st = self.state[p]
                if "exp_avg" not in st:
                    # fp32 moments in the parameter's memory order (the kernels walk raw memory)
                    st["exp_avg"] = torch.zeros_like(p.data, dtype=torch.float32)
                    st["exp_avg_sq"] = torch.zeros_like(p.data, dtype=torch.float32)
                    st["step"] = 0
                    if self.master_weights and p.dtype in (torch.float16, torch.bfloat16):
                        st["master"] = torch.empty_like(p.data, dtype=torch.float32).copy_(p.data)
                st["step"] += 1
            for (dt, k), ps in _launch_groups(params, lambda p: int(self.state[p]["step"])):
                mixed = self.master_weights and dt in (torch.float16, torch.bfloat16)
                step = int(self.state[ps[0]]["step"])
                grads = [_grad_in_layout(p, dt) for p in ps]
                lists = [[p.data for p in ps], grads, [self.state[p]["exp_avg"] for p in ps], [self.state[p]["exp_avg_sq"] for p in ps]]
                if mixed:
                    lists.append([self.state[p]["master"] for p in ps])
                plan = _cached_plan(self._multi, (gi, dt, k), lists)
                sums = self._sums.get((gi, dt, k))
                if sums is None or sums.shape[0] < plan.n_blocks:
                    sums = self._sums[(gi, dt, k)] = torch.empty(max(plan.n_blocks, 1), 2, dtype=torch.float64, device=ps[0].device)
                hyper = (dtype_code(dt), mixed, float(lr), float(b1), float(b2), float(eps), float(wd), step)
                C.multi_tensor_lamb_stage1(*plan.args(), *hyper, 0, sums.data_ptr(), bool(self.zero_grad_in_step), _stream())
                C.multi_tensor_lamb_stage2(*plan.args(), *hyper, sums.data_ptr(), _stream())
                self.kernel_launches += 2
                if self.zero_grad_in_step:
                    for p, g in zip(ps, grads):
                        if g is not p.grad:   # the kernel cleared a converted copy
                            p.grad.zero_()
        if only is None:
            self._grads_zeroed = self.zero_grad_in_step
        return loss

    def _torch_step(self, params, group):
        """The same rule in torch fp32 (CPU tensors)."""
        b1, b2 = group["betas"]
        eps, wd, lr = group["eps"], group["weight_decay"], group["lr"]
        for p in params:
            st = self.state[p]
            if "exp_avg" not in st:
                st["exp_avg"] = torch.zeros_like(p.data, dtype=torch.float32)
                st["exp_avg_sq"] = torch.zeros_like(p.data, dtype=torch.float32)
                st["step"] = 0
            st["step"] += 1
            g = p.grad.float()
            m, v = st["exp_avg"], st["exp_avg_sq"]
            m.mul_(b1).add_(g, alpha=1 - b1)
            v.mul_(b2).addcmul_(g, g, value=1 - b2)
            bc1, bc2 = 1 - b1 ** st["step"], 1 - b2 ** st["step"]
            w = p.data.float()
            u = (m / bc1) / (v.sqrt() / bc2 ** 0.5 + eps) + wd * w
            r = 1.0
            if wd != 0:
                wn, un = float(w.double().norm()), float(u.double().norm())
                if wn > 0 and un > 0:
                    r = float(torch.tensor(wn / un, dtype=torch.float32))
            p.data.copy_(w - (lr * r) * u)


class FusedLARS(_FusedBase):
    """LARS with layer-wise trust ratios (You et al., 2017, "Large Batch Training of Convolutional Networks"; the MLPerf
    ResNet-50 form), two multi-tensor kernels per (dtype) group and step.

    ``trust = trust_coefficient·‖w‖ / (‖g‖ + wd·‖w‖)`` over each whole parameter when ``wd ≠ 0`` and both norms are positive
    (fp64 sums, one rounding to fp32), NaN when a sum is NaN, else 1 — so a ``weight_decay=0`` group (biases, BatchNorm) gets
    plain momentum SGD; then ``v ← μ·v + (lr·trust)·(g + wd·w)``, ``w ← w − v``. No epsilon, Nesterov or dampening.

    The momentum buffer holds the lr-scaled step, as in the MLPerf reference. ``torch.optim.SGD`` keeps the unscaled one
    (``v ← μ·v + d``, ``w ← w − lr·v``); the two agree at a constant ``lr`` and differ whenever ``lr`` changes between steps (a
    warm-up or decay schedule): here an ``lr`` change only affects the new part of the step, there it rescales the whole history.

    On CUDA every step is two multi-tensor kernels per dtype: per-block fp64 ``Σw²``/``Σg²``, then the per-parameter trust (a
    fixed-order sum of the parameter's block partials) with the momentum and the update. The momentum is fp32;
    ``master_weights=True`` keeps fp32 master weights for bf16/fp16 parameters and writes the parameter rounded once.
    ``zero_grad_in_step=True`` clears the gradients in the second kernel. CPU tensors take a torch implementation of the same
    rule."""

    def __init__(self, params, lr=1e-3, momentum=0.9, weight_decay=0.0, trust_coefficient=1e-3, master_weights=True, zero_grad_in_step=True):
        defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay, trust_coefficient=trust_coefficient)
        super().__init__(params, defaults, master_weights, zero_grad_in_step)
        self._sums: Dict[tuple, torch.Tensor] = {}

    @torch.no_grad()
    def step(self, closure=None, only: Optional[set] = None):
        """``only``: see :meth:`FusedSGD.step`."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        C = native()
        for gi, group in enumerate(self.param_groups):
            lr, mom, wd, eta = group["lr"], group["momentum"], group["weight_decay"], group["trust_coefficient"]
            params = [p for p in group["params"] if p.grad is not None and (only is None or id(p) in only)]
            if not params:
                continue
            if not _kernels_apply(params):
                self._torch_step(params, group)
                continue
            for p in params:
                st = self.state[p]
                buf = st.get("momentum_buffer")
                if buf is None:   # fp32 momentum in the parameter's memory order (the kernels walk raw memory)
                    st["momentum_buffer"] = torch.zeros_like(p.data, dtype=torch.float32)
                elif buf.dtype != torch.float32 or buf.stride() != p.stride():   # e.g. a checkpoint written with another layout
                    st["momentum_buffer"] = torch.empty_like(p.data, dtype=torch.float32).copy_(buf)
                if self.master_weights and p.dtype in (torch.float16, torch.bfloat16) and "master" not in st:
                    st["master"] = torch.empty_like(p.data, dtype=torch.float32).copy_(p.data)
            for (dt, k), ps in _launch_groups(params, lambda p: 0):
                mixed = self.master_weights and dt in (torch.float16, torch.bfloat16)
                grads = [_grad_in_layout(p, dt) for p in ps]
                lists = [[p.data for p in ps], grads, [self.state[p]["momentum_buffer"] for p in ps]]
                if mixed:
                    lists.append([self.state[p]["master"] for p in ps])
                plan = _cached_plan(self._multi, (gi, dt, k), lists)
                sums = self._sums.get((gi, dt, k))
                if sums is None or sums.shape[0] < plan.n_blocks:
                    sums = self._sums[(gi, dt, k)] = torch.empty(max(plan.n_blocks, 1), 2, dtype=torch.float64, device=ps[0].device)
                C.multi_tensor_lars_stage1(*plan.args(), dtype_code(dt), mixed, 0, sums.data_ptr(), _stream())
                C.multi_tensor_lars_stage2(*plan.args(), dtype_code(dt), mixed, float(lr), float(mom), float(wd), float(eta), 0, sums.data_ptr(),
                                           bool(self.zero_grad_in_step), _stream())
                self.kernel_launches += 2
                if self.zero_grad_in_step:
                    for p, g in zip(ps, grads):
                        if g is not p.grad:   # the kernel cleared a converted copy
                            p.grad.zero_()
        if only is None:
            self._grads_zeroed = self.zero_grad_in_step
        return loss

    def _torch_step(self, params, group):
        """The same rule in torch fp32 (CPU tensors)."""
        import math

        lr, mom, wd, eta = group["lr"], group["momentum"], group["weight_decay"], group["trust_coefficient"]
        for p in params:
            st = self.state[p]
            if "momentum_buffer" not in st:
                st["momentum_buffer"] = torch.zeros_like(p.data, dtype=torch.float32)
            g, w = p.grad.float(), p.data.float()
            W, G = float(w.double().square().sum()), float(g.double().square().sum())
            trust = 1.0
            if math.isnan(W) or math.isnan(G):
                trust = float("nan")
            elif wd != 0 and W > 0 and G > 0:
                trust = eta * math.sqrt(W) / (math.sqrt(G) + wd * math.sqrt(W))
            lt = float(torch.tensor(lr, dtype=torch.float32) * torch.tensor(trust, dtype=torch.float32))
            v = st["momentum_buffer"]
            v.mul_(mom).add_(g + wd * w, alpha=lt)
            p.data.copy_(w - v)


def _lion_constants(lr, betas, weight_decay):
    """Lion's fp32 constants ``(lr, b1, c1, b2, c2, d)`` as the kernels receive them: each worked out in double, rounded once."""
    b1, b2 = float(betas[0]), float(betas[1])
    vals = (float(lr), b1, 1.0 - b1, b2, 1.0 - b2, 1.0 - float(lr) * float(weight_decay))
    return tuple(torch.tensor(v, dtype=torch.float32) for v in vals)


def _lion_sign(u: torch.Tensor) -> torch.Tensor:
    """+1 / −1, +0 for ±0 and NaN for NaN (``torch.sign`` maps NaN to 0, which would make a NaN gradient a silent no-op)."""
    return torch.where(torch.isnan(u), u, torch.sign(u))


def lion_reference_step_(w: torch.Tensor, m: torch.Tensor, x: torch.Tensor, lr, betas, weight_decay, coef=None):
    """One Lion step in torch fp32, in place on ``w`` and ``m`` (fp32 tensors), ``x`` the gradient and ``coef`` (optional fp32 0-d
    tensor) its coefficient. Every product and sum is a separate fp32 op, so it reproduces the kernels bit for bit (see lion.cuh)."""
    lr32, b1, c1, b2, c2, d = (t.to(w.device) for t in _lion_constants(lr, betas, weight_decay))
    g = x.float() if coef is None else torch.mul(x.float(), coef.to(w.device, torch.float32))
    u = torch.add(torch.mul(b1, m), torch.mul(c1, g))
    w.copy_(torch.sub(torch.mul(w, d), torch.mul(lr32, _lion_sign(u))))
    m.copy_(torch.add(torch.mul(b2, m), torch.mul(c2, g)))


class FusedLion(_FusedBase):
    """Lion (Chen et al., 2023, "Symbolic Discovery of Optimization Algorithms", Algorithm 2), one multi-tensor kernel per dtype
    group and step, the gradient cleared in the same pass.

    ``u = β1·m + (1−β1)·g``, ``w ← w·(1 − lr·wd) − lr·sign(u)``, ``m ← β2·m + (1−β2)·g``: every element moves by exactly ±lr (0 where
    ``u`` is 0, NaN where it is NaN), after the decoupled weight decay. One fp32 moment per element (``exp_avg``), half of Adam's
    state. The constants are worked out in double and rounded to fp32 once, and every product and sum is rounded separately, so
    the CPU implementation (``_torch_step``, used for CPU tensors) gives the same bits as the kernel. ``master_weights=True`` keeps
    fp32 master weights for bf16/fp16 parameters and writes the parameter rounded once. Lion wants a smaller ``lr`` and a larger
    ``weight_decay`` than AdamW (the paper suggests 3–10× and 3–10×)."""

    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0.0, master_weights=True, zero_grad_in_step=True):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        for i, b in enumerate(betas):
            if not 0.0 <= b < 1.0:
                raise ValueError(f"Invalid beta parameter at index {i}: {b}")
        defaults = dict(lr=lr, betas=betas, weight_decay=weight_decay)
        super().__init__(params, defaults, master_weights, zero_grad_in_step)

    @torch.no_grad()
    def step(self, closure=None, only: Optional[set] = None):
        """``only``: see :meth:`FusedSGD.step`."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        C = native()
        for gi, group in enumerate(self.param_groups):
            lr, (b1, b2), wd = group["lr"], group["betas"], group["weight_decay"]
            params = [p for p in group["params"] if p.grad is not None and (only is None or id(p) in only)]
            if not params:
                continue
            if not _kernels_apply(params):
                self._torch_step(params, group)
                continue
            for p in params:
                st = self.state[p]
                m = st.get("exp_avg")
                if m is None:   # fp32 moment in the parameter's memory order (the kernel walks raw memory)
                    st["exp_avg"] = torch.zeros_like(p.data, dtype=torch.float32)
                elif m.dtype != torch.float32 or m.stride() != p.stride():   # e.g. a checkpoint written with another layout
                    st["exp_avg"] = torch.empty_like(p.data, dtype=torch.float32).copy_(m)
                if self.master_weights and p.dtype in (torch.float16, torch.bfloat16) and "master" not in st:
                    st["master"] = torch.empty_like(p.data, dtype=torch.float32).copy_(p.data)
            for (dt, k), ps in _launch_groups(params, lambda p: 0):
                mixed = self.master_weights and dt in (torch.float16, torch.bfloat16)
                grads = [_grad_in_layout(p, dt) for p in ps]
                lists = [[p.data for p in ps], grads]
                if mixed:
                    lists.append([self.state[p]["master"] for p in ps])
                lists.append([self.state[p]["exp_avg"] for p in ps])
                plan = _cached_plan(self._multi, (gi, dt, k), lists)
                C.multi_tensor_lion(*plan.args(), dtype_code(dt), mixed, float(lr), float(b1), float(b2), float(wd), bool(self.zero_grad_in_step),
                                    _stream())
                self.kernel_launches += 1
                if self.zero_grad_in_step:
                    for p, g in zip(ps, grads):
                        if g is not p.grad:   # the kernel cleared a converted copy
                            p.grad.zero_()
        if only is None:
            self._grads_zeroed = self.zero_grad_in_step
        return loss

    def _torch_step(self, params, group):
        """The same rule in torch fp32 (CPU tensors), bit for bit."""
        for p in params:
            st = self.state[p]
            if "exp_avg" not in st:
                st["exp_avg"] = torch.zeros_like(p.data, dtype=torch.float32)
            lowp = p.dtype != torch.float32
            if lowp and self.master_weights and "master" not in st:
                st["master"] = p.data.float()
            w = st["master"] if lowp and self.master_weights else p.data.float()
            lion_reference_step_(w, st["exp_avg"], p.grad, group["lr"], group["betas"], group["weight_decay"])
            p.data.copy_(w)
            if self.zero_grad_in_step:
                p.grad.zero_()
