"""Centralized synchronous full-precision data parallelism (reference: bagua/torch_api/algorithms/gradient_allreduce.py:1-64).

On NVSwitch each bucket is reduced by ONE kernel (two-shot peer loads/stores or NVLS ``multimem``) that also applies
the 1/N average; ``fused_optimizer=True`` additionally folds the SGD update of the rank's 1/N shard and the all-gather
of the updated weights into that kernel (see ``FusedShardedSGD``)."""
from __future__ import annotations

from .base import Algorithm, AlgorithmImpl

__all__ = ["GradientAllReduceAlgorithm", "GradientAllReduceAlgorithmImpl"]


class GradientAllReduceAlgorithmImpl(AlgorithmImpl):
    def __init__(self, process_group, hierarchical: bool = False, average: bool = True, variant: str = "auto"):
        super().__init__(process_group)
        self.hierarchical = hierarchical
        self.average = average
        self.variant = variant

    def init_operations(self, bagua_ddp, bucket):
        bucket.clear_ops()
        hp = getattr(bagua_ddp, "_bagua_hyperparameters", None)
        variant = self.variant
        if variant == "auto" and hp is not None and getattr(hp, "allreduce_variant", "auto") != "auto":
            variant = hp.allreduce_variant
        if variant == "auto" and hp is not None and getattr(hp, "bucket_variants", None):
            # autotune service: variant per bucket, looked up by message size in the bus-bandwidth table measured at start-up
            try:
                i = [b.name for b in bagua_ddp.bagua_buckets].index(bucket.name)
                if i < len(hp.bucket_variants):
                    variant = hp.bucket_variants[i]
            except ValueError:
                pass
        bucket.append_centralized_synchronous_op(hierarchical=self.hierarchical, average=self.average, group=self.process_group, variant=variant)


class GradientAllReduceAlgorithm(Algorithm):
    def __init__(self, hierarchical: bool = False, average: bool = True, variant: str = "auto"):
        """
        Args:
            hierarchical: intra-node reduce → inter-node allreduce → intra-node broadcast when the job spans nodes.
            average: average (``True``) or sum gradients.
            variant: ``auto`` | ``one_shot`` | ``two_shot`` | ``multimem`` kernel choice (``auto`` = by size / autotune).
        """
        self.hierarchical = hierarchical
        self.average = average
        self.variant = variant

    def reify(self, process_group) -> GradientAllReduceAlgorithmImpl:
        return GradientAllReduceAlgorithmImpl(process_group, hierarchical=self.hierarchical, average=self.average, variant=self.variant)


# ---------------------------------------------------------------------------------------------------------------
# Checkpointable state of the in-bucket optimizers
# ---------------------------------------------------------------------------------------------------------------
_STATE_KEYS = {"sgd": ("master", "momentum_buffer"), "adam": ("master", "exp_avg", "exp_avg_sq")}


def consolidate_shards(shards, numel: int, layout):
    """``shards``: the per-rank fp32 state vectors of one bucket in rank order (each ``ceil(vecs/N)·16/elem`` long, the last ones
    padded); ``layout``: ``[(name, offset, numel, shape, strides)]`` of the bucket's tensors (offsets in elements of the flat
    bucket, strides = the parameter's dense memory layout, e.g. channels_last).  Returns ``{name: contiguous tensor(shape)}`` —
    the state as an unsharded optimizer would hold it, independent of world size, bucketing and memory format."""
    import torch

    full = torch.cat([s.reshape(-1) for s in shards])[:numel]
    return {name: torch.as_strided(full, shape, strides, off).contiguous().clone() for name, off, n, shape, strides in layout}


def shard_of(per_name, layout, numel: int, lo: int, hi: int, length: int, device=None):
    """Inverse of :func:`consolidate_shards` for one rank: the ``[lo, hi)`` slice of the bucket-flat vector assembled from the
    per-parameter tensors, zero-padded to the shard ``length``.  Parameters missing from ``per_name`` contribute zeros."""
    import torch

    out = torch.zeros(length, dtype=torch.float32, device=device)
    for name, off, n, shape, strides in layout:
        a, b = max(off, lo), min(off + n, hi)
        if a < b and name in per_name:
            mem = torch.empty_strided(shape, strides, dtype=torch.float32)       # the parameter's memory order
            mem.copy_(per_name[name].to(torch.float32).reshape(shape))
            flat = torch.as_strided(mem, (n,), (1,))
            out[a - lo: b - lo].copy_(flat[a - off: b - off])
    return out


class _ShardedStateMixin:
    """``state_dict()`` / ``load_state_dict()`` of the optimizers whose state lives in 1/N shards next to the buckets.

    The saved form is *consolidated*: per parameter name, full-shape fp32 ``master`` weights and moments (all-gathered from the
    shards — a collective, every rank must call ``state_dict()``; ``collective_state_dict`` tells the checkpoint module), so
    a checkpoint does not depend on the world size or on the bucket boundaries (autotune may move them)."""

    _kind = "sgd"

    @property
    def collective_state_dict(self) -> bool:
        return bool(getattr(self, "_shards", None))

    def _gather(self, t, group):
        import torch
        import torch.distributed as dist

        out = [torch.empty_like(t) for _ in range(group.size())]
        dist.all_gather(out, t.contiguous(), group=group.torch_group)
        return out

    def state_dict(self):
        if not getattr(self, "_shards", None):
            return super().state_dict()
        state = {}
        steps = 0
        for rec in self._shards:
            for key, t in zip(_STATE_KEYS[self._kind], rec["state"]):
                for name, full in consolidate_shards(self._gather(t, rec["group"]), rec["numel"], rec["layout"]).items():
                    state.setdefault(name, {})[key] = full.cpu()
            steps = max(steps, int(rec["op"].steps()))
        groups = [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]
        # parameters outside the buckets (MoE experts, ignored ones) are stepped by the base class: their state in torch's format
        return {"sharded_fused": self._kind, "steps": steps, "state": state, "param_groups": groups, "uncovered": super().state_dict()}

    def load_state_dict(self, sd):
        if not isinstance(sd, dict) or "sharded_fused" not in sd:
            return super().load_state_dict(sd)
        if sd["sharded_fused"] != self._kind:
            raise ValueError(f"checkpoint holds {sd['sharded_fused']} state, this optimizer is {self._kind}")
        if sd.get("uncovered") is not None:
            super().load_state_dict(sd["uncovered"])
        for g, saved in zip(self.param_groups, sd["param_groups"]):
            g.update(saved)
        if not getattr(self, "_shards", None):
            self._pending_state = sd          # applied bucket by bucket when the algorithm builds the ops (with_bagua)
            return
        for rec in self._shards:
            self._apply_to_shard(rec, sd)
        self._sync_hyper()

    def _apply_to_shard(self, rec, sd):
        for key, t in zip(_STATE_KEYS[self._kind], rec["state"]):
            per_name = {name: st[key] for name, st in sd["state"].items() if key in st}
            t.copy_(shard_of(per_name, rec["layout"], rec["numel"], rec["lo"], rec["hi"], t.numel(), device=t.device))
        rec["op"].set_steps(int(sd.get("steps", 0)))

    def refresh_master_weights(self):
        """Re-read the fp32 master shards from the model weights (call after loading or editing weights without optimizer
        state: the next bucket kernel writes ``master − lr·update`` over the parameters)."""
        if not getattr(self, "_shards", None):
            return super().refresh_master_weights() if hasattr(super(), "refresh_master_weights") else None
        for rec in self._shards:
            lo, hi = rec["lo"], min(rec["hi"], rec["numel"])
            if hi > lo:
                rec["state"][0][: hi - lo].copy_(rec["weights"][lo:hi].float())

    def _step_uncovered(self):
        """Parameters that no bucket kernel updates — MoE experts (excluded from data parallelism), ignored parameters —
        get the ordinary fused update here; their gradients are cleared like the bucketed ones."""
        candidates = getattr(self, "_uncovered_cache", None)
        if candidates is None:  # the parameter list is static between (re-)initialisations: looked up once, usually empty
            covered = getattr(self, "_covered", set())
            candidates = self._uncovered_cache = [p for g in self.param_groups for p in g["params"] if id(p) not in covered]
        left = [p for p in candidates if p.grad is not None]
        if left:
            super().step(only={id(p) for p in left})
            import torch

            torch._foreach_zero_([p.grad for p in left])

    def _register_shard(self, rec):
        if not hasattr(self, "_shards"):
            self._shards = []
        if not hasattr(self, "_covered"):
            self._covered = set()
        self._covered.update(rec.get("param_ids", ()))
        self._uncovered_cache = None
        self._shards.append(rec)
        pending = getattr(self, "_pending_state", None)
        if pending is not None:
            self._apply_to_shard(rec, pending)



# ---------------------------------------------------------------------------------------------------------------
# Gradient allreduce with the optimizer folded into the communication kernel
# ---------------------------------------------------------------------------------------------------------------
class ShardedFusedSGD(object):
    """Marker mix-in: see :func:`make_sharded_fused_sgd`."""


def make_sharded_fused_sgd(params, lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False):
    """SGD whose update runs *inside* each bucket's NVSwitch kernel (``allreduce_sgd_kernel``): reduce-scatter of the
    gradients → SGD(momentum) on this rank's 1/N shard with fp32 master weights → all-gather of the updated weights, one
    launch per bucket, overlapped with the rest of backward.  Optimizer state is sharded N ways (ZeRO-1-like) and the
    gradient bucket is cleared on the way out.  Use together with ``FusedGradientAllReduceAlgorithm``; with one process (or
    without a peer engine) it behaves like :class:`bagua_b200.ops.optim.FusedSGD`."""
    from ...ops.optim import FusedSGD

    class _ShardedFusedSGD(_ShardedStateMixin, FusedSGD, ShardedFusedSGD):
        _kind = "sgd"

        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self._comm_ops = []   # AllReduceSgdOp per bucket once the algorithm has taken over
            self._shards = []

        def _sync_hyper(self):
            groups = getattr(self, "_comm_groups", ())
            for i, op in enumerate(self._comm_ops):
                g = self.param_groups[groups[i] if i < len(groups) else 0]   # every bucket op serves one parameter group
                op.set_hyper(float(g["lr"]), float(g["momentum"]), float(g["dampening"]), float(g["weight_decay"]), bool(g["nesterov"]))

        def step(self, closure=None):
            if not self._comm_ops:
                return super().step(closure)
            # the update already happened in the bucket kernels of this iteration; publish hyper-parameters for the next
            self._sync_hyper()
            self._step_uncovered()
            self._grads_zeroed = True
            self.kernel_launches += len(self._comm_ops)
            return None

    return _ShardedFusedSGD(params, lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov,
                            master_weights=True, zero_grad_in_step=True)


class ShardedFusedAdam(object):
    """Marker mix-in: see :func:`make_sharded_fused_adam`."""


def make_sharded_fused_adam(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, adamw=False):
    """Adam / AdamW counterpart of :func:`make_sharded_fused_sgd`: the update of this rank's 1/N shard (fp32 master weights
    and both moments) runs inside each bucket's reduce-scatter → all-gather kernel (``allreduce_adam_kernel``).  With one
    process (or without a peer engine) it behaves like :class:`bagua_b200.ops.optim.FusedAdam`."""
    from ...ops.optim import FusedAdam

    class _ShardedFusedAdam(_ShardedStateMixin, FusedAdam, ShardedFusedAdam):
        _kind = "adam"

        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self._comm_ops = []
            self._shards = []

        def _sync_hyper(self):
            groups = getattr(self, "_comm_groups", ())
            for i, op in enumerate(self._comm_ops):
                g = self.param_groups[groups[i] if i < len(groups) else 0]
                op.set_hyper(float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"]), bool(g["adamw"]))

        def step(self, closure=None):
            if not self._comm_ops:
                return super().step(closure)
            self._sync_hyper()
            self._step_uncovered()
            self._grads_zeroed = True
            self.kernel_launches += len(self._comm_ops)
            return None

    return _ShardedFusedAdam(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, adamw=adamw, master_weights=True,
                             zero_grad_in_step=True)


class FusedGradientAllReduceAlgorithmImpl(GradientAllReduceAlgorithmImpl):
    def __init__(self, process_group, optimizer, average: bool = True):
        super().__init__(process_group, hierarchical=False, average=average)
        self.optimizer = optimizer
        self._weight_slices = []

    @property
    def bucket_pieces(self) -> int:
        return max(1, len(self.optimizer.param_groups))

    def init_forward_pre_hook(self, bagua_ddp):
        """The update of iteration *i* runs inside the bucket kernels of *i*'s backward pass, before ``optimizer.step()`` is
        called — so the hyper-parameters are published at the start of every iteration (after any ``lr_scheduler.step()`` of
        the previous one), not only from ``step()``."""
        opt = self.optimizer

        def hook(input):
            if getattr(opt, "_comm_ops", None):
                opt._sync_hyper()

        # _reset_buckets builds this hook after the last init_operations: every new shard has consumed the carried-over state
        # (checkpoint loaded before with_bagua, or the snapshot taken in tensors_to_buckets) — it must not be applied again
        opt._pending_state = None
        return hook

    def _carry_state_over(self):
        """Called at the start of every (re-)bucketing — with_bagua, the autotune service moving bucket boundaries every 100 steps,
        the find_unused_parameters rebuild: snapshot the sharded master weights / moments / step count in their consolidated
        (world-size and bucketing independent) form and forget the old shards; ``init_operations`` re-shards from the snapshot.
        Collective (an all-gather per state tensor), like re-bucketing itself."""
        opt = self.optimizer
        if getattr(opt, "_shards", None):
            opt._pending_state = opt.state_dict()
        opt._comm_ops = []
        opt._comm_groups = []
        opt._shards = []
        opt._covered = set()
        opt._uncovered_cache = None

    def tensors_to_buckets(self, tensors, do_flatten):
        from ...bucket import BaguaBucket

        assert do_flatten, "the fused optimizer needs flattened buckets"
        self._carry_state_over()
        es = tensors[0][0].bagua_getter_closure().element_size()
        # One bucket kernel applies ONE set of hyper-parameters: with several parameter groups (weight decay / no weight decay)
        # every suggested bucket is split so that each piece holds tensors of a single group. The pieces keep their place in
        # the bucket order, so they become ready at about the same point of the backward pass as the original bucket.
        group_of = {id(p): gi for gi, g in enumerate(self.optimizer.param_groups) for p in g["params"]}
        multi = len(self.optimizer.param_groups) > 1
        buckets = []
        for i, b in enumerate(tensors):
            if not multi:
                buckets.append(BaguaBucket(b, flatten=True, name=str(i), alignment=max(1, 16 // es), group=self.process_group))
                continue
            pieces = {}
            for t in b:
                pieces.setdefault(group_of.get(id(t), 0), []).append(t)
            for gi in sorted(pieces):
                bk = BaguaBucket(pieces[gi], flatten=True, name=f"{i}.g{gi}", alignment=max(1, 16 // es), group=self.process_group)
                bk._fused_group = gi
                buckets.append(bk)
        return buckets

    def init_operations(self, bagua_ddp, bucket):
        import os

        import torch

        from ...core import dtype_code, native
        from ...tensor import dense_strides

        bucket.clear_ops()
        eng = bucket._engine(self.process_group)
        opt = self.optimizer
        is_adam = isinstance(opt, ShardedFusedAdam)
        if eng is None or bucket._slice is None or not (isinstance(opt, ShardedFusedSGD) or is_adam):
            return super().init_operations(bagua_ddp, bucket)
        group_index = getattr(bucket, "_fused_group", 0)
        C = native()
        flat = bucket.backend_tensor
        n, rank = self.process_group.size(), self.process_group.rank()
        nbytes = flat.numel() * flat.element_size()
        assert nbytes % 16 == 0
        # weights mirror the gradient bucket layout inside their own symmetric slice (peers write them in the kernel)
        wslice = eng.alloc(nbytes)
        bucket._companion_slices.append(wslice)
        wflat = wslice.view(flat.dtype, flat.numel())
        wflat.zero_()
        base = flat.data_ptr()
        with torch.no_grad():
            for t in bucket.tensors:
                g = t.bagua_getter_closure()
                assert t.dtype == flat.dtype, "weights and gradients must share a dtype for the fused kernel"
                off = (g.data_ptr() - base) // flat.element_size()
                # as_strided's offset is ABSOLUTE in the storage (the symmetric slab), not relative to wflat: without the slice's own
                # offset the parameter would alias whatever sits at the start of the slab — the gradient arena the kernel zeroes
                view = torch.as_strided(wflat, t.shape, dense_strides(t), wflat.storage_offset() + off)
                assert view.data_ptr() == wflat.data_ptr() + off * flat.element_size()
                view.copy_(t.data)
                t.data = view
        vecs = nbytes // 16
        vpr = (vecs + n - 1) // n
        per = 16 // flat.element_size()
        lo, hi = rank * vpr * per, min((rank + 1) * vpr * per, flat.numel())
        master = torch.zeros(vpr * per, dtype=torch.float32, device=flat.device)
        if hi > lo:
            master[: hi - lo].copy_(wflat[lo:hi].float())
        momentum = torch.zeros(vpr * per, dtype=torch.float32, device=flat.device)
        # NVLS whenever the fabric offers it (the variant validated on 2 and 8 GPUs); peer ld/st two-shot otherwise
        use_mc = bool(wslice.has_multicast and bucket._slice.has_multicast and eng.has_multicast)
        # with 2 ranks the in-switch reduction buys nothing (each GPU pulls half the bucket either way), so the peer ld/st
        # kernel is used: same policy as PeerEngine.choose_variant. BAGUA_FUSED_MULTIMEM=0/1 forces either flavour.
        force = os.environ.get("BAGUA_FUSED_MULTIMEM", "auto")
        if force == "0" or (force != "1" and n <= 2):
            use_mc = False
        # multimem flavour: 16 CTAs (measured on 8 GPUs, round 1); the peer ld/st flavour (1-2 ranks) also streams a large optimizer
        # shard per rank and wants 64 (VGG16 N=1 self-peer: 8 CTAs 5.43 ms/step, 32: 4.34, 64: 4.23 = the flat-optimizer path)
        cfg = eng.launch_cfg("multimem" if use_mc else "two_shot", nbytes, blocks=int(os.environ.get("BAGUA_FUSED_BLOCKS", "0")) or (16 if use_mc else 64))
        scale = (1.0 / n) if self.average else 1.0
        if is_adam:
            second = torch.zeros(vpr * per, dtype=torch.float32, device=flat.device)
            bucket._fused_state = (master, momentum, second)
            op = C.AllReduceAdamOp(eng.comm, bucket._slice.buf, wslice.buf, bucket._slice.offset, wslice.offset, nbytes, dtype_code(flat.dtype),
                                   master.data_ptr(), momentum.data_ptr(), second.data_ptr(), scale, True, use_mc, cfg)
        else:
            bucket._fused_state = (master, momentum)
            op = C.AllReduceSgdOp(eng.comm, bucket._slice.buf, wslice.buf, bucket._slice.offset, wslice.offset, nbytes, dtype_code(flat.dtype),
                                  master.data_ptr(), momentum.data_ptr(), scale, True, use_mc, cfg)
        bucket.backend_bucket.append_op(op)
        bucket._ops_keepalive.append(op)
        bucket.allreduce_variant = ("fused_adam_" if is_adam else "fused_sgd_") + ("multimem" if use_mc else "two_shot")
        opt._comm_ops.append(op)
        if not hasattr(opt, "_comm_groups"):
            opt._comm_groups = []
        opt._comm_groups.append(group_index)
        layout = [(t.bagua_tensor_name, (t.bagua_getter_closure().data_ptr() - base) // flat.element_size(), t.bagua_getter_closure().numel(),
                   tuple(t.shape), tuple(dense_strides(t))) for t in bucket.tensors if not t.bagua_tensor_name.startswith("bagua_padding_tensor")]
        opt._register_shard({"bucket": bucket.name, "group": self.process_group, "numel": flat.numel(), "lo": lo, "hi": hi, "layout": layout,
                             "state": bucket._fused_state, "op": op, "weights": wflat, "param_ids": [id(t) for t in bucket.tensors]})
        opt._sync_hyper()


class FusedGradientAllReduceAlgorithm(Algorithm):
    """Gradient allreduce whose buckets also apply the optimizer update (see :func:`make_sharded_fused_sgd` /
    :func:`make_sharded_fused_adam`)."""

    def __init__(self, optimizer, average: bool = True):
        self.optimizer = optimizer
        self.average = average

    def reify(self, process_group):
        # optimizer state is carried across (re-)bucketing by the impl (tensors_to_buckets → _carry_state_over)
        return FusedGradientAllReduceAlgorithmImpl(process_group, self.optimizer, average=self.average)
