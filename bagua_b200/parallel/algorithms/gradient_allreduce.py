"""Centralized synchronous full-precision data parallelism (reference: bagua/torch_api/algorithms/gradient_allreduce.py:1-64).

On NVSwitch each bucket is reduced by ONE kernel (two-shot peer loads/stores or NVLS ``multimem``) that also applies
the 1/N average; ``fused_optimizer=True`` additionally folds the SGD update of the rank's 1/N shard and the all-gather
of the updated weights into that kernel (see ``FusedShardedSGD``)."""
from __future__ import annotations

import contextlib

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
_STATE_KEYS = {"sgd": ("master", "momentum_buffer"), "adam": ("master", "exp_avg", "exp_avg_sq"), "lamb": ("master", "exp_avg", "exp_avg_sq"),
               "lars": ("master", "momentum_buffer"), "lion": ("master", "exp_avg")}
# what set_hyper of a rule's bucket ops takes, from a parameter group (a LAMB or LARS bucket's two ops take the same)
_HYPER = {"sgd": lambda g: (float(g["lr"]), float(g["momentum"]), float(g["dampening"]), float(g["weight_decay"]), bool(g["nesterov"])),
          "adam": lambda g: (float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"]), bool(g["adamw"])),
          "lamb": lambda g: (float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"])),
          "lars": lambda g: (float(g["lr"]), float(g["momentum"]), float(g["weight_decay"]), float(g["trust_coefficient"])),
          "lion": lambda g: (float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["weight_decay"]))}
# the rules whose trust ratio is a norm over a whole parameter: phase A in the bucket program, then per-bucket norms, one
# per-parameter exchange and the per-bucket update in step()
_PER_PARAMETER = ("lamb", "lars")
# the native ops of a rule: the fused bucket op (update inside backward; none for the per-parameter rules) and the phase-B op step() runs.
# Both constructors take the rule's fp32 state in _STATE_KEYS order; the per-parameter rules' phase-B op is built by _per_param_ops.
_OPS = {"sgd": ("AllReduceSgdOp", "ShardSgdOp"), "adam": ("AllReduceAdamOp", "ShardAdamOp"), "lion": ("AllReduceLionOp", "ShardLionOp"),
        "lamb": (None, "ShardLambOp"), "lars": (None, "ShardLarsOp")}


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


class _Bucketing:
    """What an in-bucket optimizer holds for one bucketing of the model. ``FusedGradientAllReduceAlgorithm`` replaces it as a whole
    whenever the buckets are (re-)built; with no peer engine it stays empty and the optimizer takes the flat path."""

    def __init__(self):
        self.shards = []       # one record per bucket, see FusedGradientAllReduceAlgorithmImpl.init_operations
        self.hyper_ops = []    # (op, parameter-group index) of every op that takes hyper-parameters
        self.covered = set()   # ids of the bucketed parameters
        self.uncovered = None  # the parameters outside the buckets, looked up once
        self.clip = None       # the norm exchange shared by all buckets (max_grad_norm and / or loss_scaling), see _clip_state
        self.lamb = None       # the per-parameter exchange shared by all buckets (LAMB and LARS), see _per_param_state
        self.unit = None       # fp32 1.0 on the device: the coefficient of an accumulated update without a norm exchange
        # the program step() runs after the norm exchange, on the current stream of `device`: every bucket's pre-update op (LAMB
        # moments, LARS norms), the per-parameter exchange, every bucket's update op; empty when the updates run in the bucket kernels
        self.pre_ops = []
        self.update_ops = []
        self.device = None
        self.launches = 0      # optimizer-update kernels per step, in the bucket programs or in step()
        self.ema = None        # ema_decay: the EmaOp over every bucket's [master, EMA] shard pair and its table, built with the last bucket


class _ShardedStateMixin:
    """``state_dict()`` / ``load_state_dict()`` of the optimizers whose state lives in 1/N shards next to the buckets.

    The saved form is *consolidated*: per parameter name, full-shape fp32 ``master`` weights and moments (all-gathered from the
    shards — a collective, every rank must call ``state_dict()``; ``collective_state_dict`` tells the checkpoint module), so
    a checkpoint does not depend on the world size or on the bucket boundaries (autotune may move them)."""

    _kind = "sgd"
    max_grad_norm = None
    loss_scaling = False
    accumulate_grads = False
    ema_decay = None
    ema_every = 1
    _ema = False                     # built with ema_decay: an fp32 EMA next to every master

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._bucketing = _Bucketing()
        self._pending_state = None   # a checkpoint loaded while no shard exists, applied bucket by bucket by _register_shard
        self._norm_pending = False   # clip_grad_norm_ has computed this step's norm
        self._last_norm = None
        self._loss_scale = None      # the device tensor the norm exchange reads the loss scale from (None: a constant 1)
        self._ema_calls = 0          # step() calls so far: the EMA updates on every ema_every-th
        self._ema_swapped = False    # inside ema_weights()
        self._ema_plans = {}         # tables (and EmaOps) of the local EMA launches, by role
        self._param_names = {}       # id(parameter) → its name in the model, for ema_state_dict()

    def _state_keys(self):
        return _STATE_KEYS[self._kind] + (("ema",) if self._ema else ())

    @property
    def collective_state_dict(self) -> bool:
        return bool(self._bucketing.shards)

    @property
    def native_ops_in_step(self) -> bool:
        """Whether ``step()`` runs native kernels once the bucket kernels are live: the norm exchange and the clipped update with
        ``max_grad_norm`` or ``loss_scaling``, LAMB's and LARS's per-bucket norms, per-parameter exchange and update always. They carry
        per-call host state (box parity, step count), so such a step cannot be captured in a CUDA graph. With ``accumulate_grads``
        the update always runs in ``step()``, which also restarts the accumulated sum; with ``ema_decay`` ``step()`` runs the EMA
        update on every ``ema_every``-th call."""
        return self.max_grad_norm is not None or self.loss_scaling or self._kind in _PER_PARAMETER or self.accumulate_grads or self._ema

    def _gather(self, t, group):
        import torch
        import torch.distributed as dist

        out = [torch.empty_like(t) for _ in range(group.size())]
        dist.all_gather(out, t.contiguous(), group=group.torch_group)
        return out

    def state_dict(self):
        if not self._bucketing.shards:
            sd = super().state_dict()
            if self._ema:
                sd["ema_calls"] = self._ema_calls
            return sd
        state = {}
        steps = 0
        for rec in self._bucketing.shards:
            for key, t in zip(self._state_keys(), rec["state"]):
                for name, full in consolidate_shards(self._gather(t, rec["group"]), rec["numel"], rec["layout"]).items():
                    state.setdefault(name, {})[key] = full.cpu()
            steps = max(steps, int(rec["step_ops"][0].steps()))
        if self.loss_scaling:   # launches include skipped steps: the count that the kernels use is the device's
            steps = int(self._bucketing.clip["t"].item())
        groups = [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]
        # parameters outside the buckets (MoE experts, ignored ones) are stepped by the base class: their state in torch's format
        out = {"sharded_fused": self._kind, "steps": steps, "state": state, "param_groups": groups, "uncovered": super().state_dict()}
        if self._ema:
            out["ema_calls"] = self._ema_calls
        return out

    def _load_local_ema(self, sd):
        """The local EMAs (fallback path, parameters outside the buckets) travel as ``state[p]["ema"]`` in torch's format: dropped
        when this optimizer keeps none; when the checkpoint has none they start from the loaded master at their next use."""
        if not self._ema:
            for st in self.state.values():
                if isinstance(st, dict):
                    st.pop("ema", None)
        elif isinstance(sd, dict):
            self._ema_calls = int(sd.get("ema_calls", 0))

    def load_state_dict(self, sd):
        if not isinstance(sd, dict) or "sharded_fused" not in sd:
            out = super().load_state_dict(sd)
            self._load_local_ema(sd)
            return out
        if sd["sharded_fused"] != self._kind:
            raise ValueError(f"checkpoint holds {sd['sharded_fused']} state, this optimizer is {self._kind}")
        if sd.get("uncovered") is not None:
            super().load_state_dict(sd["uncovered"])
        self._load_local_ema(sd)
        for g, saved in zip(self.param_groups, sd["param_groups"]):
            g.update(saved)
        if not self._bucketing.shards:
            self._pending_state = sd          # applied bucket by bucket when the algorithm builds the ops (with_bagua)
            return
        for rec in self._bucketing.shards:
            self._apply_to_shard(rec, sd)
        self._sync_hyper()

    def _apply_to_shard(self, rec, sd):
        for key, t in zip(self._state_keys(), rec["state"]):
            if key == "ema":   # a checkpoint written without an EMA starts it from the loaded master
                per_name = {name: st["ema"] if "ema" in st else st["master"] for name, st in sd["state"].items() if "ema" in st or "master" in st}
            else:
                per_name = {name: st[key] for name, st in sd["state"].items() if key in st}
            t.copy_(shard_of(per_name, rec["layout"], rec["numel"], rec["lo"], rec["hi"], t.numel(), device=t.device))
        for op in rec["step_ops"]:
            op.set_steps(int(sd.get("steps", 0)))
        if self.loss_scaling:
            self._bucketing.clip["t"].fill_(int(sd.get("steps", 0)))
        if sd.get("grad_sum") is not None and rec.get("grad_op") is not None:   # a re-bucketing mid-accumulation: continue the sum
            rec["shard"].copy_(shard_of(sd["grad_sum"], rec["layout"], rec["numel"], rec["lo"], rec["hi"], rec["shard"].numel(), device=rec["shard"].device))
            rec["grad_op"].resume()

    # ---- gradient accumulation (``accumulate_grads``) ----------------------------------------------------------------------
    def _grad_sum(self):
        """The pending accumulated gradient in consolidated form (``{name: fp32 tensor}``, like a state tensor), or ``None`` when no
        micro-batch has been reduced since the last ``step()`` / ``zero_grad()``. Collective when a sum is pending; phase A is a
        collective too, so every rank agrees on that."""
        recs = [rec for rec in self._bucketing.shards if rec.get("grad_op") is not None]
        if not any(rec["grad_op"].pending() for rec in recs):
            return None
        out = {}
        for rec in recs:   # a bucket whose phase A has not run since the restart holds the last step's shard: it contributes zeros
            t = rec["shard"] if rec["grad_op"].pending() else rec["shard"].new_zeros(rec["shard"].shape)
            out.update(consolidate_shards(self._gather(t, rec["group"]), rec["numel"], rec["layout"]))
        return out

    def _restart_grad_sums(self):
        """The next phase A of every bucket overwrites its shard: the accumulated gradient is consumed or discarded."""
        for rec in self._bucketing.shards:
            if rec.get("grad_op") is not None:
                rec["grad_op"].restart()

    def zero_grad(self, set_to_none: bool = False):
        """Also discards the gradient accumulated in the shards (``accumulate_grads``), except right after ``step()``, which has
        started a new sum already."""
        if self.accumulate_grads and not self._grads_zeroed:
            self._restart_grad_sums()
        return super().zero_grad(set_to_none)

    def refresh_master_weights(self):
        """Re-read the fp32 master shards from the model weights (call after loading or editing weights without optimizer
        state: the next bucket kernel writes ``master − lr·update`` over the parameters). With ``ema_decay`` the EMA restarts from the
        refreshed master: the old average belongs to other weights."""
        if not self._bucketing.shards:
            out = super().refresh_master_weights() if hasattr(super(), "refresh_master_weights") else None
            self._restart_local_ema(self._all_params())
            return out
        for rec in self._bucketing.shards:
            lo, hi = rec["lo"], min(rec["hi"], rec["numel"])
            if hi > lo:
                rec["state"][0][: hi - lo].copy_(rec["weights"][lo:hi].float())
            if self._ema:
                rec["state"][-1].copy_(rec["state"][0])
        self._restart_local_ema(self._local_ema_params())

    def _sync_hyper(self):
        hyper = _HYPER[self._kind]
        for op, group_index in self._bucketing.hyper_ops:
            op.set_hyper(*hyper(self.param_groups[group_index]))

    def _uncovered(self):
        b = self._bucketing
        if b.uncovered is None:  # the parameter list is static between (re-)initialisations: looked up once, usually empty
            b.uncovered = [p for g in self.param_groups for p in g["params"] if id(p) not in b.covered]
        return [p for p in b.uncovered if p.grad is not None]

    def _step_uncovered(self, coef=None, found_inf=None):
        """Parameters that no bucket kernel updates — MoE experts (excluded from data parallelism), ignored parameters —
        get the ordinary fused update here (their gradients scaled by the coefficient ``coef`` first, when given);
        their gradients are cleared like the bucketed ones. Their kernels count steps on the host, so with loss scaling the vote
        ``found_inf`` is read here — the one host synchronisation ``torch.amp.GradScaler.step`` also makes, and only for models
        that have such parameters — and an overflowed step leaves them alone."""
        left = self._uncovered()
        if left:
            import torch

            if found_inf is None or not bool(found_inf.item()):
                if coef is not None:
                    torch._foreach_mul_([p.grad for p in left], coef)
                super().step(only={id(p) for p in left})
            torch._foreach_zero_([p.grad for p in left])

    # ---- exponential moving average of the weights (``ema_decay``) -------------------------------------------------------
    def _ema_weight(self) -> float:
        """``w = float(1 − double(ema_decay))``: the host's double difference, rounded once to fp32 by the op."""
        d = self.ema_decay
        if d is None or not 0.0 < float(d) < 1.0:
            raise ValueError(f"ema_decay must be a number in (0, 1), got {d}")
        return 1.0 - float(d)

    def _ema_source(self, p):
        """The fp32 weights the EMA of a parameter outside the buckets (or of any parameter on the fallback) follows: its fp32 master,
        or the parameter itself when it is fp32 (a low-precision one without a master yet: its value, which the master starts from)."""
        import torch

        m = self.state[p].get("master") if p in self.state else None
        if m is not None and p.dtype != torch.float32:
            return m
        return p.data if p.dtype == torch.float32 else p.data.float()

    def _local_ema_pairs(self, params):
        """``[(source, ema)]`` of the local EMAs, kept as ``state[p]["ema"]`` in the source's memory layout (the kernel walks raw memory)."""
        import torch

        pairs = []
        for p in params:
            src = self._ema_source(p)
            if src.stride() != torch.empty_like(src).stride():   # not dense (a view with gaps): the kernel reads a contiguous copy
                src = src.contiguous()
            st = self.state[p]
            e = st.get("ema")
            if e is None:
                e = st["ema"] = torch.empty_like(src).copy_(src)
            elif e.device != src.device or e.dtype != torch.float32 or e.stride() != src.stride():   # e.g. a loaded checkpoint
                e = st["ema"] = torch.empty_like(src).copy_(e)
            pairs.append((src, e))
        return pairs

    def _local_ema_params(self):
        b = self._bucketing
        if not b.hyper_ops:
            return self._all_params()
        self._uncovered()
        return b.uncovered

    def _start_local_ema(self):
        """Before the first update: a local EMA starts from the weights the update begins with, as the bucket shards do."""
        local = self._local_ema_params()
        if any("ema" not in self.state[p] for p in local):
            self._local_ema_pairs(local)

    def _restart_local_ema(self, params):
        if self._ema:
            for src, e in self._local_ema_pairs(params or []):
                e.copy_(src)

    def _run_ema(self, op, stream_device):
        import torch

        from ...core import native

        op.set_weight(self._ema_weight())
        native().run_op(op, torch.cuda.current_stream(stream_device).cuda_stream, stream_device.index)
        self.kernel_launches += 1

    def _local_ema(self, role, params, vote):
        """One EmaOp launch over the local EMAs of ``params`` (the table is rebuilt only when a pointer changes); on the CPU the same
        three fp32 roundings in torch."""
        import torch

        pairs = self._local_ema_pairs(params)
        if not pairs:
            return
        if pairs[0][0].device.type != "cuda":
            w = torch.tensor(self._ema_weight(), dtype=torch.float32)
            for src, e in pairs:
                e.add_(torch.mul(torch.sub(src, e), w))
            return
        from ...core import native
        from ...ops.optim import _cached_plan

        plan = _cached_plan(self._ema_plans, role, [[s for s, _ in pairs], [e for _, e in pairs]])
        if getattr(plan, "ema_op", None) is None or plan.ema_vote != vote:
            plan.ema_op, plan.ema_vote = native().EmaOp(*plan.args(), self._ema_weight(), vote), vote
        self._run_ema(plan.ema_op, pairs[0][0].device)

    def _ema_after_step(self, vote=0):
        """Every ``ema_every``-th ``step()``: ``e ← e + w·(m − e)`` over every master (one launch for the bucket shards, at most one for
        the parameters outside the buckets), skipped on the device when the loss-scaled step's vote (``found_inf``) is set."""
        if not self._ema:
            return
        self._ema_calls += 1
        if self._ema_calls % self.ema_every:
            return
        b = self._bucketing
        if b.hyper_ops:
            if b.ema is None:
                raise RuntimeError("the EMA table was not built: not every bucket of the model has been initialised")
            self._run_ema(b.ema["op"], b.device)
        self._local_ema("local", self._local_ema_params(), vote)

    @contextlib.contextmanager
    def ema_weights(self):
        """Evaluate (or save) the model with its EMA weights: on entry every rank's parameters receive the EMA rounded once to their
        dtype, on exit the live weights come back bit for bit (the fp32 master is republished, rounded as every update kernel rounds
        it). A collective: every rank enters and leaves together. ``step()`` inside raises. Buffers (BatchNorm running statistics)
        are not averaged: they stay the live model's, as with ``AveragedModel(use_buffers=False)``."""
        import torch

        if not self._ema:
            raise RuntimeError("this optimizer keeps no EMA; build it with ema_decay=...")
        if self._ema_swapped:
            raise RuntimeError("already inside ema_weights()")
        local = self._local_ema_params()
        saved = []
        with torch.no_grad():
            for p, (_, e) in zip(local, self._local_ema_pairs(local)):   # the local EMAs are swapped in and out with copies
                saved.append((p, p.data.clone()))
                p.data.copy_(e)
            self._ema_publish(0)
        self._ema_swapped = True
        try:
            yield self
        finally:
            self._ema_swapped = False
            with torch.no_grad():
                self._ema_publish(1)
                for p, keep in saved:
                    p.data.copy_(keep)

    def _ema_publish(self, which):
        """Every bucket's EMA (0) or master (1) shard all-gathered into the weights, one launch per bucket."""
        import torch

        from ...core import native

        b = self._bucketing
        if not b.shards:
            return
        C, stream, dev = native(), torch.cuda.current_stream(b.device).cuda_stream, b.device.index
        for rec in b.shards:
            C.run_op(rec["publish"][which], stream, dev)
        self.kernel_launches += len(b.shards)

    def ema_state_dict(self):
        """``{parameter name: full-shape fp32 EMA}`` in the model's parameter order, on the CPU — for saving an averaged model for
        inference. A collective on the bucket path (an all-gather per bucket), like ``state_dict()``."""
        if not self._ema:
            raise RuntimeError("this optimizer keeps no EMA; build it with ema_decay=...")
        out = {}
        b = self._bucketing
        for rec in b.shards:
            for name, full in consolidate_shards(self._gather(rec["state"][-1], rec["group"]), rec["numel"], rec["layout"]).items():
                out[name] = full.cpu()
        local = self._local_ema_params()
        for i, (p, (_, e)) in enumerate(zip(local, self._local_ema_pairs(local))):
            out[self._param_names.get(id(p), f"param{i}")] = e.detach().reshape(p.shape).contiguous().cpu().clone()
        order = {n: i for i, n in enumerate(self._param_names.values())}
        return dict(sorted(out.items(), key=lambda kv: order.get(kv[0], len(order))))

    # ---- global gradient-norm clipping (``max_grad_norm``) ---------------------------------------------------------------
    @property
    def last_grad_norm(self):
        """Global L2 norm of the averaged gradient at the last step that clipped: a device fp32 0-d tensor with the same bits on
        every rank, overwritten by the next step (no host synchronisation). ``None`` before the first one."""
        return self._last_norm

    # ---- dynamic loss scaling (``loss_scaling``) --------------------------------------------------------------------------
    @property
    def last_step_skipped(self):
        """Whether the last step overflowed and was skipped on every rank: a device fp32 0-d tensor (1.0 / 0.0, the same bits
        on every rank), overwritten by the next step (no host synchronisation). ``None`` without ``loss_scaling`` or before the
        bucket kernels are live."""
        clip = self._bucketing.clip
        return clip["out"][2] if self.loss_scaling and clip is not None else None

    def set_loss_scale(self, scale):
        """The loss scale of the following steps: a 1-element fp32 tensor on the optimizer's device that the norm exchange reads
        when it runs (so a scaler may keep updating it in place), or ``None`` for a constant 1.
        :class:`bagua_b200.amp.ShardedGradScaler` calls this from ``step()``."""
        if not self.loss_scaling:
            raise RuntimeError("this optimizer was built without loss_scaling=True")
        if scale is not None and (scale.numel() != 1 or str(scale.dtype) != "torch.float32"):
            raise ValueError("the loss scale must be a 1-element fp32 tensor")
        if self._norm_pending and scale is not self._loss_scale:
            raise RuntimeError("clip_grad_norm_() has already computed this step's norm with another loss scale; hand the scale to the "
                               "optimizer before clipping (ShardedGradScaler.attach(optimizer)), or clip with max_grad_norm")
        self._loss_scale = scale

    def clip_grad_norm_(self, max_norm: float, norm_type: float = 2.0):
        """Clip by the global L2 norm of the averaged gradient with bound ``max_norm`` for this step and return the norm (device
        fp32 0-d tensor), like ``torch.nn.utils.clip_grad_norm_`` after a data-parallel all-reduce.

        With the bucket kernels live the gradients are consumed during backward, so this needs an optimizer built with
        ``max_grad_norm``: the call then computes the norm that the following ``step()`` applies (``step()`` computes it itself
        when this is not called). Without a peer engine the gradients are ordinary all-reduced tensors and the flat path clips
        them in place."""
        live = bool(self._bucketing.hyper_ops)
        if float(norm_type) != 2.0 and (live or self.max_grad_norm is not None):
            raise ValueError(f"the sharded fused optimizers clip by the L2 norm only, got norm_type={norm_type}")
        if not live:
            total = super().clip_grad_norm_(max_norm, norm_type)
            self._norm_pending, self._last_norm = True, total
            return total
        if self._bucketing.clip is None and self.accumulate_grads:
            raise RuntimeError("this in-bucket optimizer has no norm exchange; construct it with max_grad_norm=... to clip the accumulated gradient")
        if self._bucketing.clip is None:
            raise RuntimeError("the in-bucket optimizer applied this step's update during backward, so its gradients cannot be clipped "
                               "afterwards; construct it with max_grad_norm=... (make_sharded_fused_sgd / make_sharded_fused_adam) to clip "
                               "on this path")
        if self.loss_scaling and self._norm_pending:
            raise RuntimeError("with loss_scaling the norm exchange also casts the overflow vote and counts the step: clip_grad_norm_() can "
                               "run once per step")
        return self._launch_norm(max_norm).clone()

    def _launch_norm(self, max_norm):
        import torch

        from ...core import native

        clip = self._bucketing.clip
        loose = [p.grad for p in self._uncovered()]
        if loose:   # each rank adds the local Σx² of its parameters outside the buckets: every expert counts once in the total
            clip["extra"].copy_(torch.stack([torch.linalg.vector_norm(g, dtype=torch.float64) for g in loose]).square().sum())
            clip["extra_set"] = True
        elif clip["extra_set"]:
            clip["extra"].zero_()
            clip["extra_set"] = False
        if self.loss_scaling:   # the norm and the bound are the unscaled gradient's; no bound: the exchange only unscales and votes
            scale = clip["unit"] if self._loss_scale is None else self._loss_scale
            if scale.device != clip["out"].device:
                raise ValueError(f"the loss scale lives on {scale.device}, the optimizer's buckets on {clip['out'].device}")
            clip["scale"] = scale   # kept alive until the next exchange has replaced it
            clip["norm_op"].set_scale_ptr(scale.data_ptr())
        clip["norm_op"].set_max_norm(float("inf") if max_norm is None else float(max_norm))
        dev = clip["out"].device
        native().run_op(clip["norm_op"], torch.cuda.current_stream(dev).cuda_stream, dev.index)
        self.kernel_launches += 1
        self._norm_pending = True
        self._last_norm = clip["out"][0]
        return self._last_norm

    def step(self, closure=None):
        """Without a peer engine: the flat optimizer (clipping first with ``max_grad_norm``). Otherwise: publish the
        hyper-parameters; with ``max_grad_norm`` or ``loss_scaling`` run the norm exchange (unless ``clip_grad_norm_`` ran it);
        run the step program of the bucketing on the current stream (see :class:`_Bucketing`; empty when the bucket kernels of
        this iteration's backward already applied the update); then step the parameters outside the buckets, their gradients
        scaled by the exchange's coefficient. No host synchronisation, except with ``loss_scaling`` when the model has parameters
        outside the buckets (see ``_step_uncovered``). With ``accumulate_grads`` the update consumes the gradient accumulated since the
        last ``step()`` and the next backward starts a new sum, also when the step was skipped.

        With ``loss_scaling`` the exchange also unscales by the loss scale (``set_loss_scale``; 1 when ``step()`` is called
        without a scaler) and votes on overflow: a step whose averaged gradient holds an inf or a NaN changes no weight, no
        optimizer state and not the step count, on any rank (``last_step_skipped``)."""
        b = self._bucketing
        if self._ema_swapped:
            raise RuntimeError("step() inside ema_weights(): the parameters hold the EMA, leave the context first")
        if self._ema:
            self._start_local_ema()
        if not b.hyper_ops:
            if self.max_grad_norm is not None and not self._norm_pending:
                self._last_norm = super().clip_grad_norm_(self.max_grad_norm)
            self._norm_pending = False
            out = super().step(closure)
            self._ema_after_step()
            return out
        self._sync_hyper()
        coef = found_inf = None
        if b.clip is not None:
            if not self._norm_pending:
                self._launch_norm(self.max_grad_norm)
            self._norm_pending = False
            coef = b.clip["out"][1]
            found_inf = b.clip["out"][2] if self.loss_scaling else None
        if b.update_ops:
            # Ordering: the post-backward hook made this stream wait for the comm stream, so every phase-A bucket kernel (shard +
            # partials) has finished; the next iteration's bucket launches wait for ready events recorded after this step() on
            # this stream. So phase A, the exchanges and the updates of one PeerComm stay totally ordered, the shards and the
            # partials are never overwritten while read, and the weights are all-gathered before the next forward reads them.
            import torch

            from ...core import native

            if b.lamb is not None and b.lamb["ratio_op"] is None:
                raise RuntimeError(f"the {self._kind.upper()} per-parameter exchange was not built: not every bucket of the model has been initialised")
            C, stream, dev = native(), torch.cuda.current_stream(b.device).cuda_stream, b.device.index
            for op in b.pre_ops:
                C.run_op(op, stream, dev)
            if b.lamb is not None:
                C.run_op(b.lamb["ratio_op"], stream, dev)
            for op in b.update_ops:
                C.run_op(op, stream, dev)
        if self.accumulate_grads:
            self._restart_grad_sums()
        self._step_uncovered(coef, found_inf)
        self._grads_zeroed = True
        self.kernel_launches += b.launches
        self._ema_after_step(found_inf.data_ptr() if found_inf is not None else 0)
        return None

    def _register_shard(self, rec):
        b = self._bucketing
        b.covered.update(rec.get("param_ids", ()))
        b.uncovered = None
        b.shards.append(rec)
        if self._pending_state is not None:
            self._apply_to_shard(rec, self._pending_state)



# ---------------------------------------------------------------------------------------------------------------
# Gradient allreduce with the optimizer folded into the communication kernel
# ---------------------------------------------------------------------------------------------------------------
class ShardedFusedSGD(object):
    """Marker mix-in: see :func:`make_sharded_fused_sgd`."""


def _check_bound(max_grad_norm):
    if max_grad_norm is not None and not float(max_grad_norm) > 0:
        raise ValueError(f"max_grad_norm must be a positive number or None, got {max_grad_norm}")
    return None if max_grad_norm is None else float(max_grad_norm)


def _configure(opt, max_grad_norm, loss_scaling, accumulate_grads, ema_decay, ema_every):
    """The options every sharded in-bucket optimizer factory takes."""
    opt.max_grad_norm, opt.loss_scaling, opt.accumulate_grads = _check_bound(max_grad_norm), bool(loss_scaling), bool(accumulate_grads)
    if ema_decay is None:
        return opt
    if not 0.0 < float(ema_decay) < 1.0:
        raise ValueError(f"ema_decay must be a number in (0, 1) or None, got {ema_decay}")
    if int(ema_every) != ema_every or int(ema_every) < 1:
        raise ValueError(f"ema_every must be a positive integer, got {ema_every}")
    opt._ema, opt.ema_decay, opt.ema_every = True, float(ema_decay), int(ema_every)
    return opt


def make_sharded_fused_sgd(params, lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, max_grad_norm=None, loss_scaling=False,
                           accumulate_grads=False, ema_decay=None, ema_every=1):
    """SGD whose update runs *inside* each bucket's NVSwitch kernel (``allreduce_update_kernel``): reduce-scatter of the
    gradients → SGD(momentum) on this rank's 1/N shard with fp32 master weights → all-gather of the updated weights, one
    launch per bucket, overlapped with the rest of backward.  Optimizer state is sharded N ways (ZeRO-1-like) and the
    gradient bucket is cleared on the way out.  Use together with ``FusedGradientAllReduceAlgorithm``; with one process (or
    without a peer engine) it behaves like :class:`bagua_b200.ops.optim.FusedSGD`.

    ``max_grad_norm``: clip by the global L2 norm of the averaged gradient, as ``torch.nn.utils.clip_grad_norm_`` after a
    data-parallel all-reduce.  The bucket kernels then only reduce-scatter the gradients into an fp32 shard during backward
    (4 bytes per element / N of extra memory) and ``step()`` runs the norm exchange and the clipped update; see
    ``docs/algorithms.md``.

    ``loss_scaling``: dynamic loss scaling for fp16 training, driven by :class:`bagua_b200.amp.ShardedGradScaler`. The bucket
    program is the one of ``max_grad_norm`` (which stays optional: the norm it bounds and reports is the unscaled gradient's);
    the norm exchange also divides by the loss scale and decides, with the same bits on every rank, whether the step overflowed;
    an overflowed step changes nothing anywhere and does not count (``last_step_skipped``).

    ``accumulate_grads``: gradient accumulation over micro-batches in the fp32 shard. Every backward pass that communicates adds
    its averaged gradient into this rank's fp32 gradient shard (the bucket program is the one of ``max_grad_norm``, and the update
    always runs in ``step()``, with a coefficient of exactly 1 when nothing clips or unscales); ``step()`` applies the update to
    the sum, clipped and unscaled as a whole, and starts a new sum, also when loss scaling skips the step. ``zero_grad()`` between
    two ``step()`` calls discards the sum. Micro-batches under ``no_sync()`` add up locally in the bucket and join the sum with the
    next communicating backward. Needs ``FusedGradientAllReduceAlgorithm(average=True)``. Without a peer engine the bucket
    all-reduce averages the locally accumulated bucket in place on each communicating backward, so the sum is kept in the
    model's dtype there. Without the flag a second backward before ``step()`` overwrites the shard on the two-phase programs (and
    SGD / Adam without clipping update the weights inside every backward): only the last micro-batch reaches the update."""
    from ...ops.optim import FusedSGD

    class _ShardedFusedSGD(_ShardedStateMixin, FusedSGD, ShardedFusedSGD):
        _kind = "sgd"

    opt = _ShardedFusedSGD(params, lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov,
                           master_weights=True, zero_grad_in_step=True)
    return _configure(opt, max_grad_norm, loss_scaling, accumulate_grads, ema_decay, ema_every)


class ShardedFusedAdam(object):
    """Marker mix-in: see :func:`make_sharded_fused_adam`."""


def make_sharded_fused_adam(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, adamw=False, max_grad_norm=None, loss_scaling=False,
                            accumulate_grads=False, ema_decay=None, ema_every=1):
    """Adam / AdamW counterpart of :func:`make_sharded_fused_sgd`: the update of this rank's 1/N shard (fp32 master weights
    and both moments) runs inside each bucket's reduce-scatter → all-gather kernel (``allreduce_update_kernel``).  With one
    process (or without a peer engine) it behaves like :class:`bagua_b200.ops.optim.FusedAdam`.  ``max_grad_norm``,
    ``loss_scaling``, ``accumulate_grads``: see :func:`make_sharded_fused_sgd`."""
    from ...ops.optim import FusedAdam

    class _ShardedFusedAdam(_ShardedStateMixin, FusedAdam, ShardedFusedAdam):
        _kind = "adam"

    opt = _ShardedFusedAdam(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, adamw=adamw, master_weights=True,
                            zero_grad_in_step=True)
    return _configure(opt, max_grad_norm, loss_scaling, accumulate_grads, ema_decay, ema_every)


class ShardedFusedLamb(object):
    """Marker mix-in: see :func:`make_sharded_fused_lamb`."""


def make_sharded_fused_lamb(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01, max_grad_norm=None, loss_scaling=False,
                            accumulate_grads=False, ema_decay=None, ema_every=1):
    """LAMB (apex ``FusedLAMB`` semantics, see :class:`bagua_b200.ops.optim.FusedLAMB`) on the in-bucket sharded path: each rank
    keeps fp32 master weights and both moments for its 1/N slice of every bucket.

    The trust ratio ``‖w‖/‖u‖`` is a norm over a whole parameter, and a bucket's slices cut parameters anywhere, so the update
    cannot run during backward: each bucket kernel only reduce-scatters the averaged gradient into an fp32 shard (4 bytes per
    element / N), and ``step()`` then runs, on the current stream: the norm exchange when ``max_grad_norm`` is set (as for
    :func:`make_sharded_fused_sgd`), the moments of every shard with fp64 partial ``Σw²``/``Σu²`` per parameter segment, one
    exchange of the per-parameter sums between the ranks (every rank obtains the same fp32 ratios), and the update plus the
    all-gather of the weights per bucket — ``2·buckets + 1`` launches (+1 with clipping). A parameter group with
    ``weight_decay=0`` gets no layer adaptation (ratio 1). With one process, or without a peer engine, it behaves like
    :class:`bagua_b200.ops.optim.FusedLAMB`; see ``docs/algorithms.md``. ``loss_scaling``: see :func:`make_sharded_fused_sgd`;
    a skipped step also leaves the moments alone, and its ratio exchange runs with an unused result. ``accumulate_grads``: see
    :func:`make_sharded_fused_sgd`; the moments and the trust ratios see the accumulated gradient."""
    from ...ops.optim import FusedLAMB

    class _ShardedFusedLamb(_ShardedStateMixin, FusedLAMB, ShardedFusedLamb):
        _kind = "lamb"

    opt = _ShardedFusedLamb(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, master_weights=True, zero_grad_in_step=True)
    return _configure(opt, max_grad_norm, loss_scaling, accumulate_grads, ema_decay, ema_every)


class ShardedFusedLars(object):
    """Marker mix-in: see :func:`make_sharded_fused_lars`."""


def make_sharded_fused_lars(params, lr=1e-3, momentum=0.9, weight_decay=0.0, trust_coefficient=1e-3, max_grad_norm=None, loss_scaling=False,
                            accumulate_grads=False, ema_decay=None, ema_every=1):
    """LARS (see :class:`bagua_b200.ops.optim.FusedLARS`) on the in-bucket sharded path: each rank keeps fp32 master weights and
    the momentum for its 1/N slice of every bucket.

    The trust ratio ``trust_coefficient·‖w‖/(‖g‖ + wd·‖w‖)`` is a norm over a whole parameter, so the program is LAMB's (see
    :func:`make_sharded_fused_lamb`): each bucket kernel only reduce-scatters the averaged gradient into an fp32 shard, and
    ``step()`` runs the norm exchange when ``max_grad_norm`` or ``loss_scaling`` is set, the fp64 partial ``Σw²``/``Σg²`` of every
    shard per parameter segment, one exchange of the per-parameter sums between the ranks (every rank obtains the same bits), and
    the momentum, the update and the all-gather of the weights per bucket — ``2·buckets + 1`` launches (+1 with the norm
    exchange). The gradient the norms and the update see is the clipped / unscaled one. Put parameters with ``ndim ≤ 1``
    (biases, BatchNorm) in a ``weight_decay=0`` group: they get plain momentum SGD. With one process, or without a peer engine, it
    behaves like :class:`bagua_b200.ops.optim.FusedLARS`; ``loss_scaling``, ``accumulate_grads``: see :func:`make_sharded_fused_sgd`."""
    from ...ops.optim import FusedLARS

    class _ShardedFusedLars(_ShardedStateMixin, FusedLARS, ShardedFusedLars):
        _kind = "lars"

    opt = _ShardedFusedLars(params, lr=lr, momentum=momentum, weight_decay=weight_decay, trust_coefficient=trust_coefficient, master_weights=True,
                            zero_grad_in_step=True)
    return _configure(opt, max_grad_norm, loss_scaling, accumulate_grads, ema_decay, ema_every)


class ShardedFusedLion(object):
    """Marker mix-in: see :func:`make_sharded_fused_lion`."""


def make_sharded_fused_lion(params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0.0, max_grad_norm=None, loss_scaling=False, accumulate_grads=False,
                            ema_decay=None, ema_every=1):
    """Lion (see :class:`bagua_b200.ops.optim.FusedLion`) on the in-bucket sharded path: each rank keeps fp32 master weights and the
    one moment ``exp_avg`` for its 1/N slice of every bucket, 4 bytes per element / N less than Adam. The rule is element-wise, so
    like SGD and Adam the update runs inside each bucket's reduce-scatter → all-gather kernel (``allreduce_update_kernel``),
    overlapped with the rest of backward. With ``max_grad_norm``, ``loss_scaling`` or ``accumulate_grads`` the bucket kernels only
    reduce-scatter into the fp32 gradient shard and ``step()`` runs the update (``shard_update_kernel``); see
    :func:`make_sharded_fused_sgd`. With one process, or without a peer engine, it behaves like :class:`bagua_b200.ops.optim.FusedLion`."""
    from ...ops.optim import FusedLion

    class _ShardedFusedLion(_ShardedStateMixin, FusedLion, ShardedFusedLion):
        _kind = "lion"

    opt = _ShardedFusedLion(params, lr=lr, betas=betas, weight_decay=weight_decay, master_weights=True, zero_grad_in_step=True)
    return _configure(opt, max_grad_norm, loss_scaling, accumulate_grads, ema_decay, ema_every)


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
        sharded = isinstance(opt, _ShardedStateMixin)

        def hook(input):
            if sharded and opt._bucketing.hyper_ops:
                opt._sync_hyper()

        if sharded and opt._ema:   # the names ema_state_dict() gives the local EMAs
            opt._param_names = {id(p): name for name, p in bagua_ddp.module.named_parameters()}
        # _reset_buckets builds this hook after the last init_operations: every new shard has consumed the carried-over state
        # (checkpoint loaded before with_bagua, or the snapshot taken in tensors_to_buckets) — it must not be applied again
        opt._pending_state = None
        return hook

    def _carry_state_over(self):
        """Called at the start of every (re-)bucketing — with_bagua, the autotune service moving bucket boundaries every 100 steps,
        the find_unused_parameters rebuild: snapshot the sharded master weights / moments / step count in their consolidated
        (world-size and bucketing independent) form and forget the old bucketing; ``init_operations`` re-shards from the snapshot.
        Collective (an all-gather per state tensor), like re-bucketing itself. A gradient accumulated in the shards since the last
        ``step()`` (``accumulate_grads``) is carried over the same way, and the new phase-A ops add to it."""
        opt = self.optimizer
        if not isinstance(opt, _ShardedStateMixin):
            return
        if opt._bucketing.shards:
            opt._pending_state = opt.state_dict()
            if opt.accumulate_grads:
                opt._pending_state["grad_sum"] = opt._grad_sum()
        opt._bucketing = _Bucketing()

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

    def _clip_state(self, eng, bagua_ddp, bucket, device, scaled):
        """Buffers of the norm exchange, shared by all buckets: fp64 partial sums [bucket][CTA] (slots of unused CTAs stay 0), the
        fp64 Σx² of the parameters outside the buckets, out = {total, coef} in fp32, and the symmetric norm box (2·MAX_PEERS doubles,
        freed with the first bucket's other symmetric slices when the buckets are rebuilt). With loss scaling (``scaled``) the
        exchange is LossScaleNormOp: out = {total, coef, found_inf}, ``t`` is the effective step count it advances (32 bits on the
        device) and ``unit`` the scale of a step taken without a scaler."""
        import torch

        from ...core import native

        C = native()
        st = {"partials": torch.zeros(len(bagua_ddp.bagua_buckets), C.MAX_COMM_BLOCKS, dtype=torch.float64, device=device),
              "extra": torch.zeros((), dtype=torch.float64, device=device), "extra_set": False,
              "out": torch.zeros(3 if scaled else 2, dtype=torch.float32, device=device)}
        box = eng.alloc(2 * C.MAX_PEERS * 8)
        bucket._companion_slices.append(box)
        st["box"] = box
        if scaled:
            st["t"], st["unit"] = torch.zeros(1, dtype=torch.int32, device=device), torch.ones(1, dtype=torch.float32, device=device)
            st["norm_op"] = C.LossScaleNormOp(eng.comm, box.buf, box.offset, st["partials"].data_ptr(), st["partials"].numel(), st["extra"].data_ptr(),
                                              st["out"].data_ptr(), st["t"].data_ptr())
            return st
        st["norm_op"] = C.GradNormOp(eng.comm, box.buf, box.offset, st["partials"].data_ptr(), st["partials"].numel(), st["extra"].data_ptr(),
                                     st["out"].data_ptr())
        return st

    def init_operations(self, bagua_ddp, bucket):
        import os

        import torch

        from ...core import dtype_code, native
        from ...tensor import dense_strides

        bucket.clear_ops()
        eng = bucket._engine(self.process_group)
        opt = self.optimizer
        if eng is None or bucket._slice is None or not isinstance(opt, _ShardedStateMixin):
            return super().init_operations(bagua_ddp, bucket)
        kind = opt._kind
        per_param = kind in _PER_PARAMETER
        bk = opt._bucketing
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
        # the rule's fp32 state in _STATE_KEYS order: the master, then its moments
        state = (master,) + tuple(torch.zeros(vpr * per, dtype=torch.float32, device=flat.device) for _ in _STATE_KEYS[kind][1:])
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
        code = dtype_code(flat.dtype)
        clip, scaled, accum = opt.max_grad_norm is not None, opt.loss_scaling, opt.accumulate_grads
        exchange = clip or scaled   # the norm exchange runs in step(), so the update does too
        two_phase = exchange or per_param or accum
        layout = [(t.bagua_tensor_name, (t.bagua_getter_closure().data_ptr() - base) // flat.element_size(), t.bagua_getter_closure().numel(),
                   tuple(t.shape), tuple(dense_strides(t))) for t in bucket.tensors if not t.bagua_tensor_name.startswith("bagua_padding_tensor")]
        rec = {"bucket": bucket.name, "group": self.process_group, "numel": flat.numel(), "lo": lo, "hi": hi, "layout": layout,
               "state": state, "weights": wflat,
               "param_ids": [id(t) for t in bucket.tensors], "shard": None}
        if opt._ema:
            # the EMA shard starts equal to the master (a carried-over or loaded state overwrites both); publishing it, or the master
            # back, is one launch per bucket on entry to and exit from ema_weights()
            ema = master.clone()
            rec["state"] += (ema,)
            rec["publish"] = tuple(C.ShardPublishOp(eng.comm, wslice.buf, wslice.offset, nbytes, code, src.data_ptr(), use_mc, cfg) for src in (ema, master))
        bk.device = flat.device
        if two_phase:
            # phase A in the bucket program: reduce-scatter into the fp32 shard (added to it when accumulating) + per-CTA Σx² into
            # this bucket's row of partials (read by the norm exchange; nothing reads them without clipping); the update runs in step()
            if per_param and bk.lamb is None:
                bk.lamb = self._per_param_state(eng, bagua_ddp, bucket, flat.device)
            if exchange and bk.clip is None:
                bk.clip = self._clip_state(eng, bagua_ddp, bucket, flat.device, scaled)
            if exchange or per_param:
                row = (bk.clip if exchange else bk.lamb)["partials"][[b.name for b in bagua_ddp.bagua_buckets].index(bucket.name)]
            else:   # SGD / Adam / Lion accumulating without a norm exchange: partials nobody reads, and an update coefficient of exactly 1
                row = rec["partials"] = torch.zeros(C.MAX_COMM_BLOCKS, dtype=torch.float64, device=flat.device)
                if bk.unit is None:
                    bk.unit = torch.ones(1, dtype=torch.float32, device=flat.device)
            shard = rec["shard"] = torch.zeros(vpr * per, dtype=torch.float32, device=flat.device)
            args = (eng.comm, bucket._slice.buf, bucket._slice.offset, nbytes, code, shard.data_ptr(), row.data_ptr(), scale, True, use_mc, cfg)
            red = rec["grad_op"] = C.ShardGradOp(*args, True) if accum else C.ShardGradOp(*args)
            bucket.backend_bucket.append_op(red)
            bucket._ops_keepalive.append(red)
            coef_ptr = bk.clip["out"][1:].data_ptr() if exchange else (bk.unit.data_ptr() if not per_param else 0)
        fused_op, shard_op = _OPS[kind]
        ptrs = [t.data_ptr() for t in state]
        if per_param:
            op, moments = self._per_param_ops(eng, bk, rec, wslice, nbytes, code, use_mc, cfg, coef_ptr, kind == "lars")
        elif two_phase:
            op = getattr(C, shard_op)(eng.comm, wslice.buf, wslice.offset, nbytes, code, shard.data_ptr(), coef_ptr, *ptrs, use_mc, cfg)
        else:
            op = getattr(C, fused_op)(eng.comm, bucket._slice.buf, wslice.buf, bucket._slice.offset, wslice.offset, nbytes, code, *ptrs, scale, True,
                                      use_mc, cfg)
        if two_phase:
            bk.update_ops.append(op)
        else:
            bucket.backend_bucket.append_op(op)
        bucket._ops_keepalive.append(op)
        bucket.allreduce_variant = f"fused_{kind}_" + ("accum_" if accum else "") + ("scaled_" if scaled else "") + ("clip_" if clip else "") + ("multimem" if use_mc else "two_shot")
        rec["step_ops"] = (op, moments) if per_param else (op,)   # the update op first: state_dict() saves its count
        if scaled:   # the ops obey the exchange's vote and take the step count it keeps on the device
            for o in rec["step_ops"]:
                o.set_device_step(coef_ptr, bk.clip["t"].data_ptr())
        bk.hyper_ops += [(o, group_index) for o in rec["step_ops"]]
        bk.launches += len(rec["step_ops"])
        opt._register_shard(rec)
        opt._sync_hyper()
        if opt._ema and len(bk.shards) == len(bagua_ddp.bagua_buckets):
            # one launch per step over every bucket's [master, EMA] pair; with loss scaling it obeys the vote on the device
            from ...ops.optim import multi_tensor_plan

            plan = multi_tensor_plan([[r["state"][0] for r in bk.shards], [r["state"][-1] for r in bk.shards]])
            vote = bk.clip["out"][2:].data_ptr() if scaled else 0
            bk.ema = {"plan": plan, "op": C.EmaOp(*plan.args(), opt._ema_weight(), vote)}

    def _per_param_state(self, eng, bagua_ddp, bucket, device):
        """State of the per-parameter exchange of LAMB and LARS (LambRatioOp), shared by all buckets: a global index of the bucketed
        parameters (bucket order, padding excluded), the per-parameter outputs (fp32 LAMB ratio, unused by LARS; the global fp64
        pairs, {Σw², Σu²} for LAMB and {Σw², Σg²} for LARS), the stage-1 partial tables filled in bucket by
        bucket, the phase-A partial sums when no norm exchange provides them, and the symmetric box (2 halves × MAX_PEERS ×
        parameters × 2 doubles, freed with the first bucket's other symmetric slices when the buckets are rebuilt)."""
        import torch

        from ...core import native

        C = native()
        names = [t.bagua_tensor_name for b in bagua_ddp.bagua_buckets for t in b.tensors if not t.bagua_tensor_name.startswith("bagua_padding_tensor")]
        box = eng.alloc(C.LambRatioOp.box_bytes(len(names)))
        bucket._companion_slices.append(box)
        return {"index": {n: i for i, n in enumerate(names)}, "pending": set(names), "box": box,
                "ratio": torch.ones(len(names), dtype=torch.float32, device=device),
                "sums": torch.zeros(len(names), 2, dtype=torch.float64, device=device),
                "seg_ptr": [0] * len(names), "seg_nblk": [0] * len(names), "ratio_op": None,
                "partials": torch.zeros(len(bagua_ddp.bagua_buckets), C.MAX_COMM_BLOCKS, dtype=torch.float64, device=device)}

    def _per_param_ops(self, eng, bk, rec, wslice, nbytes, code, use_mc, cfg, coef_ptr, lars):
        """The ops of one LAMB or LARS bucket, after phase A: the stage-1 op over the shard's segments (parameter ∩ [lo, hi),
        shard-local offsets) — LAMB's moments over [master, shard, m1, m2], LARS's norms over [master, shard] — whose per-block
        partials the exchange sums per parameter, and the apply op. The exchange is built once every bucketed parameter has its
        table entry."""
        import torch

        from ...core import native
        from ...ops.optim import multi_tensor_plan

        C = native()
        lam = bk.lamb
        master, shard, lo, hi, dev = rec["state"][0], rec["shard"], rec["lo"], rec["hi"], bk.device
        lists = (master, shard) if lars else (master, shard) + tuple(rec["state"][1:3])
        Stage1 = C.LarsNormsOp if lars else C.LambMomentsOp
        segs, views = [], [[] for _ in lists]
        for name, off, n, _, _ in rec["layout"]:
            a, b = max(off, lo), min(off + n, hi)
            if a < b:
                segs.append((a - lo, b - lo, lam["index"][name]))
                for lst, buf in zip(views, lists):
                    lst.append(buf[a - lo: b - lo])
        if segs:
            plan = multi_tensor_plan(views)
            partials = torch.zeros(max(plan.n_blocks, 1), 2, dtype=torch.float64, device=dev)
            moments = Stage1(*plan.args(), coef_ptr, partials.data_ptr())
            blk = 0
            for a, b, t in segs:   # the plan gives each segment ceil(len / CHUNK) consecutive blocks, in segment order
                nb = (b - a + plan.CHUNK - 1) // plan.CHUNK
                lam["seg_ptr"][t], lam["seg_nblk"][t] = partials.data_ptr() + 16 * blk, nb
                blk += nb
            assert blk == plan.n_blocks
        else:   # an empty slice (small bucket, many ranks): no moments to update, but the rank still takes part in every exchange
            plan, partials = None, torch.zeros(1, 2, dtype=torch.float64, device=dev)
            moments = Stage1(0, 0, 0, 0, 0, 0, 65536, coef_ptr, partials.data_ptr())
        table = torch.tensor([v for s in segs for v in s] or [0, 0, 0], dtype=torch.int32, device=dev)
        if lars:
            op = C.ShardLarsOp(eng.comm, wslice.buf, wslice.offset, nbytes, code, shard.data_ptr(), coef_ptr, master.data_ptr(), rec["state"][1].data_ptr(),
                               table.data_ptr(), len(segs), lam["sums"].data_ptr(), use_mc, cfg)
        else:
            op = C.ShardLambOp(eng.comm, wslice.buf, wslice.offset, nbytes, code, master.data_ptr(), rec["state"][1].data_ptr(), rec["state"][2].data_ptr(),
                               table.data_ptr(), len(segs), lam["ratio"].data_ptr(), use_mc, cfg)
        rec["lamb_tables"] = (plan, partials, table, segs)
        bk.pre_ops.append(moments)
        lam["pending"] -= {name for name, *_ in rec["layout"]}
        if not lam["pending"]:
            ptrs = torch.tensor(lam["seg_ptr"], dtype=torch.int64, device=dev)
            nblk = torch.tensor(lam["seg_nblk"], dtype=torch.int32, device=dev)
            lam["tables"] = (ptrs, nblk)
            lam["ratio_op"] = C.LambRatioOp(eng.comm, lam["box"].buf, lam["box"].offset, ptrs.data_ptr(), nblk.data_ptr(), len(lam["index"]),
                                            lam["ratio"].data_ptr(), lam["sums"].data_ptr())
            bk.launches += 1
        return op, moments


class FusedGradientAllReduceAlgorithm(Algorithm):
    """Gradient allreduce whose buckets also apply the optimizer update (see :func:`make_sharded_fused_sgd` /
    :func:`make_sharded_fused_adam` / :func:`make_sharded_fused_lamb` / :func:`make_sharded_fused_lars` /
    :func:`make_sharded_fused_lion`)."""

    def __init__(self, optimizer, average: bool = True):
        self.optimizer = optimizer
        self.average = average

    def reify(self, process_group):
        # On the fallback path the bucket all-reduce runs in place on an already accumulated bucket: right only when it averages.
        if getattr(self.optimizer, "accumulate_grads", False) and not self.average:
            raise ValueError("accumulate_grads=True needs FusedGradientAllReduceAlgorithm(average=True): the accumulated gradient is the sum of the "
                             "micro-batches' averaged gradients")
        # optimizer state is carried across (re-)bucketing by the impl (tensors_to_buckets → _carry_state_over)
        return FusedGradientAllReduceAlgorithmImpl(process_group, self.optimizer, average=self.average)
