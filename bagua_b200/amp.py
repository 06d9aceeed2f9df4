"""Dynamic loss scaling (fp16 training) for the in-bucket sharded optimizers.

``torch.amp.GradScaler.step`` unscales ``p.grad``, looks for overflow on the host and then decides whether to call
``optimizer.step()``. With the bucket kernels live there is nothing for it to look at: the gradients were reduced into 1/N shards
and cleared during backward. :class:`ShardedGradScaler` keeps everything else of torch's scaler — the scale is torch's device
tensor, ``update()`` is torch's growth / backoff — and lets an optimizer built with ``loss_scaling=True`` unscale, vote on overflow
and skip the step on the device, see ``docs/algorithms.md``."""
from __future__ import annotations

from torch.amp.grad_scaler import GradScaler, OptState

__all__ = ["ShardedGradScaler"]


def _live(optimizer) -> bool:
    """The optimizer's update runs in the bucket kernels / its native step program (not the flat fallback)."""
    from .parallel.algorithms.gradient_allreduce import _ShardedStateMixin

    return isinstance(optimizer, _ShardedStateMixin) and bool(optimizer._bucketing.hyper_ops)


class ShardedGradScaler(GradScaler):
    """``torch.amp.GradScaler`` (device ``"cuda"``) that can drive ``make_sharded_fused_{sgd,adam,lamb,lars,lion}(loss_scaling=True)``::

        scaler.scale(loss).backward()
        scaler.step(opt)        # no host synchronisation while the bucket kernels are live
        scaler.update()

    ``scale()``, ``update()``, ``get_scale()``, ``state_dict()`` and ``load_state_dict()`` are torch's. For any optimizer whose
    gradients are ordinary tensors (torch optimizers, a sharded optimizer on the fallback path) ``step()`` and ``unscale_()`` are
    torch's too."""

    def __init__(self, init_scale: float = 2.0 ** 16, growth_factor: float = 2.0, backoff_factor: float = 0.5, growth_interval: int = 2000,
                 enabled: bool = True, device: str = "cuda"):
        super().__init__(device, init_scale=init_scale, growth_factor=growth_factor, backoff_factor=backoff_factor,
                         growth_interval=growth_interval, enabled=enabled)

    def attach(self, optimizer):
        """Hand the scale tensor to a live ``loss_scaling=True`` optimizer ahead of ``step()`` — needed only when
        ``optimizer.clip_grad_norm_(bound)`` is called between ``backward()`` and ``step()``, so that it bounds the norm of the
        unscaled gradient. A no-op for every other optimizer."""
        if self._enabled and _live(optimizer) and optimizer.loss_scaling:
            if self._scale is None:
                self._lazy_init_scale_growth_tracker(optimizer._bucketing.device)
            optimizer.set_loss_scale(self._scale)

    def unscale_(self, optimizer):
        """torch's ``unscale_``; raises for a live in-bucket optimizer, whose gradients no longer exist as tensors."""
        if self._enabled and _live(optimizer):
            raise RuntimeError("the in-bucket optimizer consumed its gradients during backward, so they cannot be unscaled as tensors; to clip, "
                               "build it with max_grad_norm=... or call optimizer.clip_grad_norm_(bound) after ShardedGradScaler.attach(optimizer): "
                               "both bound the norm of the unscaled gradient")
        return super().unscale_(optimizer)

    def step(self, optimizer, *args, **kwargs):
        """For a live in-bucket optimizer built with ``loss_scaling=True``: hand it the device scale tensor, run its step program
        (which unscales, votes on overflow with the same bits on every rank and skips the step everywhere if it did overflow) and
        record its device ``found_inf`` for ``update()``. For a live in-bucket optimizer without ``loss_scaling``: an error,
        because its update already ran during backward. Otherwise torch's ``step()``."""
        if not self._enabled or not _live(optimizer):
            return super().step(optimizer, *args, **kwargs)
        if not optimizer.loss_scaling:
            raise RuntimeError("this in-bucket optimizer applied the update during backward, with the still-scaled gradients: a step that "
                               "overflowed can no longer be skipped. Build it with loss_scaling=True (make_sharded_fused_sgd / _adam / _lamb / _lars / _lion)")
        if "closure" in kwargs or args:
            raise RuntimeError("Closure use is not currently supported if GradScaler is enabled.")
        self._check_scale_growth_tracker("step")
        state = self._per_optimizer_states[id(optimizer)]
        if state["stage"] is OptState.STEPPED:
            raise RuntimeError("step() has already been called since the last update().")
        optimizer.set_loss_scale(self._scale)
        retval = optimizer.step()
        found_inf = optimizer.last_step_skipped
        # update() may add the entries of several optimizers in place: it gets a copy, the optimizer keeps its own word
        state["found_inf_per_device"] = {found_inf.device: found_inf.reshape(1).clone()}
        state["stage"] = OptState.STEPPED
        return retval
