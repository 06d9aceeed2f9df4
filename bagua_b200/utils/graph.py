"""Whole-step CUDA graph capture for launch-bound training loops.

The VGG16 step issues ≈ 120 kernels and the host needs about as long to launch them as the GPU needs to run them, so any
extra host work — data loading, logging, a slower CPU — shows up as idle GPU time.
:class:`GraphedTrainStep` records one complete step (zero_grad → forward → loss → backward → optimizer) into a
``torch.cuda.CUDAGraph`` and replays it with a single launch; new inputs are copied into the static input tensors first.

Scope (deliberately narrow, see docs/kernels.md):

* one rank (or a micro-step under ``no_sync()``): the gradient hooks are switched off for the step, nothing is communicated;
* several ranks: the scheduler is put in *inline issue* mode (``Backend::set_inline``, csrc/scheduler.h) — the autograd thread
  that marks a bucket's last gradient launches the bucket's kernels itself on the communication stream, so every CUDA call
  of the step happens on capturing streams (fork: comm stream waits for the "gradients ready" event; join: the main stream
  waits for the bucket's done event in the post-backward hook).  The peer kernels read their barrier epochs from device
  memory, so a replay is indistinguishable from a fresh launch as long as every rank replays the same graph.  Bucket
  programs that contain python ops (gloo / NCCL fallbacks, QAdam's momentum op) run on the worker thread and are refused;
* optimizers whose kernel arguments do not change from step to step: :class:`bagua_b200.ops.optim.FusedSGD`,
  ``torch.optim.SGD`` and torch optimizers constructed with ``capturable=True``.  :class:`FusedAdam` passes the step count
  (bias correction) by value and is rejected.  A changed learning rate is detected on the next call and triggers a re-capture.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch

__all__ = ["GraphedTrainStep", "graph_safe_optimizer"]


def graph_safe_optimizer(opt: torch.optim.Optimizer) -> Optional[str]:
    """``None`` when ``opt`` may run inside a captured graph, else the reason it may not."""
    from ..ops.optim import FusedAdam, FusedLAMB, FusedLARS, FusedLion, FusedSGD

    if isinstance(opt, FusedSGD):
        return None
    if isinstance(opt, FusedAdam):
        return "FusedAdam passes the step count to its kernel by value (bias correction changes every step)"
    if isinstance(opt, FusedLAMB):
        return "FusedLAMB passes the step count to its kernels by value (bias correction changes every step)"
    if isinstance(opt, FusedLARS):
        return ("FusedLARS cannot be captured: it builds its multi-tensor tables and momentum buffers on the host at the step that "
                "first sees a parameter and may copy gradients into fresh buffers each step")
    if isinstance(opt, FusedLion):
        return ("FusedLion cannot be captured: it builds its multi-tensor tables and moment buffers on the host at the step that first "
                "sees a parameter and may copy gradients into fresh buffers each step")
    if isinstance(opt, torch.optim.SGD):
        return None
    if all(g.get("capturable", False) for g in opt.param_groups):
        return None
    return f"{type(opt).__name__} keeps per-step host state; construct it with capturable=True"


class GraphedTrainStep:
    """``step = GraphedTrainStep(model, train_step, (x, y), optimizers=[opt])`` then ``loss = step(x, y)`` every iteration.

    ``train_step(*inputs) -> loss`` is the eager step (it must do everything, including ``zero_grad`` and ``optimizer.step``);
    it is run ``warmup`` times on a side stream (cuDNN autotuning, lazy optimizer state, bucket construction), captured once,
    and replayed afterwards.  The warm-up iterations are real optimisation steps on the example batch (as in PyTorch's own
    whole-network capture recipe).  The returned loss is a static device tensor that the next call overwrites."""

    def __init__(self, model: torch.nn.Module, train_step: Callable[..., torch.Tensor], example_inputs: Sequence[torch.Tensor],
                 optimizers: Sequence[torch.optim.Optimizer] = (), warmup: int = 3):
        self.model, self.train_step, self.optimizers = model, train_step, list(optimizers)
        for opt in self.optimizers:
            if getattr(opt, "native_ops_in_step", False):
                raise NotImplementedError(f"{type(opt).__name__} runs native kernels from step() with per-call host state (box parity, "
                                          "step count, the restart of an accumulated gradient); it cannot be captured in a CUDA graph")
            why = graph_safe_optimizer(opt)
            if why is not None:
                raise ValueError(f"optimizer cannot be captured in a CUDA graph: {why}")
        inner = getattr(model, "inner", None)  # DistributedDataParallel wrapper: .inner is the engine
        self.ddp = getattr(model, "bagua_ddp", None) or (inner if hasattr(inner, "require_backward_grad_sync") else None)
        # world 1 communicates too in self-peer mode (BAGUA_SELF_PEER=1: the bucket programs exist and run with this GPU as its only peer)
        multi = self.ddp is not None and (self.ddp.process_group.size() > 1 or getattr(self.ddp.process_group, "_peer_engine", None) is not None)
        self.communicates = bool(multi and self.ddp.require_backward_grad_sync)
        if self.communicates and getattr(self.ddp, "_speed_metrics_switch_on", False):
            raise NotImplementedError("autotune / speed metrics record timing events every step and cannot be captured; switch them off")
        if not torch.cuda.is_available() or any(not t.is_cuda for t in example_inputs):
            raise RuntimeError("GraphedTrainStep needs a CUDA device and CUDA example inputs")
        self.static_inputs: List[torch.Tensor] = [t.detach().clone() for t in example_inputs]
        self.warmup = max(int(warmup), 3)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.static_loss: Optional[torch.Tensor] = None
        self._captured_hyper = None
        self.replays = 0
        self.captures = 0

    # -- capture ---------------------------------------------------------------------------------------------------------
    def _hyper(self):
        return tuple(tuple(sorted((k, v) for k, v in g.items() if isinstance(v, (int, float, bool)))) for opt in self.optimizers for g in opt.param_groups)

    def _without_hooks(self):
        """Gradient hooks call into the scheduler (event records + a worker thread): switched off for the step — there is
        nothing to communicate in the supported configurations."""
        ddp = self.ddp if not self.communicates else None   # communicating replicas keep their hooks: the buckets are captured too

        class _Ctx:
            def __enter__(self_inner):
                self_inner.prev = ddp.require_backward_grad_sync if ddp is not None else None
                if ddp is not None:
                    ddp.require_backward_grad_sync = False

            def __exit__(self_inner, *exc):
                if ddp is not None:
                    ddp.require_backward_grad_sync = self_inner.prev

        return _Ctx()

    def capture(self):
        """First call: warm up (real steps), verify that the bucket programs are capturable, capture.  Later calls (a
        hyper-parameter changed): capture only — nothing executes during a capture, so no extra optimisation step is taken."""
        first = self.graph is None
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        backend = self.ddp._bagua_backend if self.communicates else None
        if backend is not None:
            backend.set_inline(True)
            backend.set_profile(False)      # the profile polls timing events (cudaEventQuery), which a capture forbids
            issued_before, scheduled_before = backend.inline_total(), backend.scheduled_total()
        with self._without_hooks():
            if first:
                with torch.cuda.stream(side):
                    for _ in range(self.warmup):
                        self.train_step(*self.static_inputs)
                torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            if backend is not None and first:
                inline, total = backend.inline_total() - issued_before, backend.scheduled_total() - scheduled_before
                if total == 0 or inline != total:
                    raise NotImplementedError(f"{total - inline} of {total} bucket launches went through the scheduler's worker thread "
                                              "(python ops in the bucket program): this algorithm cannot be captured in a CUDA graph")
                if not backend.graph_capturable():
                    raise NotImplementedError("a bucket op passes step-dependent arguments (Adam step count, rotating shift_one partner): "
                                              "a CUDA graph would freeze them")
            self.graph = torch.cuda.CUDAGraph()
            # thread_local: torch's NCCL watchdog thread polls its events with cudaEventQuery, which a global-mode capture
            # would take as a violation; the threads that launch into the capture (this one, autograd's device thread) only
            # make capturable calls
            with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
                self.static_loss = self.train_step(*self.static_inputs)
        self._captured_hyper = self._hyper()
        self.captures += 1

    # -- replay ----------------------------------------------------------------------------------------------------------
    def __call__(self, *inputs: torch.Tensor) -> torch.Tensor:
        if self.graph is None or self._hyper() != self._captured_hyper:  # first call, or e.g. a learning-rate schedule stepped
            self.capture()
        for dst, src in zip(self.static_inputs, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        self.replays += 1
        return self.static_loss
