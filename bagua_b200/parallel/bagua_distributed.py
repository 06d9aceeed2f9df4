"""The data-parallel engine behind ``module.with_bagua(...)`` and the DDP-compatible wrapper.

Capability parity with ``bagua/torch_api/data_parallel/bagua_distributed.py`` (hooks :93-148, param build :155-212,
state broadcast :229-323, autotune :325-391, hook registration :417-481, bucket reset :483-496).

H100-first changes of the hot path:

* one forward-pre hook and one *post-accumulate-grad* hook per parameter whose closure is built once per
  (re)initialisation — the reference rebuilds the algorithm's hook closure for every gradient of every iteration
  (bagua_distributed.py:431);
* a gradient is handed to the native scheduler with its producing stream; the scheduler records ONE event per bucket;
* the end of backward does not block the host: the compute stream is made to wait (on the device) for the last bucket's
  completion event, so ``optimizer.step()`` launches while collectives are still in flight;
* all buckets of a model live in one contiguous arena of NVSwitch symmetric memory, so (a) each bucket op is a single
  fused kernel with no staging copy and (b) the fused optimizer updates the whole model with one launch.
"""
from __future__ import annotations

import collections
import logging
import os
import time
from types import MethodType
from typing import Dict, List, Optional, Tuple

import torch

from .. import communication as comm_mod
from .. import env
from ..bucket import BaguaBucket, BucketArena, bucket_arena
from ..core import to_bagua_datatype
from ..define import BaguaHyperparameter, TensorDeclaration
from ..core import native
from ..tensor import dense_strides
from ..utils import StatisticalAverage

logger = logging.getLogger(__name__)

_hooks_ext = [False]


def _native_hooks_ext():
    """The optional torch extension with the C++ autograd hooks, or ``None`` (not built / not loadable → Python hooks)."""
    if _hooks_ext[0] is False:
        try:
            from .. import _C_torch  # noqa: F401  (built by bagua_b200/_build.py:build_torch_hooks)

            _hooks_ext[0] = _C_torch
        except Exception as e:  # noqa: BLE001
            logger.warning("bagua_b200: native autograd hooks unavailable (%s); using Python hooks", e)
            _hooks_ext[0] = None
    return _hooks_ext[0]

__all__ = ["BaguaDistributedDataParallel"]


def _is_moe_param(param: torch.Tensor) -> bool:
    return bool(getattr(param, "expert", False))


class _States:
    """Bookkeeping object stored on the wrapped module (so a second ``with_bagua`` can undo the first)."""


def summarize_timeline(buckets: List[dict], step_begin: List[dict], backward_end: List[dict]) -> List[dict]:
    """Per training step: when backward ended, when the last bucket's communication ended, the part of it that was NOT hidden behind
    backward (``exposed_ms``) and the bucket that finished last.  A step is the window from its begin mark (forward-pre hook) to the
    next step's; bucket executions and the backward-end mark are assigned to the window they start in.  Steps without a backward
    (evaluation forward in train mode) or without communication (``no_sync``) are skipped."""
    begins = sorted(step_begin, key=lambda m: m["ms"])
    out = []
    for i, b in enumerate(begins):
        lo, hi = b["ms"], (begins[i + 1]["ms"] if i + 1 < len(begins) else float("inf"))
        mine = [x for x in buckets if lo <= x["start_ms"] < hi]
        ends = [m for m in backward_end if lo <= m["ms"] < hi]
        if not mine or not ends:
            continue
        last = max(mine, key=lambda x: x["start_ms"] + x["device_ms"])
        comm_end, bwd_end = last["start_ms"] + last["device_ms"], ends[-1]["ms"]
        out.append({"step": b["step"], "begin_ms": lo, "backward_end_ms": bwd_end, "comm_end_ms": comm_end, "exposed_ms": max(0.0, comm_end - bwd_end),
                    "last_bucket": last["bucket"], "buckets": len(mine), "comm_busy_ms": sum(x["device_ms"] for x in mine)})
    return out


class BaguaDistributedDataParallel:
    """The data-parallel engine behind ``module.with_bagua`` / ``DistributedDataParallel`` (reference
    bagua/torch_api/data_parallel/bagua_distributed.py:27-505): builds the tensor list and the buckets with the algorithm, installs
    the forward-pre / gradient / post-backward / optimizer hooks, broadcasts parameters and optimizer state from rank 0, talks to
    the autotune service, and hands ready gradients to the C++ scheduler."""
    def __init__(
        self,
        module: torch.nn.Module,
        optimizers: List[torch.optim.Optimizer],
        algorithm,
        process_group,
        bagua_module_name: Optional[str] = None,
        gradient_as_bucket_view: bool = True,
        find_unused_parameters: bool = False,
        broadcast_buffers: bool = True,
    ) -> None:
        self.module = module
        self.broadcast_buffers = broadcast_buffers
        self.bagua_module_name = bagua_module_name
        self.bagua_optimizers = optimizers
        self.process_group = process_group
        self.bagua_algorithm = algorithm.reify(process_group)
        self.gradient_as_bucket_view = gradient_as_bucket_view
        self.find_unused_parameters = find_unused_parameters
        self.parameters_to_ignore: List[str] = []
        for attr in ("_bagua_params_and_buffers_to_ignore", "_ddp_params_and_buffers_to_ignore"):
            if hasattr(module, attr):
                self.parameters_to_ignore.extend(getattr(module, attr))

        self.bagua_train_step_counter = 0
        self.bagua_buckets: List[BaguaBucket] = []
        self._bagua_autotune_last_report_time = time.time()
        self._bagua_autotune_completed = False
        self._is_post_backward_callback_queued = False
        self.require_backward_grad_sync = True
        self.autograd_graph_params: Dict[str, torch.nn.Parameter] = {}
        self.params_in_use = set()
        self._arena = None

        if hasattr(module, "_bagua_states"):
            self._reset_algorithm_state()
        module._bagua_states = _States()
        module._bagua_states._bagua_autograd_hooks = []
        module._bagua_states._bagua_framework_hooks = []

        self._bagua_backend = comm_mod.get_backend(self.bagua_module_name)
        if os.environ.get("BAGUA_INLINE_COMM", "0") == "1":
            # native bucket programs are launched by the autograd thread that completes the bucket (no hand-off to the
            # scheduler's worker thread); python ops keep using the worker. Required for CUDA-graph capture (utils/graph.py).
            self._bagua_backend.set_inline(True)
        self._bagua_hyperparameters = BaguaHyperparameter()
        self._report_metrics = env.is_report_metrics_switch_on()   # BAGUA_REPORT_METRICS / --report_metrics
        self._report_every = 100
        self._speed_metrics_switch_on = env.get_autotune_level() >= 1 or self._report_metrics
        self._speed_metrics = StatisticalAverage()
        self._on_cuda = any(p.is_cuda for p in module.parameters())
        self._stream_cache = 0
        self._native_state = None      # csrc/torch_hooks HookState when BAGUA_NATIVE_HOOKS=1
        self._native_hooked = []
        self._bagua_autotune_client = None
        if env.get_autotune_level() >= 1:
            from ..service.autotune_service import AutotuneClient

            port = comm_mod.get_autotune_service_port()
            assert port is not None, "autotune level > 0 but the autotune service was not started by init_process_group"
            self._bagua_autotune_client = AutotuneClient(comm_mod.get_autotune_service_host(), port)
            self._bagua_backend.set_record_spans(True)

        ddp = self

        def forward_pre_hook(mod, inputs):
            ddp._stream_cache = ddp._consumer_stream()  # backward runs on the forward's stream: one lookup per step, not per parameter
            ddp.autograd_graph_params.clear()
            if mod.training:
                ddp.bagua_train_step_counter += 1
                if getattr(ddp, "_timeline_on", False):
                    ddp._timeline_mark("begin")
                if ddp.bagua_algorithm.need_reset():
                    ddp._bagua_init_algorithm()
                ddp._fwd_pre_hook(inputs)
                ddp._record_speed_metrics_event()
                if ddp._bagua_autotune_client is not None and not ddp._bagua_autotune_completed:
                    ddp._bagua_autotune_step()
                if ddp._report_metrics:
                    ddp._log_metrics()
            ddp._is_post_backward_callback_queued = False
            if ddp._native_state is not None:
                ddp._native_state.new_pass(ddp.bagua_train_step_counter, ddp._stream_cache, ddp.require_backward_grad_sync)

        module._bagua_states._bagua_framework_hooks.append(module.register_forward_pre_hook(forward_pre_hook))
        self._bagua_init_algorithm()

    # ---------------------------------------------------------------------------------------------------------
    # parameters
    # ---------------------------------------------------------------------------------------------------------
    def bagua_build_params(self) -> List[Tuple[str, torch.nn.Parameter]]:
        """``(name, parameter)`` for every parameter that requires grad, is not ignored, is not a MoE expert parameter
        (experts are not data-parallel), deduplicated; sparse-gradient modules are rejected (reference :155-212)."""
        out: List[Tuple[str, torch.nn.Parameter]] = []
        seen = set()
        for module_name, sub in self.module.named_modules():
            if isinstance(sub, (torch.nn.Embedding, torch.nn.EmbeddingBag)) and sub.sparse:
                raise NotImplementedError("sparse gradient not supported yet")
            for pname, p in sub.named_parameters(recurse=False):
                full = f"{module_name}.{pname}" if module_name else pname
                if not p.requires_grad or full in self.parameters_to_ignore or _is_moe_param(p):
                    continue
                if self.find_unused_parameters and self.autograd_graph_params and full not in self.autograd_graph_params:
                    continue
                if id(p) in seen:
                    continue
                seen.add(id(p))
                out.append((full, p))
        return out

    # ---------------------------------------------------------------------------------------------------------
    # state broadcast
    # ---------------------------------------------------------------------------------------------------------
    def _bagua_broadcast_parameters(self):
        """Rank 0's parameters and optimizer state become everybody's (coalesced: one message per dtype)."""
        comm = self.process_group.get_global_communicator()
        if comm.nranks() == 1:
            return
        tensors = [p.data for _, p in self.bagua_build_params()]
        # The reference stops here (trainable, non-ignored parameters only, bagua_distributed.py:314-321). Replicas must
        # also agree on what is NOT trained: frozen parameters and buffers (BatchNorm statistics, position tables) are
        # synchronised like torch DDP does at construction; ignored names and MoE expert parameters stay rank-local.
        seen = set(t.data_ptr() for t in tensors)
        for name, p in self.module.named_parameters():
            if not p.requires_grad and name not in self.parameters_to_ignore and not _is_moe_param(p) and p.data_ptr() not in seen:
                seen.add(p.data_ptr())
                tensors.append(p.data)
        if self.broadcast_buffers:
            for name, b in self.module.named_buffers():
                if name not in self.parameters_to_ignore and b.numel() > 0 and b.data_ptr() not in seen:
                    seen.add(b.data_ptr())
                    tensors.append(b.data)
        if tensors:
            comm_mod.broadcast_coalesced(tensors, src=0, comm=comm)
        for opt in self.bagua_optimizers:
            self._bagua_broadcast_optimizer_state(opt)

    def _bagua_broadcast_optimizer_state(self, optimizer):
        if isinstance(optimizer, torch.optim.LBFGS):
            raise ValueError("cannot broadcast torch.optim.LBFGS state")
        comm = self.process_group.get_global_communicator()
        if getattr(optimizer, "collective_state_dict", False):
            return  # state sharded across ranks by construction (in-bucket optimizers): nothing to replicate
        sd = optimizer.state_dict()
        if len(sd["state"]) == 0:
            return
        state_tensors, scalars = [], collections.OrderedDict()
        for gi, group in enumerate(sd["param_groups"]):
            for k in sorted(group.keys()):
                if k != "params":
                    scalars[f"group{gi}.{k}"] = group[k]
            for pid in sorted(group["params"]):
                st = sd["state"].get(pid)
                if st is None:
                    continue
                for k in sorted(st.keys(), key=str):
                    v = st[k]
                    if isinstance(v, torch.Tensor):
                        state_tensors.append(v)
                    else:
                        scalars[f"state{pid}.{k}"] = v
        want = "cuda" if self._on_cuda else "cpu"
        on_dev = [t for t in state_tensors if t.device.type == want]
        off_dev = [t for t in state_tensors if t.device.type != want]
        if on_dev:
            comm_mod.broadcast_coalesced(on_dev, src=0, comm=comm)
        for t in off_dev:  # e.g. CPU "step" tensors of GPU optimizers
            dev = "cuda" if self._on_cuda else "cpu"
            tmp = t.to(dev)
            comm_mod.broadcast(tmp, src=0, comm=comm)
            t.copy_(tmp.to(t.device))
        scalars = comm_mod.broadcast_object(scalars, src=0, comm=comm)
        for gi, group in enumerate(optimizer.param_groups):
            for k in list(group.keys()):
                key = f"group{gi}.{k}"
                if k != "params" and key in scalars:
                    group[k] = scalars[key]
        pid_to_param = {}
        idx = 0
        for group in optimizer.param_groups:
            for p in group["params"]:
                pid_to_param[idx] = p
                idx += 1
        for key, v in scalars.items():
            if key.startswith("state"):
                pid_s, name = key[len("state"):].split(".", 1)
                p = pid_to_param.get(int(pid_s))
                if p is not None and p in optimizer.state:
                    optimizer.state[p][name] = v

    # ---------------------------------------------------------------------------------------------------------
    # autotune / bucketing
    # ---------------------------------------------------------------------------------------------------------
    def _tensor_declarations(self) -> List[TensorDeclaration]:
        return [
            TensorDeclaration(name=t.bagua_tensor_name, num_elements=t.bagua_getter_closure().numel(), dtype=to_bagua_datatype(t.bagua_getter_closure().dtype))
            for t in self._bagua_tensors
        ]

    def _bagua_autotune_register_tensors(self):
        if self._bagua_autotune_client is None:
            return
        # the allreduce variants are measured once on this fabric (every rank derives the same table: MAX-reduced event times) and
        # handed to the service, which then picks the kernel variant per bucket from the bucket's message size
        table = None
        if self._on_cuda:
            eng = self.process_group.peer_engine()
            if eng is not None and eng.world > 1:
                table = eng.variant_table or eng.calibrate()
        rsp = self._bagua_autotune_client.register_tensors(model_name=self.bagua_module_name, tensor_list=self._tensor_declarations(), variant_table=table)
        assert rsp.status_code == 200, f"Unexpected rsp={rsp}"

    def _bagua_autotune_get_buckets(self) -> List[List[torch.Tensor]]:
        if self._bagua_autotune_client is None:
            from ..service.autotune_task_manager import split_bucket_by_bucket_size

            size = self._bagua_hyperparameters.bucket_size or env.get_default_bucket_size()
            self._bagua_hyperparameters.bucket_size = size
            decl = split_bucket_by_bucket_size(self._tensor_declarations(), size)
            self._bagua_hyperparameters.buckets = decl
            return [[self._bagua_tensor_map[td["name"]] for td in b] for b in decl]
        self._flush_ready_spans()
        rsp = self._bagua_autotune_client.ask_hyperparameters(model_name=self.bagua_module_name, rank=env.get_rank(), train_iter=self.bagua_train_step_counter)
        assert rsp.status_code == 200, f"Unexpected rsp={rsp}"
        body = rsp.json()
        self._bagua_hyperparameters.update(body["recommended_hyperparameters"])
        self._bagua_autotune_completed = body["is_autotune_completed"]
        return [[self._bagua_tensor_map[td["name"]] for td in b] for b in body["recommended_hyperparameters"]["buckets"]]

    def _flush_ready_spans(self):
        """Tensor-ready order recorded by the native scheduler → autotune service (the reference streams OpenTelemetry
        spans from Rust, bagua-opentelemetry/src/exporter/agent.rs:31-43)."""
        if self._bagua_autotune_client is None:
            return
        spans = self._bagua_backend.pop_ready_spans()
        if not spans:
            return
        last_iter = spans[-1][2]
        payload = [
            {"trace_id": int(it), "action": "tensor_ready", "tensor_name": name, "start_time": int(t), "end_time": int(t)}
            for name, t, it in spans
            if it == last_iter
        ]
        try:
            self._bagua_autotune_client.report_tensor_execution_order(payload)
        except Exception as e:  # noqa: BLE001
            logger.debug("report_tensor_execution_order failed: %s", e)

    def _bagua_autotune_step(self):
        CYCLE_STEP = 100
        if self.bagua_train_step_counter != 0 and self.bagua_train_step_counter % CYCLE_STEP == 0:
            since = time.time() - self._bagua_autotune_last_report_time
            speed = self._speed_metrics.get(since)
            rsp = self._bagua_autotune_client.report_metrics(
                model_name=self.bagua_module_name,
                rank=env.get_rank(),
                train_iter=self.bagua_train_step_counter,
                hyperparameters=self._bagua_hyperparameters.dict(),
                speed=speed,
            )
            assert rsp.status_code == 200, f"Unexpected rsp={rsp}"
            self._reset_buckets()
            self._bagua_autotune_last_report_time = time.time()

    def _record_speed_metrics_event(self):
        if not self._speed_metrics_switch_on:
            return
        if self._on_cuda:
            pair = getattr(self, "_last_event_pair", None)
            if pair is not None:
                start, stop = pair
                try:
                    elapsed = start.elapsed_time(stop) / 1000.0
                    gb = sum(b.bytes() for b in self.bagua_buckets) / 1024.0 ** 3
                    if elapsed > 0:
                        self._speed_metrics.record(gb / elapsed)
                except RuntimeError as err:
                    logger.debug("ignore cuda err=%s", err)
            start_event = torch.cuda.Event(enable_timing=True)
            self._speed_metrics_end_event = torch.cuda.Event(enable_timing=True)
            torch.cuda.current_stream().record_event(start_event)
            self._last_event_pair = (start_event, self._speed_metrics_end_event)
        else:
            now = time.time()
            t0, t1 = getattr(self, "_last_time_pair", (None, None))
            if t0 is not None and t1 is not None and t1 > t0:
                gb = sum(b.bytes() for b in self.bagua_buckets) / 1024.0 ** 3
                self._speed_metrics.record(gb / (t1 - t0))
            self._last_time_pair = (now, None)

    # ---------------------------------------------------------------------------------------------------------
    # (re)initialisation
    # ---------------------------------------------------------------------------------------------------------
    def _bagua_init_algorithm(self):
        self._bagua_cleanup_algorithm()
        self._bagua_broadcast_parameters()
        self._bagua_tensors = self.bagua_algorithm.init_tensors(self)
        self._bagua_tensor_map = {t.bagua_tensor_name: t for t in self._bagua_tensors}
        self._bagua_autotune_register_tensors()
        self._reset_buckets()
        self._register_autograd_hooks()
        self._register_optimizer_hooks()

    @property
    def require_backward_grad_sync(self) -> bool:
        """Cleared inside ``no_sync()``: gradients accumulate locally and nothing is marked ready."""
        return self._require_backward_grad_sync

    @require_backward_grad_sync.setter
    def require_backward_grad_sync(self, value: bool):
        self._require_backward_grad_sync = bool(value)
        state = getattr(self, "_native_state", None)
        if state is not None:
            state.set_enabled(bool(value))

    def _bagua_cleanup_algorithm(self):
        # let in-flight work of the previous program drain before its buffers are recycled
        try:
            self._bagua_backend.wait_pending_comm_ops(self._consumer_stream(), not self._on_cuda)
        except Exception:  # noqa: BLE001
            pass

    def _consumer_stream(self) -> int:
        return torch.cuda.current_stream().cuda_stream if self._on_cuda else 0

    def _reset_buckets(self):
        raw = self._bagua_autotune_get_buckets()
        old = self.bagua_buckets
        for b in old:
            b.clear_ops()
        old_arena = self._arena
        self._arena = None
        if self.gradient_as_bucket_view and raw:
            sizes = [sum(t.bagua_getter_closure().numel() * t.bagua_getter_closure().element_size() for t in b) for b in raw]
            dev = raw[0][0].bagua_getter_closure().device
            # an algorithm may cut every suggested bucket into several pieces (one per optimizer parameter group): room for their padding
            pieces = max(1, int(getattr(self.bagua_algorithm, "bucket_pieces", 1)))
            self._arena = BucketArena(self.process_group, dev, BucketArena.required_bytes(sizes, slack=2 * 1024 * pieces))
        with bucket_arena(self._arena):
            self.bagua_buckets = self.bagua_algorithm.tensors_to_buckets(raw, self.gradient_as_bucket_view)
        for bucket in self.bagua_buckets:
            self.bagua_algorithm.init_operations(self, bucket)
        self._bagua_backend.register_ordered_buckets([b.backend_bucket for b in self.bagua_buckets])
        for b in old:
            b.release()
        if old_arena is not None:
            old_arena.free()
        self.params_in_use = set(name for name, _ in self.bagua_build_params())
        self._fwd_pre_hook = self.bagua_algorithm.init_forward_pre_hook(self)
        self._backward_hook = self.bagua_algorithm.init_backward_hook(self)
        self._post_backward_hook = self.bagua_algorithm.init_post_backward_hook(self)
        if self._native_hooked:  # native hooks hold the scheduler records and gradient addresses of the OLD buckets
            self._register_autograd_hooks()

    # ---------------------------------------------------------------------------------------------------------
    # per-bucket communication profile
    # ---------------------------------------------------------------------------------------------------------
    def _log_metrics(self):
        """``BAGUA_REPORT_METRICS=1``: every ``_report_every`` training steps rank 0 logs the smoothed communication speed and
        the per-bucket profile (the reference defines the switch, env.py:88-92, but nothing consumes it)."""
        step = self.bagua_train_step_counter
        if step == 1:
            self.comm_profile(True)
        if step % self._report_every or env.get_rank() != 0:
            return
        rows = self.comm_report(reset=True)
        speed = self._speed_metrics.get(30.0)
        logger.warning("[bagua metrics] module=%s step=%d comm_speed=%.3f GiB/s buckets=%s", self.bagua_module_name, step, speed,
                       [{k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items() if k in ("bucket", "variant", "bytes", "launches", "mean_ms", "algbw_GBps")}
                        for r in rows])

    def comm_profile(self, enable: bool = True):
        """Start / stop measuring every bucket's communication program (timing events on the comm stream, see
        ``Backend::set_profile``).  Costs two event records per bucket launch; off by default."""
        self._bagua_backend.set_profile(bool(enable))
        if enable:
            self._bagua_backend.bucket_stats(True)

    def comm_timeline(self, enable: bool = True):
        """Start / stop recording the per-bucket timeline: every execution of every bucket's op list with its start on the
        communication stream's device timeline and its duration (``Backend::set_timeline``), the moment backward ended on the compute
        stream in the same timebase, and the tensor-ready marks.  Off by default; costs two event records per bucket launch and one
        per step.  Read it with :meth:`comm_timeline_collect` or ``bagua_b200.utils.trace.export_chrome_trace``."""
        self._timeline_marks = []
        self._timeline_on = bool(enable)
        self._bagua_backend.set_record_spans(bool(enable) or self._bagua_autotune_client is not None)
        self._bagua_backend.set_timeline(bool(enable))

    def _timeline_mark(self, kind: str):
        """``kind`` = "begin" (forward-pre hook of a training step) or "backward_end" (post-backward hook, BEFORE the algorithm waits for
        communication).  No synchronisation: an event on the compute stream, or a host time stamp on the CPU backend."""
        marks = self._timeline_marks
        if len(marks) >= 16384:
            return
        if self._on_cuda:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(torch.cuda.current_stream())
            marks.append((self.bagua_train_step_counter, kind, ev, None))
        else:
            marks.append((self.bagua_train_step_counter, kind, None, time.monotonic_ns()))

    def comm_timeline_collect(self) -> dict:
        """Everything recorded since :meth:`comm_timeline` was switched on (and not collected yet):
        ``{"buckets": [{bucket, iteration, issue_ns, start_ms, device_ms, queue_ms}], "backward_end": [{step, ms}],
        "ready": [{tensor, iteration, ms}], "steps": [{step, backward_end_ms, comm_end_ms, exposed_ms, last_bucket}]}`` — ``ms`` values
        share one timebase (device time of the comm stream's reference event on GPUs, the host's monotonic clock on CPUs; tensor-ready
        marks are host times shifted to the same zero).  ``exposed_ms`` is how long communication ran on after backward had ended.
        Call after a ``torch.cuda.synchronize()`` — kernels still in flight are reported by the next call."""
        be = self._bagua_backend
        buckets = list(be.pop_bucket_timeline())
        ref_ns = be.timeline_ref_ns()
        resolved, keep = {"begin": [], "backward_end": []}, []
        for step, kind, ev, host_ns in getattr(self, "_timeline_marks", []):
            if ev is None:
                if host_ns >= ref_ns:
                    resolved[kind].append({"step": step, "ms": (host_ns - ref_ns) / 1e6})
            elif not ev.query():
                keep.append((step, kind, ev, host_ns))      # still in flight: reported by the next call
            else:
                ms = be.timeline_ms_of_event(ev.cuda_event)
                if ms >= 0:
                    resolved[kind].append({"step": step, "ms": ms})
        self._timeline_marks = keep
        ready = [{"tensor": name, "iteration": int(it), "ms": (t - ref_ns) / 1e6} for name, t, it in be.pop_ready_spans() if t >= ref_ns] \
            if self._bagua_autotune_client is None else []
        return {"buckets": buckets, "step_begin": resolved["begin"], "backward_end": resolved["backward_end"], "ready": ready,
                "steps": summarize_timeline(buckets, resolved["begin"], resolved["backward_end"])}

    def comm_report(self, reset: bool = False) -> List[dict]:
        """Per bucket: launches, mean / max device time of its op list, achieved GB/s over the bucket bytes (algorithmic
        bandwidth), mean host-side queueing delay and the kernel variant in use."""
        variants = {b.name: getattr(b, "allreduce_variant", None) for b in self.bagua_buckets}
        out = []
        for st in self._bagua_backend.bucket_stats(reset):
            n = max(int(st["count"]), 1)
            mean_ms = st["total_ms"] / n
            out.append({
                "bucket": st["name"], "ops": st["ops"], "variant": variants.get(st["name"]), "bytes": int(st["bytes"]), "launches": int(st["count"]),
                "mean_ms": mean_ms, "max_ms": st["max_ms"], "queue_ms": st["queue_ms"] / n,
                "algbw_GBps": (st["bytes"] / 1e9) / (mean_ms / 1e3) if st["count"] and mean_ms > 0 else 0.0,
            })
        return out

    def _delay_allreduce(self):
        for name, p in self.bagua_build_params():
            self._backward_hook(name, p)
        self._post_backward_hook()

    def _rebuild_for_used_parameters(self):
        """``find_unused_parameters``: the parameters that took part in this backward differ from the bucketed set, so
        exactly those are registered again and re-bucketed (the reference re-buckets at the same point,
        bagua_distributed.py:440-446).  Tensors that drop out get private storage first — the arena they lived in is
        recycled by ``_reset_buckets``."""
        old = list(getattr(self, "_bagua_tensors", []))
        self._bagua_tensors = self.bagua_algorithm.init_tensors(self)
        keep = set(id(t) for t in self._bagua_tensors)
        for t in old:
            if id(t) in keep:
                continue
            eff = t.bagua_getter_closure()
            if eff is None:
                continue
            private = torch.empty_strided(eff.shape, dense_strides(eff), dtype=eff.dtype, device=eff.device)
            private.copy_(eff)
            t.bagua_set_storage(private.untyped_storage(), 0)
        self._bagua_tensor_map = {t.bagua_tensor_name: t for t in self._bagua_tensors}
        self._bagua_autotune_register_tensors()
        self._reset_buckets()

    # ---------------------------------------------------------------------------------------------------------
    # hooks
    # ---------------------------------------------------------------------------------------------------------
    def _cleanup_autograd_hooks(self):
        st = self.module._bagua_states
        for h in st._bagua_autograd_hooks:
            h.remove()
        st._bagua_autograd_hooks.clear()
        # native hook records live on the MODULE state like the Python handles: a later with_bagua() builds a new engine object
        # and must be able to take down what its predecessor installed
        native_hooked = getattr(st, "_bagua_native_hooked", [])
        if native_hooked:
            ext, C = _native_hooks_ext(), native()
            for p, handle in native_hooked:
                ext.HookState.remove(p)
                C.tensor_handle_free(handle)
        st._bagua_native_hooked = []
        self._native_hooked = st._bagua_native_hooked
        self._native_state = None

    def _register_autograd_hooks(self):
        self._cleanup_autograd_hooks()
        st = self.module._bagua_states
        ddp = self

        def queue_post_backward():
            if not ddp._is_post_backward_callback_queued:
                ddp._is_post_backward_callback_queued = True
                # parameters with native hooks share the "already queued" flag of this backward pass
                if ddp._native_state is None or ddp._native_state.try_queue():
                    torch.autograd.Variable._execution_engine.queue_callback(ddp._real_post_backward_hook)

        def factory(name: str):
            def hook(param):
                if not ddp.require_backward_grad_sync:
                    return
                if ddp.find_unused_parameters:
                    ddp.autograd_graph_params[name] = param
                    if name not in ddp.params_in_use:  # not bucketed right now: picked up by the post-backward rebuild
                        queue_post_backward()
                        return
                ddp._backward_hook(name, param)
                queue_post_backward()

            return hook

        # Fast path for algorithms that keep the default "mark the gradient ready" hook (gradient all-reduce, ByteGrad, the fused
        # optimizer variants): one flat closure per parameter — pointer check, one call into the scheduler with the stream
        # cached at forward-pre — instead of four Python frames. ~400 parameters fire per BERT-large backward, on the thread
        # that also launches the backward kernels.
        from .algorithms.base import AlgorithmImpl

        default_hook = type(self.bagua_algorithm).init_backward_hook is AlgorithmImpl.init_backward_hook and not self.find_unused_parameters
        comm_names = getattr(self.bagua_algorithm, "_communication_tensor_names", set())
        mark = self._bagua_backend.mark_ready_on_stream

        def fast_factory(name: str, param):
            def hook(p):
                if not ddp.require_backward_grad_sync:
                    return
                bt = p._bagua_backend_tensor
                # pointer contract (the gradient is still the registered bucket view): verified on the first steps and then
                # periodically — it only breaks when user code replaces .grad, which shows up immediately
                step = ddp.bagua_train_step_counter
                if (step < 4 or not step & 63) and bt.data_ptr() != p.grad.data_ptr():
                    raise AssertionError("bagua backend tensor data_ptr should match parameter grad (the gradient must stay the bucket view: "
                                         "use zero_grad(set_to_none=False) and do not assign a new tensor to .grad)")
                mark(bt, ddp._stream_cache)
                if not ddp._is_post_backward_callback_queued:
                    queue_post_backward()

            return hook

        # Opt-in (BAGUA_NATIVE_HOOKS=1): the same fast path as a C++ hook object (csrc/torch_hooks) — no GIL, no Python frame per
        # parameter; Python is entered once per backward pass to queue the post-backward callback.
        ext = _native_hooks_ext() if (default_hook and os.environ.get("BAGUA_NATIVE_HOOKS", "0") == "1") else None
        if ext is not None:
            C = native()
            self._native_state = ext.HookState(C.backend_raw_ptr(self._bagua_backend), C.native_mark_ready_fn(), self._real_post_backward_hook)
            self._native_state.new_pass(self.bagua_train_step_counter, self._stream_cache, self.require_backward_grad_sync)
        for name, p in self.module.named_parameters():
            if p.requires_grad:
                fast = default_hook and name in comm_names and hasattr(p, "_bagua_backend_tensor")
                if fast and ext is not None and p.grad is not None:
                    handle = C.tensor_handle_new(p._bagua_backend_tensor)
                    if self._native_state.install(p, handle, p.grad.data_ptr(), name):
                        self._native_hooked.append((p, handle))
                        continue
                    C.tensor_handle_free(handle)
                st._bagua_autograd_hooks.append(p.register_post_accumulate_grad_hook(fast_factory(name, p) if fast else factory(name)))

    def _real_post_backward_hook(self):
        if getattr(self, "_timeline_on", False):
            self._timeline_mark("backward_end")
        self._post_backward_hook()
        if self._speed_metrics_switch_on:
            if self._on_cuda:
                torch.cuda.current_stream().record_event(self._speed_metrics_end_event)
            else:
                t0, _ = getattr(self, "_last_time_pair", (None, None))
                self._last_time_pair = (t0, time.time())
        if self.find_unused_parameters and set(self.autograd_graph_params.keys()) != self.params_in_use:
            self._rebuild_for_used_parameters()
            self._delay_allreduce()

    def _register_optimizer_hooks(self):
        hook = self.bagua_algorithm.init_post_optimizer_step_hook(self)
        bucketed = set()
        for t in getattr(self, "_bagua_tensors", []):
            bucketed.add(id(t))
        for optimizer in self.bagua_optimizers:
            if not hasattr(optimizer, "_bagua_original_step"):
                optimizer._bagua_original_step = optimizer.step
            if not hasattr(optimizer, "_bagua_original_zero_grad"):
                optimizer._bagua_original_zero_grad = optimizer.zero_grad

            def new_step(self_opt, *args, **kwargs):
                result = self_opt._bagua_original_step(*args, **kwargs)
                hook(self_opt)
                return result

            def new_zero_grad(self_opt, set_to_none: bool = False):
                # gradients are views into the bucket arena: they must stay allocated (SURVEY Appendix C)
                return self_opt._bagua_original_zero_grad(set_to_none=False)

            optimizer.step = MethodType(new_step, optimizer)
            optimizer._bagua_post_step_hook = hook  # fuse_step() triggers it too
            optimizer.zero_grad = MethodType(new_zero_grad, optimizer)
        # same contract for ``model.zero_grad()`` (nn.Module defaults to set_to_none=True since torch 2.0)
        module = self.module
        if not hasattr(module, "_bagua_original_zero_grad"):
            module._bagua_original_zero_grad = module.zero_grad

            def module_zero_grad(self_mod, set_to_none: bool = False):
                return self_mod._bagua_original_zero_grad(set_to_none=False)

            module.zero_grad = MethodType(module_zero_grad, module)

    def _reset_algorithm_state(self):
        st = self.module._bagua_states
        for h in getattr(st, "_bagua_framework_hooks", []):
            h.remove()
        if hasattr(st, "_bagua_autograd_hooks"):
            self._cleanup_autograd_hooks()

    # used by the default algorithm hooks ------------------------------------------------------------------------
    def mark_tensor_ready(self, tensor: torch.Tensor):
        """Fast ready mark: the scheduler records one event on the current stream when the tensor's bucket completes."""
        self._bagua_backend.mark_ready_on_stream(tensor._bagua_backend_tensor, self._consumer_stream())

    def wait_pending_comm_ops(self) -> int:
        """Order the current stream after every scheduled bucket (device-side wait on GPU, host wait on CPU).  Also the point where
        a peer kernel that gave up (barrier time-out / abort) in an earlier iteration becomes a Python exception: its error word is
        mirrored in host-mapped memory, so the check costs a load, not a synchronisation."""
        n = self._bagua_backend.wait_pending_comm_ops(self._consumer_stream(), not self._on_cuda)
        if self._on_cuda:
            eng = getattr(self.process_group, "_peer_engine", None)
            if eng is not None:
                eng.check_error()
        return n
