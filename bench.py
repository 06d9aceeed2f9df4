#!/usr/bin/env python
"""Headline benchmark (BASELINE.json): VGG16 images/s (GradientAllReduce) AND BERT-large samples/s (ByteGrad), bf16, synthetic
data of the named shapes, random-init weights, device-timed (CUDA events), max over ranks.

``python bench.py --gpus N --steps K --warmup W`` (launched through torchrun for N > 1) prints ONE JSON line from rank 0.  The top-level ``metric`` / ``value`` / ``e2e`` / … describe the VGG16 workload — the reference's own
synthetic benchmark shape (examples/benchmark/synthetic_benchmark.py: bs 32/GPU, SGD, cross-entropy, fixed random batch) — and
the ``bert_large_bytegrad`` block carries the same fields for the second half of the metric: BERT-large question answering on
SQuAD-shaped batches (seq 384, bs 6/GPU as examples/squad/README.md:19-28) with the ByteGrad algorithm and AdamW.

Arms (``--impl``):
  ours           the framework as a user gets it: fused NVSwitch bucket kernels, fused optimizers.
  nccl_baseline  SAME models / optimizers / bucketing / scheduler with ``BAGUA_ALLREDUCE_VARIANT=nccl``: one NCCL all-reduce per
                 bucket, ByteGrad as the reference's 7-step compress → alltoall → … pipeline on torch.distributed — the re-expression
                 of the reference's schedule that SURVEY §6 prescribes as the same-box baseline.  Context only.
  ddp            stock PyTorch: ``DistributedDataParallel`` + ``torch.optim`` + eager modules (no bagua_b200 kernel). Context.
  reference      the unmodified reference from ``baseline/_ref``; it cannot be installed offline in this image (Rust core: cargo,
                 setuptools_rust, mpicxx and a downloaded NCCL are all missing, DESIGN.md §3), so the arm reports itself unavailable.

Every N runs the SAME program: at N = 1 the engine is built in self-peer mode (``BAGUA_SELF_PEER=1``: this GPU is its own and
only peer), so the bucket kernels (reduce-scatter → optimizer → all-gather, fused ByteGrad) do at N = 1 exactly the per-GPU work
they do at N = 8 — the scaling base is not flattered by a cheaper single-GPU code path.

After each workload's timed regions six more steps run with the scheduler's per-bucket timeline on; the summary (``comm_timeline``:
communication left exposed after backward, the bucket that finishes last, device time per bucket) explains the step time, it is
not part of any timed region.  A failure of the second workload is reported in its block and does not take the first one's line with it.

``--dump-outputs DIR`` writes, after the timed region of each workload, what its last timed step computed as float32 ``.npy``
files: ``<workload>_loss.npy`` (the loss the step returned) and ``<workload>_params_sample.npy`` (the updated weights at a fixed,
seeded sample of 2^20 positions of the parameters in model order).  Inputs and initial weights come from fixed seeds, so two runs
or two builds with the same arguments can be compared output for output.  Such a run uses deterministic algorithms throughout
(see main()) and is therefore slower than the plain throughput run.

``--selftest-cpu`` runs the same code end to end on the host with tiny shapes for the test-suite (marked ``selftest``).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.abspath(__file__))
# context only (BASELINE.md): VGG16 fp32, Bagua + Bagua-Net, 32 x V100 over 100 Gb TCP (rust/bagua-net/README.md:52-67); BASELINE.json publishes
# no number for this hardware / dtype, so `vs_baseline` is null
PUBLISHED_CONTEXT = {"vgg16_img_s_per_gpu": 126.5, "hardware": "32x V100, fp32, 100 Gb TCP", "source": "rust/bagua-net/README.md:52-67"}


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--impl", default="ours", choices=["ours", "reference", "nccl_baseline", "ddp"])
    p.add_argument("--workloads", default="vgg16,bert", help="comma list out of vgg16, resnet50, bert")
    p.add_argument("--batch-size", type=int, default=32, help="images per GPU (vgg16 / resnet50)")
    p.add_argument("--bert-batch-size", type=int, default=6, help="sequences per GPU (reference: examples/squad/README.md)")
    p.add_argument("--seq-len", type=int, default=384)
    p.add_argument("--momentum", type=float, default=0.0)
    p.add_argument("--no-e2e", action="store_true")
    p.add_argument("--no-verify", action="store_true", help="skip the fused-vs-unfused weight check that precedes the timed region")
    p.add_argument("--no-self-peer", action="store_true", help="N = 1: plain single-GPU path (flat fused optimizer, no bucket kernels)")
    p.add_argument("--profile", default="", help="write a torch.profiler kernel table of 3 steps per workload to this file prefix (not a benchmark run)")
    p.add_argument("--fused-shard", dest="fused_shard", action="store_true", default=None,
                   help="fold the SGD update into the allreduce kernel (sharded optimizer state); default: on whenever the group has a peer engine")
    p.add_argument("--no-fused-shard", dest="fused_shard", action="store_false")
    p.add_argument("--cuda-graph", action="store_true", help="experimental: replay the whole VGG16 step from a CUDA graph (utils.graph.GraphedTrainStep)")
    p.add_argument("--dump-outputs", default="", metavar="DIR", help="write the last timed step's loss and a seeded sample of the updated weights as .npy files")
    p.add_argument("--selftest-cpu", action="store_true", help=argparse.SUPPRESS)
    p.add_argument("--image-size", type=int, default=224, help=argparse.SUPPRESS)
    return p.parse_args()


def reference_arm(args):
    ref = os.path.join(REPO, "baseline", "_ref")
    why = None
    if not os.path.isdir(os.path.join(ref, "bagua")):
        why = ("reference not installed: `pip install --no-index --no-build-isolation --find-links /opt/wheelhouse --target baseline/_ref /root/reference` fails at "
               "metadata generation (No module named 'setuptools_rust'); its Rust core also needs cargo/rustc, mpicxx and a downloaded NCCL tarball — none available offline")
    else:
        sys.path.insert(0, ref)
        try:
            import bagua_core  # noqa: F401
        except Exception as e:  # noqa: BLE001
            why = f"reference python package present but its native module bagua_core is missing: {e!r}"
    if why is None:
        why = "reference arm runner not wired: baseline/_ref unexpectedly importable — rerun after inspecting it"
    if int(os.environ.get("RANK", "0")) == 0:  # under torchrun every rank gets here: one line, from rank 0
        print(json.dumps({"impl": "reference", "unavailable": why}))
    return 0


class ClockSampler:
    """nvidia-smi clock / throttle-reason sampler.  ONE sampler runs for the whole process (nvidia-smi takes a moment to deliver
    its first line, so a sampler started right before a 90 ms timed region can come back empty); every sample carries
    nvidia-smi's own timestamp and ``region()`` / ``stop(begin, end)`` select the samples taken DURING a timed region."""

    FIELDS = ("timestamp,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
              "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.proc = None
        self.index = index
        self._buf = []
        self._thread = None

    def start(self):
        import threading

        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.FIELDS}", "--format=csv,noheader,nounits", "-lms", "50"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:  # noqa: BLE001
            self.proc = None
            return self

        def pump():
            for line in self.proc.stdout:
                self._buf.append(line)

        self._thread = threading.Thread(target=pump, daemon=True)
        self._thread.start()
        return self

    @staticmethod
    def now() -> float:
        import time

        return time.time()

    def _parse(self):
        import datetime

        rows = []
        for line in list(self._buf):
            parts = [x.strip() for x in line.split(",")]
            if len(parts) < 8:
                continue
            try:
                ts = datetime.datetime.strptime(parts[0], "%Y/%m/%d %H:%M:%S.%f").timestamp()
                rows.append((ts, float(parts[1]), float(parts[2]), float(parts[3]), parts[4:8]))
            except ValueError:
                continue
        return rows

    def summary(self, begin: float = None, end: float = None):
        """Clock record of the samples with ``begin <= t <= end`` (host wall clock; all samples when omitted)."""
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        rows = self._parse()
        note = None
        if not rows:   # the looping sampler delivered nothing (died, or an nvidia-smi that rejects the interval): ask once, now
            try:
                one = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.FIELDS}", "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=20).stdout
                self._buf.extend(ln + "\n" for ln in one.splitlines() if ln.strip())
                rows = self._parse()
                note = "the looping sampler delivered no line; one query right after the timed region"
            except Exception:  # noqa: BLE001
                rows = []
        sel = [r for r in rows if (begin is None or r[0] >= begin - 0.05) and (end is None or r[0] <= end + 0.05)]
        if not sel and rows and begin is not None:   # region shorter than the sampling period: take the two nearest samples
            sel = sorted(rows, key=lambda r: min(abs(r[0] - begin), abs(r[0] - end)))[:2]
            note = note or "no sample inside the timed region (50 ms sampling period): nearest samples"
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({n for r in sel for n, v in zip(names, r[4]) if v == "Active"})
        sm = sorted(r[1] for r in sel)
        under_load = sm[len(sm) // 2:] if len(sm) > 3 else sm    # upper half: the samples under load
        out = {"sm_mhz": statistics.median(under_load) if under_load else None, "sm_max_mhz": max((r[2] for r in sel), default=None),
               "power_w_max": max((r[3] for r in sel), default=None), "reasons": reasons, "samples": len(sel)}
        if note:
            out["note"] = note
        return out

    def stop(self, begin: float = None, end: float = None):
        out = self.summary(begin, end)
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=5)
            except Exception:  # noqa: BLE001
                self.proc.kill()
        return out


class Ctx:
    """Everything a workload needs from the launch environment."""


def make_ctx(args):
    import torch
    import torch.distributed as dist

    c = Ctx()
    c.args = args
    c.world = int(os.environ.get("WORLD_SIZE", "1"))
    c.rank = int(os.environ.get("RANK", "0"))
    c.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    c.cpu = args.selftest_cpu
    if c.cpu:
        c.dev, c.dtype = torch.device("cpu"), torch.float32
    else:
        torch.cuda.set_device(c.local_rank)
        c.dev, c.dtype = torch.device("cuda", c.local_rank), torch.bfloat16
    c.torch, c.dist = torch, dist

    def sync_all():
        if c.world > 1:
            dist.barrier()
        if not c.cpu:
            torch.cuda.synchronize()

    def timed(fn, steps, whole_loop=False):
        """Exactly ``steps`` calls (or one ``fn(steps)`` loop) between barrier + synchronize pairs; CUDA events on the launching
        stream; MAX over ranks."""
        sync_all()
        if c.cpu:
            import time

            t0 = time.perf_counter()
            fn(steps) if whole_loop else [fn(i) for i in range(steps)]
            ms = torch.tensor([(time.perf_counter() - t0) * 1e3])
            if c.world > 1:
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            return float(ms.item())
        import time

        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.nvtx.range_push("timed")
        h0 = time.perf_counter()
        start.record()
        if whole_loop:
            fn(steps)
        else:
            for i in range(steps):
                fn(i)
        end.record()
        c.last_host_ms = (time.perf_counter() - h0) * 1e3   # time the host needed to ISSUE the steps (diagnostic: ~= the device time when launch-bound)
        torch.cuda.nvtx.range_pop()
        torch.cuda.synchronize()
        ms = torch.tensor([start.elapsed_time(end)], device=c.dev)
        if c.world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            dist.barrier()
        return float(ms.item())

    c.sync_all, c.timed = sync_all, timed
    return c


def launch_counter(c):
    if c.args.impl == "ddp":
        return lambda: 0
    from bagua_b200.core import native

    return native().launch_count  # every kernel of this library counts itself (csrc/common.h: count_launch)


DUMP_SAMPLE = 1 << 20   # weights per workload in --dump-outputs (4 MB of float32)


def sample_params(torch, params, n=DUMP_SAMPLE, seed=20240601):
    """float32 values of the parameters (flattened and concatenated in model order) at ``n`` positions drawn from a fixed seed."""
    params = list(params)
    sizes = [p.numel() for p in params]
    total = sum(sizes)
    pos = torch.randint(0, total, (min(n, total),), generator=torch.Generator().manual_seed(seed)).sort().values
    out, off = [], 0
    for p, k in zip(params, sizes):
        lo, hi = torch.searchsorted(pos, off), torch.searchsorted(pos, off + k)
        if hi > lo:
            out.append(p.detach().reshape(-1)[(pos[lo:hi] - off).to(p.device)].float().cpu())
        off += k
    return torch.cat(out)


def measure(c, name, train_step, dev_batch, host_batches, to_model_format, per_step_items, unit, finish=None, params=None):
    """Warm-up, device-timed region, e2e region (pinned host batches → prefetcher → step → loss read-back).  With
    ``--dump-outputs`` the loss and a weight sample of the last timed step are kept in ``c.dumps`` before anything else runs."""
    torch = c.torch
    args = c.args
    from bagua_b200.utils.data import DevicePrefetcher, LossReader

    sampler = getattr(c, "sampler", None)
    warm = max(args.warmup, 3)
    loss = None
    for _ in range(warm):
        loss = train_step(*dev_batch)
    if args.profile and not c.cpu:
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            for _ in range(3):
                train_step(*dev_batch)
            torch.cuda.synchronize()
        if c.rank == 0:
            with open(f"{args.profile}.{name}.txt", "w") as f:
                f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=60, max_name_column_width=90))
    count = launch_counter(c)
    c.sync_all()
    n0 = count()
    holder = {"loss": loss}

    def one(_i):
        holder["loss"] = train_step(*dev_batch)

    t_begin = ClockSampler.now()
    ms = c.timed(one, args.steps)
    t_end = ClockSampler.now()
    if finish is not None:
        finish()
    launches = count() - n0
    host_ms = getattr(c, "last_host_ms", None)
    host_ms = host_ms / args.steps if host_ms is not None else None
    clocks = sampler.summary(t_begin, t_end) if sampler is not None else None
    loss_val = float(holder["loss"].detach().float().item())     # the loss of the last timed step, read after the timed region
    if loss_val != loss_val or loss_val in (float("inf"), float("-inf")):
        raise SystemExit(f"{name}: non-finite loss {loss_val} after the timed region — the number would be a throughput of nothing")
    if args.dump_outputs and params is not None:
        c.dumps[f"{name}_loss"] = holder["loss"].detach().float().reshape(1).cpu().numpy()
        c.dumps[f"{name}_params_sample"] = sample_params(torch, params()).numpy()
    value = per_step_items * c.world * args.steps / (ms / 1e3)
    e2e = None
    if not args.no_e2e:
        reader = LossReader(c.dev, lag=int(os.environ.get("BAGUA_BENCH_LOSS_LAG", "2")))

        def loop(steps):
            for batch in DevicePrefetcher(host_batches(steps), c.dev, to_model_format):
                reader.push(train_step(*batch))
            return reader.flush()

        try:
            loop(max(args.warmup, 3))   # the prefetcher's side-stream buffers and the cast kernels warm up too
            ms_e2e = c.timed(loop, args.steps, whole_loop=True)
            if finish is not None:
                finish()
            first = next(iter(host_batches(1)))
            h2d = sum(t.numel() * t.element_size() for t in first)
            e2e = {"value": per_step_items * c.world * args.steps / (ms_e2e / 1e3), "unit": unit, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                   "ms_per_step": ms_e2e / args.steps, "last_loss": reader.last}
        except Exception as exc:  # noqa: BLE001 - the device-timed number above must still be reported
            e2e = {"error": f"{type(exc).__name__}: {exc}"}
    return {"value": value, "unit": unit, "ms_per_step": ms / args.steps, "gpu_launches": int(launches), "clocks": clocks, "e2e": e2e, "final_loss": loss_val,
            "host_issue_ms_per_step": host_ms}


def timeline_probe(c, model, step_fn, dev_batch, finish, steps=6):
    """AFTER the timed regions: a few more steps with the scheduler's per-bucket timeline on (engine.comm_timeline): when each bucket's
    communication ran on the comm stream, when backward ended on the compute stream, and how many milliseconds of communication were NOT
    hidden behind backward in each step — the attribution of the gap between N = 1 and N > 1.  Never fails the benchmark."""
    try:
        eng = model.bagua_ddp
        torch = c.torch
        eng.comm_timeline(True)
        for _ in range(steps):
            step_fn(*dev_batch)
        if finish is not None:
            finish()
        if not c.cpu:
            torch.cuda.synchronize()
        tl = eng.comm_timeline_collect()
        eng.comm_timeline(False)
        rows = tl["steps"][1:] or tl["steps"]          # the first step after the switch pays for event creation
        if not rows:
            return {"steps": 0}
        exposed = sorted(r["exposed_ms"] for r in rows)
        last = {}
        for r in rows:
            last[r["last_bucket"]] = last.get(r["last_bucket"], 0) + 1
        per_bucket = {}
        for b in tl["buckets"]:
            per_bucket.setdefault(b["bucket"], []).append(b["device_ms"])
        return {"steps": len(rows), "exposed_ms_median": exposed[len(exposed) // 2], "exposed_ms_max": exposed[-1],
                "comm_busy_ms_median": sorted(r["comm_busy_ms"] for r in rows)[len(rows) // 2],
                "step_begin_to_backward_end_ms_median": sorted(r["backward_end_ms"] - r["begin_ms"] for r in rows)[len(rows) // 2],
                "bucket_finishing_last": max(last, key=last.get), "buckets_per_step": rows[0]["buckets"],
                "device_ms_per_bucket_median": {k: sorted(v)[len(v) // 2] for k, v in sorted(per_bucket.items())[:64]},
                "what": "engine.comm_timeline: per-bucket device timeline of the comm stream vs the end of backward on the compute stream, "
                        f"{len(rows)} untimed steps after the measurement"}
    except Exception as e:  # noqa: BLE001 - diagnostics only
        return {"error": f"{type(e).__name__}: {e}"[:300]}


def _bucket_programs(model):
    """The op list the scheduler runs per bucket, as the native core reports it (kinds such as ``allreduce_sgd``, ``bytegrad_fused``,
    ``allreduce_multimem``; a ``python`` entry would be a torch.distributed fallback) with how many buckets carry each program."""
    import collections
    import re

    progs = collections.Counter(re.sub(r"^bucket \S+ ", "", b.backend_bucket.print_ops()) for b in model.bagua_buckets)
    return {k: v for k, v in sorted(progs.items())}


def verify_fused_update(c, build_model, fused_model, optimizer, batch, loss_fn, lr, steps=2):
    """Outside every timed region: the update rule of the fused bucket kernels (reduce-scatter → SGD on fp32 master shards →
    all-gather) against a plain twin — same architecture and initial weights, gradients all-reduced in FP32 by torch.distributed,
    fp32 master weights updated by hand.  Same RNG seed before each twin's step so dropout masks coincide.

    Tolerance per element: one ulp of the weight dtype (the model copy is the fp32 master rounded to bf16) plus what rounding the
    gradient SUM to bf16 may move the weight — the NVLS flavour (``multimem.ld_reduce … .acc::f32.bf16x2``) accumulates in fp32 inside
    the switch but returns bf16, 2^-8 relative on the gradient, i.e. ``lr · 2^-8 · |g|`` per step; the peer ld/st flavour sums the
    bf16 gradients in fp32 registers and is exact.  A few violations in 10^4 (cuDNN's atomics make the twins' own gradients differ
    in the last bit) are recorded; more than 1 % means the update rule itself is wrong and the benchmark refuses to report a number."""
    torch, dist = c.torch, c.dist
    twin = build_model()
    twin.load_state_dict({k: v.clone() for k, v in fused_model.state_dict().items()})
    masters = [p.detach().float().clone() for p in twin.parameters()]
    w0 = [m.clone() for m in masters]
    gabs = [torch.zeros_like(m) for m in masters]
    for s in range(steps):
        torch.manual_seed(4242 + s)
        optimizer.zero_grad()
        loss_fn(fused_model, *batch).backward()
        optimizer.step()
        torch.manual_seed(4242 + s)
        for p in twin.parameters():
            p.grad = None
        loss_fn(twin, *batch).backward()
        with torch.no_grad():
            for p, m, ga in zip(twin.parameters(), masters, gabs):
                g = p.grad.float()
                if c.world > 1:
                    dist.all_reduce(g)
                    g /= c.world
                ga += g.abs()
                m.add_(g, alpha=-lr)
                p.copy_(m)
    if not c.cpu:
        fused_model.bagua_ddp.wait_pending_comm_ops()
        torch.cuda.synchronize()
    eps = 2.0 ** -7 if c.dtype == torch.bfloat16 else 2.0 ** -22
    viol, total, worst, num, den = 0, 0, 0.0, 0.0, 0.0
    for a, b, z, ga in zip(fused_model.parameters(), twin.parameters(), w0, gabs):
        a32, b32 = a.detach().float(), b.detach().float()
        d = (a32 - b32).abs()
        tol = torch.maximum(a32.abs(), b32.abs()) * eps + lr * (2.0 ** -7) * ga + 1e-7
        viol += int((d > tol).sum().item())
        total += d.numel()
        worst = max(worst, float((d / tol).max().item()))
        num += float((a32 - b32).pow(2).sum().item())
        den += float((b32 - z).pow(2).sum().item())
    del twin, masters, w0, gabs
    frac = viol / max(total, 1)
    out = {"what": f"{steps} steps of the fused bucket kernels vs fp32 all-reduce + hand-written SGD on a twin model",
           "tolerance": "1 ulp of the weight dtype + lr * 2^-7 * |g| (bf16 rounding of the in-switch gradient sum)",
           "fraction_outside_tolerance": frac, "worst_diff_over_tolerance": worst,
           "rel_l2_of_weight_diff_vs_update": (num / den) ** 0.5 if den > 0 else 0.0, "ok": bool(frac <= 1e-3)}
    if frac > 1e-2:
        raise SystemExit(f"fused bucket update disagrees with the unfused oracle on {frac:.2%} of the weights — refusing to report a throughput of a wrong update: {out}")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# workloads
# ---------------------------------------------------------------------------------------------------------------------
def run_cnn(c, model_name):
    torch, args = c.torch, c.args
    import torch.nn.functional as F

    from bagua_b200.models import get_model

    world, dev, dtype, cpu = c.world, c.dev, c.dtype, c.cpu
    bs, img = args.batch_size, args.image_size
    lr = 0.01 * world
    torch.manual_seed(1234)

    def build():
        m = get_model(model_name)
        if args.impl == "ddp" and hasattr(m, "fuse_epilogues"):
            m.fuse_epilogues = False  # stock eager Conv2d → ReLU → MaxPool2d modules on this arm
        m = m.to(dev).to(dtype)
        return m.to(memory_format=torch.channels_last) if not cpu else m

    def loss_fn(m, x, y):
        return F.cross_entropy(m(x).float(), y)

    model = build()
    verify = None
    finish = None
    cfg = {}
    if args.impl == "ddp":
        if world > 1:
            model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[c.local_rank], gradient_as_bucket_view=True)
        optimizer = torch.optim.SGD(model.parameters(), lr=lr, momentum=args.momentum)
        cfg["optimizer"] = f"torch.optim.SGD(momentum={args.momentum}) on bf16 parameters"
        cfg["allreduce_variants"] = ["torch DDP (NCCL)"]
    else:
        import bagua_b200 as bagua
        from bagua_b200.ops.optim import FusedSGD
        from bagua_b200.parallel.algorithms import Algorithm

        eng = bagua.communication._get_default_group().peer_engine() if not cpu else None
        fused = args.fused_shard if args.fused_shard is not None else (eng is not None)
        if fused:
            from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_sgd

            optimizer = make_sharded_fused_sgd(model.parameters(), lr=lr, momentum=args.momentum)
            algorithm = FusedGradientAllReduceAlgorithm(optimizer)
            cfg["optimizer"] = "SGD fused into the bucket reduce-scatter→all-gather kernel (fp32 master weights, state sharded N ways)"
        else:
            optimizer = FusedSGD(model.parameters(), lr=lr, momentum=args.momentum, master_weights=True, zero_grad_in_step=True)
            algorithm = Algorithm.init("gradient_allreduce")
            cfg["optimizer"] = f"FusedSGD(momentum={args.momentum}, fp32 master weights), one flat kernel per step"
        model = model.with_bagua([optimizer], algorithm)
        cfg["allreduce_variants"] = sorted({getattr(b, "allreduce_variant", "none") for b in model.bagua_buckets})
        cfg["buckets"] = len(model.bagua_buckets)
        cfg["bucket_programs"] = _bucket_programs(model)
        finish = model.bagua_ddp.wait_pending_comm_ops
        if fused and not args.no_verify and model_name == "vgg16" and args.momentum == 0.0:
            xv = torch.randn(bs, 3, img, img, device=dev).to(dtype)
            xv = xv.contiguous(memory_format=torch.channels_last) if not cpu else xv
            yv = torch.randint(0, 1000, (bs,), device=dev)
            verify = verify_fused_update(c, build, model, optimizer, (xv, yv), loss_fn, lr)

    torch.manual_seed(1234 + c.rank)
    x_dev = torch.randn(bs, 3, img, img, device=dev).to(dtype)
    x_dev = x_dev.contiguous(memory_format=torch.channels_last) if not cpu else x_dev
    y_dev = torch.randint(0, 1000, (bs,), device=dev)
    n_host = 4
    pin = (lambda t: t) if cpu else (lambda t: t.pin_memory())
    x_host = [pin(torch.randn(bs, 3, img, img)) for _ in range(n_host)]
    y_host = [pin(torch.randint(0, 1000, (bs,))) for _ in range(n_host)]

    def train_step(x, y):
        optimizer.zero_grad()
        loss = loss_fn(model, x, y)
        loss.backward()
        optimizer.step()
        return loss

    step_fn = train_step
    if args.cuda_graph and args.impl == "ours" and not cpu:
        from bagua_b200.utils.graph import GraphedTrainStep

        step_fn = GraphedTrainStep(model, train_step, (x_dev, y_dev), optimizers=[optimizer])
        step_fn(x_dev, y_dev)

    def to_model_format(x, y):
        if cpu:
            return x.to(dtype), y
        out = torch.empty(x.shape, dtype=dtype, device=x.device, memory_format=torch.channels_last)
        out.copy_(x)                      # fp32 NCHW → bf16 NHWC in ONE kernel on the prefetch stream
        return out, y

    def host_batches(n):
        for i in range(n):
            yield x_host[i % n_host], y_host[i % n_host]

    res = measure(c, model_name, step_fn, (x_dev, y_dev), host_batches, to_model_format, bs, "images/s", finish, params=model.parameters)
    if args.impl != "ddp" and not args.cuda_graph:
        res["comm_timeline"] = timeline_probe(c, model, step_fn, (x_dev, y_dev), finish)
    algo = "GradientAllReduce"
    res["metric"] = f"{model_name} synthetic-ImageNet training throughput ({algo})"
    res["config"] = dict(cfg, model=model_name, global_batch=bs * world, per_gpu_batch=bs, image=f"3x{img}x{img}", parallelism=f"dp{world}",
                         algorithm=algo, lr=lr, momentum=args.momentum, cuda_graph=bool(args.cuda_graph),
                         l2_policy="working set (276 MB bf16 weights + activations) far exceeds the 50 MB L2 of an H100; no explicit flush")
    if verify is not None:
        res["verify"] = verify
    del model, optimizer
    return res


def run_bert(c):
    torch, args = c.torch, c.args
    from bagua_b200 import models

    world, dev, dtype, cpu = c.world, c.dev, c.dtype, c.cpu
    bs, seq = args.bert_batch_size, args.seq_len
    cfgm = models.bert_large_config() if not cpu else models.BertConfig(vocab_size=500, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128)
    if cpu:
        seq = min(seq, 32)
    torch.manual_seed(4321)
    model = models.BertForQuestionAnswering(cfgm).to(dev).to(dtype)
    cfg = {}
    finish = None
    if args.impl == "ddp":
        if world > 1:
            model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[c.local_rank], gradient_as_bucket_view=True)
        optimizer = torch.optim.AdamW(model.parameters(), lr=3e-5, weight_decay=0.01)
        cfg["optimizer"] = "torch.optim.AdamW on bf16 parameters"
        cfg["allreduce_variants"] = ["torch DDP (NCCL, uncompressed bf16)"]
        algo = "none (plain DDP all-reduce; stock PyTorch has no ByteGrad)"
    else:
        from bagua_b200.ops.optim import FusedAdam
        from bagua_b200.parallel.algorithms import bytegrad

        optimizer = FusedAdam(model.parameters(), lr=3e-5, adamw=True, weight_decay=0.01) if not cpu else torch.optim.AdamW(model.parameters(), lr=3e-5)
        model = model.with_bagua([optimizer], bytegrad.ByteGradAlgorithm())
        cfg["optimizer"] = "FusedAdam(adamw, fp32 master weights + moments), one flat kernel per step"
        cfg["allreduce_variants"] = sorted({getattr(b, "allreduce_variant", "none") for b in model.bagua_buckets})
        cfg["buckets"] = len(model.bagua_buckets)
        cfg["bucket_programs"] = _bucket_programs(model)
        finish = model.bagua_ddp.wait_pending_comm_ops
        algo = "ByteGrad (MinMaxUInt8)"

    torch.manual_seed(99 + c.rank)

    def make(device, pinned=False):
        t = (torch.randint(0, cfgm.vocab_size, (bs, seq)), torch.randint(0, 2, (bs, seq)), torch.ones(bs, seq, dtype=torch.int64),
             torch.randint(0, seq, (bs,)), torch.randint(0, seq, (bs,)))
        if pinned and not cpu:
            return tuple(x.pin_memory() for x in t)
        return tuple(x.to(device) for x in t)

    dev_batch = make(dev)
    n_host = 4
    host = [make("cpu", pinned=True) for _ in range(n_host)]

    def train_step(ids, tt, mask, sp, ep):
        optimizer.zero_grad()
        loss = model(ids, token_type_ids=tt, attention_mask=mask, start_positions=sp, end_positions=ep)[0]
        loss.backward()
        optimizer.step()
        return loss

    def host_batches(n):
        for i in range(n):
            yield host[i % n_host]

    res = measure(c, "bert", train_step, dev_batch, host_batches, None, bs, "samples/s", finish, params=model.parameters)
    if args.impl != "ddp":
        res["comm_timeline"] = timeline_probe(c, model, train_step, dev_batch, finish)
    res["metric"] = f"BERT-large SQuAD-shaped fine-tuning throughput ({algo})"
    res["config"] = dict(cfg, model="bert-large (24 layers, hidden 1024, 16 heads, 335 M parameters) + QA head" if not cpu else "tiny bert (selftest)",
                         global_batch=bs * world, per_gpu_batch=bs, seq_len=seq, parallelism=f"dp{world}", algorithm=algo,
                         reference_config="examples/squad/README.md:19-28 (seq 384, bs 6/GPU, lr 3e-5)",
                         l2_policy="670 MB of bf16 weights + 4 GB of optimizer state per step far exceed the 50 MB L2 of an H100; no explicit flush")
    del model, optimizer
    return res


def main():
    args = parse()
    if args.impl == "reference":
        return reference_arm(args)

    # Only the final JSON line may reach stdout: libraries (e.g. NCCL's "NCCL version ..." banner) print there too, so fd 1
    # is pointed at stderr for the duration of the run and restored just before the result is printed.
    sys.stdout.flush()
    saved_stdout_fd = os.dup(1)
    os.dup2(2, 1)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus and world == 1 and args.gpus > 1:
        raise SystemExit(f"--gpus {args.gpus} needs a torchrun launch with {args.gpus} ranks")
    if args.impl == "nccl_baseline":
        os.environ["BAGUA_ALLREDUCE_VARIANT"] = "nccl"      # no peer engine: every bucket op is torch.distributed on the comm stream
    elif args.impl == "ours" and world == 1 and not args.no_self_peer and not args.selftest_cpu:
        os.environ.setdefault("BAGUA_SELF_PEER", "1")       # N = 1 runs the same bucket kernels with this GPU as the only peer
    sys.path.insert(0, REPO)
    if "MASTER_PORT" not in os.environ:
        from bagua_b200.env import find_free_network_port

        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(find_free_network_port())
    os.environ.setdefault("LOCAL_WORLD_SIZE", str(world))
    if args.dump_outputs:   # deterministic mode (below) needs cuBLAS's fixed workspace split, set before its first handle exists
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    # A benchmark run should fail in minutes, not hang: in-kernel cross-GPU spins and the scheduler watchdog give up earlier than the
    # training defaults (300 s); both are fatal and reported, and the line below still carries the workloads that completed.
    os.environ.setdefault("BAGUA_PEER_TIMEOUT_S", "120")
    os.environ.setdefault("BAGUA_COMM_TIMEOUT_S", "150")

    c = make_ctx(args)
    c.dumps = {}
    torch = c.torch
    c.sampler = ClockSampler(c.local_rank).start() if (c.rank == 0 and not c.cpu) else None
    if args.impl == "ddp":
        if world > 1:
            c.dist.init_process_group("nccl" if not c.cpu else "gloo")
    else:
        import bagua_b200 as bagua

        bagua.init_process_group()
    # --dump-outputs: deterministic mode, so that two runs or two builds dump the same bits. Without it the outputs drift apart far
    # beyond rounding within the run's ~30 steps (float atomics and timing-based cuDNN algorithm choice in VGG16's backward; the
    # attention backward, amplified by the 8-bit ByteGrad exchange and Adam, in BERT). It is slower, so such a run is not a
    # throughput run; without the flag the benchmark measures the configuration a user runs.
    torch.backends.cudnn.benchmark = not args.dump_outputs
    torch.utils.deterministic.fill_uninitialized_memory = False   # deterministic mode's NaN fill of new memory: work, no reproducibility

    results = {}
    workloads = [w.strip() for w in args.workloads.split(",") if w.strip()]
    head_name = "vgg16" if "vgg16" in workloads else workloads[0]
    for wl in workloads:
        if wl not in ("vgg16", "resnet50", "bert"):
            raise SystemExit(f"unknown workload {wl}")
        # strict for BERT (its attention backward is deterministic only then); warn-only for the CNNs, whose adaptive average pool
        # (an identity at 224², one addend per element) has no deterministic backward and would raise
        torch.use_deterministic_algorithms(bool(args.dump_outputs), warn_only=wl != "bert")
        try:
            results[wl] = run_bert(c) if wl == "bert" else run_cnn(c, wl)
            if not c.cpu:
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
            c.sync_all()
        except Exception as e:  # noqa: BLE001 - a failing secondary workload must not take the headline measurement with it
            if wl == head_name or head_name not in results:
                raise
            import traceback

            traceback.print_exc(file=sys.stderr)
            results[wl] = {"error": f"{type(e).__name__}: {e}"[:600]}

    if c.rank == 0 and args.dump_outputs:
        import numpy as np

        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in c.dumps.items():
            np.save(os.path.join(args.dump_outputs, f"{k}.npy"), v.astype(np.float32))
    if c.rank == 0:
        first = next(iter(results))
        head = results.get("vgg16", results[first])
        out = {
            "metric": head["metric"], "value": head["value"], "unit": head["unit"], "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": head["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16" if not c.cpu else "fp32", "data": "synthetic (random batches of the named shapes, random-init weights)", "impl": args.impl,
            "config": head["config"], "clocks": head["clocks"], "e2e": head["e2e"], "gpu_launches": head["gpu_launches"],
            "host_issue_ms_per_step": head.get("host_issue_ms_per_step"),
            "published_context": PUBLISHED_CONTEXT,
        }
        if "verify" in head:
            out["verify"] = head["verify"]
        if "comm_timeline" in head:
            out["comm_timeline"] = head["comm_timeline"]
        if "bert" in results and "error" in results["bert"]:
            out["bert_large_bytegrad"] = {"value": None, "error": results["bert"]["error"]}
        elif "bert" in results and head is not results["bert"]:
            b = results["bert"]
            out["bert_large_bytegrad"] = {k: b[k] for k in ("metric", "value", "unit", "ms_per_step", "config", "clocks", "e2e", "gpu_launches", "final_loss", "host_issue_ms_per_step", "comm_timeline") if k in b}
            out["bert_large_bytegrad"].update(n_gpus=world, steps=args.steps, warmup=max(args.warmup, 3), higher_is_better=True, scaling="weak", dtype=out["dtype"])
        for k, v in results.items():
            if v is not head and k != "bert":
                out[k] = v
        out["config"]["self_peer_n1"] = os.environ.get("BAGUA_SELF_PEER", "0") == "1"
        if c.cpu:
            out["selftest"] = "host plumbing check, not a benchmark result"
        if c.sampler is not None:
            c.sampler.stop()
        sys.stdout.flush()
        os.dup2(saved_stdout_fd, 1)
        print(json.dumps(out), flush=True)
        os.dup2(2, 1)
    if world > 1 and not any("error" in v for v in results.values()):
        c.dist.barrier()
    return 0


if __name__ == "__main__":
    sys.exit(main())
