"""What gradient accumulation in the fp32 shard costs against local accumulation under ``no_sync()``.

BERT-large in bf16 at ``bench.py``'s shape (seq 384, batch 6), one GPU in self-peer mode (the bucket kernels run with this GPU as
its only peer), K = 4 micro-batches per optimizer step, two arms built once and timed in alternating rounds:

  a  ``make_sharded_fused_adam(max_grad_norm=1.0)``: micro-batches 1 … K−1 under ``require_backward_grad_sync = False`` add up in
     the bf16 bucket, the last one communicates                                           one reduce-scatter per step
  b  the same with ``accumulate_grads=True``: every micro-batch communicates and adds its reduced gradient into the fp32 shard
                                                                                          K reduce-scatters per step

Prints one JSON object: device-timed milliseconds per optimizer step (CUDA events around ``--steps`` steps; median, minimum and
maximum over ``--rounds``), native kernel launches per step, the card's name and power limit, and — from ``torch.profiler`` in a
separate process — the device time of one ``shard_grad_kernel`` launch with and without ``ACCUM`` on a bucket the size of
BERT-large's gradient (a virtual world of one rank). Writes ``--out`` when given.

    python scripts/accumulation_overhead.py --steps 10 --rounds 5 --out results/accumulation_overhead.json
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 4


def kernel_profile(numel, launches):
    """Device time per launch of shard_grad_kernel<bf16, 1, ld/st, ACCUM> for ACCUM = false / true, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    sys.path.insert(0, REPO)
    from bagua_b200.core import dtype_code, native
    from bagua_b200.parallel.virtual import VirtualPeerWorld

    C = native()
    w = VirtualPeerWorld(1, torch.device("cuda", 0), timeout_s=60.0)
    nbytes = numel * 2
    grads = w.alloc(nbytes)
    shard = torch.zeros(numel, device=w.device)
    partials = torch.zeros(C.MAX_COMM_BLOCKS, dtype=torch.float64, device=w.device)
    ops = {acc: C.ShardGradOp(w.comms[0], grads.buf, 0, nbytes, dtype_code(torch.bfloat16), shard.data_ptr(), partials.data_ptr(), 1.0, True, False,
                              w.cfg(64), acc) for acc in (False, True)}

    def run(acc):
        grads.view(0, torch.bfloat16, numel).normal_()
        w.run(None, ops=[ops[acc]])

    for acc in (False, True):   # an accumulating op overwrites on its first run: warm up past it
        run(acc)
        run(acc)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            run(False)
            run(True)
        torch.cuda.synchronize()
    times = {"false": [], "true": []}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and "shard_grad_kernel" in ev.name:
            args = ev.name.split("<", 1)[1].split(">", 1)[0].replace(" ", "").split(",")
            times[args[-1]].append(ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
    out = {}
    for k, v in times.items():
        v = sorted(v)
        out[f"accum_{k}"] = {"launches": len(v), "median_us": v[len(v) // 2] if v else None,
                             "GB_per_s_median": (nbytes + numel * 4 * (2 if k == "true" else 1)) / (v[len(v) // 2] * 1e3) if v else None}
    out["numel"], out["bytes_moved_note"] = numel, "bucket read + shard write (+ shard read with ACCUM); the bucket clear is not counted"
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--batch-size", type=int, default=6)
    p.add_argument("--seq-len", type=int, default=384)
    p.add_argument("--kernel-numel", type=int, default=335_141_888, help="elements of the profiled bucket (BERT-large's gradient)")
    p.add_argument("--kernel-launches", type=int, default=20)
    p.add_argument("--kernel-profile", action="store_true", help=argparse.SUPPRESS)
    p.add_argument("--out", default="")
    args = p.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("accumulation_overhead.py measures on a GPU; none is visible")
    if args.kernel_profile:
        print(json.dumps(kernel_profile(args.kernel_numel, args.kernel_launches)))
        return

    os.environ.setdefault("BAGUA_SELF_PEER", "1")
    os.environ.setdefault("RANK", "0")
    os.environ.setdefault("WORLD_SIZE", "1")
    os.environ.setdefault("LOCAL_RANK", "0")
    os.environ.setdefault("LOCAL_WORLD_SIZE", "1")
    sys.path.insert(0, REPO)
    from bagua_b200.env import find_free_network_port

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(find_free_network_port()))
    import bagua_b200 as bagua
    from bagua_b200 import models
    from bagua_b200.core import native
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam

    bagua.init_process_group()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bs, seq = args.batch_size, args.seq_len
    cfg = models.bert_large_config()

    def build(arm):
        torch.manual_seed(4321)
        model = models.BertForQuestionAnswering(cfg).to(dev).to(torch.bfloat16)
        opt = make_sharded_fused_adam(model.parameters(), lr=3e-5, adamw=True, weight_decay=0.01, max_grad_norm=1.0, accumulate_grads=arm == "b")
        return model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt)), opt

    torch.manual_seed(99)
    batch = (torch.randint(0, cfg.vocab_size, (bs, seq), device=dev), torch.randint(0, 2, (bs, seq), device=dev),
             torch.ones(bs, seq, dtype=torch.int64, device=dev), torch.randint(0, seq, (bs,), device=dev), torch.randint(0, seq, (bs,), device=dev))

    arms = {}
    for arm in "ab":
        model, opt = build(arm)

        def step(model=model, opt=opt, arm=arm):
            opt.zero_grad()
            ids, tt, mask, sp, ep = batch
            for k in range(K):
                model.bagua_ddp.require_backward_grad_sync = arm == "b" or k == K - 1
                loss = model(ids, token_type_ids=tt, attention_mask=mask, start_positions=sp, end_positions=ep)[0] / K
                loss.backward()
            opt.step()

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        arms[arm] = {"step": step, "ms": [], "variants": sorted({b.allreduce_variant for b in model.bagua_buckets})}

    C = native()
    for arm in "ab":   # launches per optimizer step: the library's own kernel counter over one step of K micro-batches
        n0 = C.launch_count()
        arms[arm]["step"]()
        torch.cuda.synchronize()
        arms[arm]["launches_per_step"] = C.launch_count() - n0

    for _ in range(args.rounds):
        for arm in "ab":
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            for _ in range(args.steps):
                arms[arm]["step"]()
            end.record()
            torch.cuda.synchronize()
            arms[arm]["ms"].append(start.elapsed_time(end) / args.steps)
    del arms["a"]["step"], arms["b"]["step"]

    prof = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-profile", "--kernel-numel", str(args.kernel_numel),
                           "--kernel-launches", str(args.kernel_launches)], capture_output=True, text=True, cwd=REPO)
    kernel = json.loads(prof.stdout.strip().splitlines()[-1]) if prof.returncode == 0 and prof.stdout.strip() else {"error": prof.stderr[-2000:]}

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "workload": f"BERT-large bf16 seq {seq} batch {bs}, self-peer world 1, "
           f"{K} micro-batches per optimizer step", "steps_per_round": args.steps, "rounds": args.rounds,
           "arms": {k: {"median_ms_per_step": sorted(v["ms"])[len(v["ms"]) // 2], "min_ms_per_step": min(v["ms"]), "max_ms_per_step": max(v["ms"]),
                        "ms_per_step_rounds": [round(x, 3) for x in v["ms"]],
                        "native_launches_per_step": v["launches_per_step"], "bucket_variants": v["variants"]} for k, v in arms.items()},
           "shard_grad_kernel": kernel,
           "legend": {"a": "sharded in-bucket AdamW, max_grad_norm=1.0, micro-batches 1..K-1 under no_sync (bf16 local accumulation)",
                      "b": "sharded in-bucket AdamW, max_grad_norm=1.0, accumulate_grads=True (every micro-batch reduce-scatters into the fp32 shard)"}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
