"""What LARS costs on the sharded in-bucket optimizer path, against momentum SGD on the same path.

ResNet-50 (bf16, channels_last, batch 32, 224×224), one GPU in self-peer mode (the bucket kernels run with this GPU as its only
peer), four arms built once and timed in alternating rounds:

  a  ``make_sharded_fused_sgd(momentum=0.9)``                      update inside the bucket kernels, overlapped with backward
  b  ``make_sharded_fused_sgd(momentum=0.9, max_grad_norm=1e9)``   the two-phase program of LARS: norm exchange + update in step()
  c  ``make_sharded_fused_lars()``                                 norms, per-parameter exchange, update in step()
  d  ``GradientAllReduceAlgorithm`` + ``FusedLARS``                 all-reduce in the buckets, two multi-tensor kernels per step

(a–c with ``FusedGradientAllReduceAlgorithm``; BatchNorm and bias parameters in a ``weight_decay=0`` group in every arm.)

Prints one JSON object: device-timed milliseconds per step (CUDA events around ``--steps`` steps; median, min and max over
``--rounds``), native kernel launches per step, and the card's name and power limit read in the same run.  Writes ``--out`` when
given.

    python scripts/lars_overhead.py --steps 20 --rounds 6 --out results/lars_overhead.json
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = "abcd"
LEGEND = {"a": "sharded in-bucket SGD, momentum 0.9 (update during backward)",
          "b": "sharded in-bucket SGD, momentum 0.9, max_grad_norm (update in step())",
          "c": "sharded in-bucket LARS (norms, exchange, update in step())",
          "d": "GradientAllReduceAlgorithm + FusedLARS"}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=6)
    p.add_argument("--batch-size", type=int, default=32)
    p.add_argument("--image-size", type=int, default=224)
    p.add_argument("--out", default="")
    args = p.parse_args()

    os.environ.setdefault("BAGUA_SELF_PEER", "1")
    os.environ.setdefault("RANK", "0")
    os.environ.setdefault("WORLD_SIZE", "1")
    os.environ.setdefault("LOCAL_RANK", "0")
    os.environ.setdefault("LOCAL_WORLD_SIZE", "1")
    sys.path.insert(0, REPO)
    import torch
    import torch.nn.functional as F

    if not torch.cuda.is_available():
        raise SystemExit("lars_overhead.py measures on a GPU; none is visible")
    from bagua_b200.env import find_free_network_port

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(find_free_network_port()))
    import bagua_b200 as bagua
    from bagua_b200 import models
    from bagua_b200.core import native
    from bagua_b200.ops.optim import FusedLARS
    from bagua_b200.parallel.algorithms.gradient_allreduce import (FusedGradientAllReduceAlgorithm, GradientAllReduceAlgorithm, make_sharded_fused_lars,
                                                                   make_sharded_fused_sgd)

    bagua.init_process_group()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bs, hw = args.batch_size, args.image_size

    def build(arm):
        torch.manual_seed(4321)
        model = models.resnet50(num_classes=1000).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
        groups = [{"params": [p for p in model.parameters() if p.dim() > 1], "weight_decay": 5e-5},
                  {"params": [p for p in model.parameters() if p.dim() <= 1], "weight_decay": 0.0}]
        if arm in "ab":
            opt = make_sharded_fused_sgd(groups, lr=0.1, momentum=0.9, max_grad_norm=1e9 if arm == "b" else None)
        elif arm == "c":
            opt = make_sharded_fused_lars(groups, lr=0.1, momentum=0.9)
        else:
            opt = FusedLARS(groups, lr=0.1, momentum=0.9)
            return model.with_bagua([opt], GradientAllReduceAlgorithm()), opt
        return model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt)), opt

    torch.manual_seed(99)
    x = torch.randn(bs, 3, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (bs,), device=dev)

    arms = {}
    for arm in ARMS:
        model, opt = build(arm)

        def step(model=model, opt=opt):
            opt.zero_grad()
            F.cross_entropy(model(x).float(), y).backward()
            opt.step()

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        arms[arm] = {"step": step, "model": model, "ms": [], "variants": sorted({b.allreduce_variant for b in model.bagua_buckets})}

    C = native()
    for arm in ARMS:   # launches per step: the library's own kernel counter over one step
        n0 = C.launch_count()
        arms[arm]["step"]()
        torch.cuda.synchronize()
        arms[arm]["launches_per_step"] = C.launch_count() - n0

    for _ in range(args.rounds):
        for arm in ARMS:
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            for _ in range(args.steps):
                arms[arm]["step"]()
            end.record()
            torch.cuda.synchronize()
            arms[arm]["ms"].append(start.elapsed_time(end) / args.steps)

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi,
           "workload": f"ResNet-50 bf16 channels_last batch {bs} {hw}x{hw}, self-peer world 1", "steps_per_round": args.steps, "rounds": args.rounds,
           "arms": {k: {"median_ms_per_step": round(sorted(v["ms"])[len(v["ms"]) // 2], 3), "min_ms_per_step": round(min(v["ms"]), 3),
                        "max_ms_per_step": round(max(v["ms"]), 3), "ms_per_step_rounds": [round(t, 3) for t in v["ms"]],
                        "native_launches_per_step": v["launches_per_step"], "bucket_variants": v["variants"]} for k, v in arms.items()},
           "legend": LEGEND}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
