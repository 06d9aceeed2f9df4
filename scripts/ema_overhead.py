"""What the sharded weight EMA (``ema_decay``) of the in-bucket optimizers costs per optimizer step.

One GPU in self-peer mode (the bucket kernels run with this GPU as its only peer), every arm built once and timed in alternating
rounds:

  a  BERT-large bf16 (seq 384, batch 6), ``make_sharded_fused_adam(adamw=True)``
  b  the same with ``ema_decay=0.9999``                    one EMA launch per step over every bucket's shard
  c  the same with ``ema_decay=0.9999, ema_every=4``       one EMA launch every fourth step
  d  ResNet-50 bf16 channels_last (224², batch 64), ``make_sharded_fused_sgd(momentum=0.9)``
  e  the same with ``ema_decay=0.9999``

Prints one JSON object: device-timed milliseconds per optimizer step (CUDA events around ``--steps`` steps; median, minimum and
maximum over ``--rounds``), native kernel launches per step (over ``4`` steps, divided by 4), the card's name and power limit.

    python scripts/ema_overhead.py --steps 10 --rounds 5 --out results/ema_overhead.json
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=8)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--out", default="")
    args = p.parse_args()

    import torch
    import torch.nn.functional as F

    if not torch.cuda.is_available():
        raise SystemExit("ema_overhead.py measures on a GPU; none is visible")
    os.environ.setdefault("BAGUA_SELF_PEER", "1")
    for k, v in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0"), ("LOCAL_WORLD_SIZE", "1")):
        os.environ.setdefault(k, v)
    sys.path.insert(0, REPO)
    from bagua_b200.env import find_free_network_port

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(find_free_network_port()))
    import bagua_b200 as bagua
    from bagua_b200 import models
    from bagua_b200.core import native
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_sgd

    bagua.init_process_group()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = models.bert_large_config()
    bs, seq = 6, 384
    torch.manual_seed(99)
    bert_batch = (torch.randint(0, cfg.vocab_size, (bs, seq), device=dev), torch.randint(0, 2, (bs, seq), device=dev),
                  torch.ones(bs, seq, dtype=torch.int64, device=dev), torch.randint(0, seq, (bs,), device=dev), torch.randint(0, seq, (bs,), device=dev))
    img = torch.randn(64, 3, 224, 224, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    lbl = torch.randint(0, 1000, (64,), device=dev)
    ema = {"a": {}, "b": {"ema_decay": 0.9999}, "c": {"ema_decay": 0.9999, "ema_every": 4}, "d": {}, "e": {"ema_decay": 0.9999}}

    def build(arm):
        torch.manual_seed(4321)
        if arm in "abc":
            model = models.BertForQuestionAnswering(cfg).to(dev).to(torch.bfloat16)
            opt = make_sharded_fused_adam(model.parameters(), lr=3e-5, adamw=True, weight_decay=0.01, **ema[arm])
            model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))

            def step():
                opt.zero_grad()
                ids, tt, mask, sp, ep = bert_batch
                model(ids, token_type_ids=tt, attention_mask=mask, start_positions=sp, end_positions=ep)[0].backward()
                opt.step()
        else:
            model = models.resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
            opt = make_sharded_fused_sgd(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4, **ema[arm])
            model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))

            def step():
                opt.zero_grad()
                F.cross_entropy(model(img).float(), lbl).backward()
                opt.step()
        return step

    C = native()
    arms = {}
    for arm in "abcde":
        step = build(arm)
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        n0 = C.launch_count()
        for _ in range(4):
            step()
        torch.cuda.synchronize()
        arms[arm] = {"step": step, "ms": [], "launches_per_step": (C.launch_count() - n0) / 4}
    for _ in range(args.rounds):
        for arm in "abcde":
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            for _ in range(args.steps):
                arms[arm]["step"]()
            end.record()
            torch.cuda.synchronize()
            arms[arm]["ms"].append(start.elapsed_time(end) / args.steps)

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "workload": "self-peer world 1; BERT-large bf16 seq 384 batch 6 (a-c), "
           "ResNet-50 bf16 channels_last 224x224 batch 64 (d-e)", "steps_per_round": args.steps, "rounds": args.rounds,
           "arms": {k: {"median_ms_per_step": sorted(v["ms"])[len(v["ms"]) // 2], "min_ms_per_step": min(v["ms"]), "max_ms_per_step": max(v["ms"]),
                        "ms_per_step_rounds": [round(x, 3) for x in v["ms"]], "native_launches_per_step": v["launches_per_step"]}
                    for k, v in arms.items()},
           "legend": {k: ("in-bucket AdamW, BERT-large" if k in "abc" else "in-bucket SGD, ResNet-50") + (f", {v}" if v else ", no EMA") for k, v in ema.items()}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
