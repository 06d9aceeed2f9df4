"""What Lion costs on the sharded in-bucket optimizer path, against AdamW on the same path.

BERT-large at ``bench.py``'s shape (bf16, seq 384, batch 6), one GPU in self-peer mode (the bucket kernels run with this GPU as
its only peer), four arms built once and timed in alternating rounds:

  a  ``make_sharded_fused_adam(adamw=True)``              AdamW inside the bucket kernels, overlapped with backward
  b  ``make_sharded_fused_lion()``                        Lion inside the bucket kernels, overlapped with backward
  c  ``make_sharded_fused_lion(max_grad_norm=1.0)``       phase A in the buckets, norm exchange + Lion update in step()
  d  ``GradientAllReduceAlgorithm`` + ``FusedLion``        all-reduce in the buckets, one multi-tensor kernel per step

(a–c with ``FusedGradientAllReduceAlgorithm``; biases and LayerNorm parameters in a ``weight_decay=0`` group in every arm.)

Prints one JSON object: device-timed milliseconds per step (CUDA events around ``--steps`` steps; median, min and max over
``--rounds``), native kernel launches per step, per arm the memory its construction and warm-up left allocated (model, buckets,
optimizer state; ``resident_bytes``) and its peak over its timed steps (``peak_bytes``: ``torch.cuda.max_memory_allocated`` minus
the other arms' memory, which does not change while this arm runs), and the card's name and power limit read in the same run.
Writes ``--out`` when given.

    python scripts/lion_overhead.py --steps 20 --rounds 6 --out results/lion_overhead.json
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = "abcd"
LEGEND = {"a": "sharded in-bucket AdamW (update during backward)",
          "b": "sharded in-bucket Lion (update during backward)",
          "c": "sharded in-bucket Lion, max_grad_norm=1.0 (update in step())",
          "d": "GradientAllReduceAlgorithm + FusedLion"}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=6)
    p.add_argument("--batch-size", type=int, default=6)
    p.add_argument("--seq-len", type=int, default=384)
    p.add_argument("--out", default="")
    args = p.parse_args()

    os.environ.setdefault("BAGUA_SELF_PEER", "1")
    os.environ.setdefault("RANK", "0")
    os.environ.setdefault("WORLD_SIZE", "1")
    os.environ.setdefault("LOCAL_RANK", "0")
    os.environ.setdefault("LOCAL_WORLD_SIZE", "1")
    sys.path.insert(0, REPO)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("lion_overhead.py measures on a GPU; none is visible")
    from bagua_b200.env import find_free_network_port

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(find_free_network_port()))
    import bagua_b200 as bagua
    from bagua_b200 import models
    from bagua_b200.core import native
    from bagua_b200.ops.optim import FusedLion
    from bagua_b200.parallel.algorithms.gradient_allreduce import (FusedGradientAllReduceAlgorithm, GradientAllReduceAlgorithm, make_sharded_fused_adam,
                                                                   make_sharded_fused_lion)

    bagua.init_process_group()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bs, seq = args.batch_size, args.seq_len
    cfg = models.bert_large_config()

    def build(arm):
        torch.manual_seed(4321)
        model = models.BertForQuestionAnswering(cfg).to(dev).to(torch.bfloat16)
        nodecay = [n.endswith("bias") or "LayerNorm" in n or "layer_norm" in n for n, _ in model.named_parameters()]
        params = [p for _, p in model.named_parameters()]
        groups = [{"params": [p for p, nd in zip(params, nodecay) if not nd], "weight_decay": 0.1},
                  {"params": [p for p, nd in zip(params, nodecay) if nd], "weight_decay": 0.0}]
        if arm == "a":
            opt = make_sharded_fused_adam(groups, lr=3e-5, adamw=True)
        elif arm in "bc":
            opt = make_sharded_fused_lion(groups, lr=3e-6, max_grad_norm=1.0 if arm == "c" else None)
        else:
            opt = FusedLion(groups, lr=3e-6)
            return model.with_bagua([opt], GradientAllReduceAlgorithm()), opt
        return model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt)), opt

    torch.manual_seed(99)
    batch = (torch.randint(0, cfg.vocab_size, (bs, seq), device=dev), torch.randint(0, 2, (bs, seq), device=dev),
             torch.ones(bs, seq, dtype=torch.int64, device=dev), torch.randint(0, seq, (bs,), device=dev), torch.randint(0, seq, (bs,), device=dev))

    arms = {}
    for arm in ARMS:
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated(dev)
        model, opt = build(arm)

        def step(model=model, opt=opt):
            opt.zero_grad()
            ids, tt, mask, sp, ep = batch
            model(ids, token_type_ids=tt, attention_mask=mask, start_positions=sp, end_positions=ep)[0].backward()
            opt.step()

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        arms[arm] = {"step": step, "model": model, "ms": [], "peak": 0, "resident": torch.cuda.memory_allocated(dev) - before,
                     "variants": sorted({b.allreduce_variant for b in model.bagua_buckets})}

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
            torch.cuda.reset_peak_memory_stats(dev)
            others = torch.cuda.memory_allocated(dev) - arms[arm]["resident"]   # the other arms' memory, unchanged while this arm runs
            start.record()
            for _ in range(args.steps):
                arms[arm]["step"]()
            end.record()
            torch.cuda.synchronize()
            arms[arm]["ms"].append(start.elapsed_time(end) / args.steps)
            arms[arm]["peak"] = max(arms[arm]["peak"], torch.cuda.max_memory_allocated(dev) - others)

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "workload": f"BERT-large bf16 seq {seq} batch {bs}, self-peer world 1",
           "steps_per_round": args.steps, "rounds": args.rounds,
           "arms": {k: {"median_ms_per_step": round(sorted(v["ms"])[len(v["ms"]) // 2], 3), "min_ms_per_step": round(min(v["ms"]), 3),
                        "max_ms_per_step": round(max(v["ms"]), 3), "ms_per_step_rounds": [round(t, 3) for t in v["ms"]],
                        "native_launches_per_step": v["launches_per_step"], "resident_bytes": v["resident"],
                        "peak_bytes": v["peak"], "bucket_variants": v["variants"]} for k, v in arms.items()},
           "legend": LEGEND}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
