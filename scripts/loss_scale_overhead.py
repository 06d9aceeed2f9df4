"""What dynamic loss scaling costs on the sharded in-bucket optimizer path.

BERT-large in fp16 at ``bench.py``'s shape (seq 384, batch 6), one GPU in self-peer mode (the bucket kernels run with this GPU as
its only peer), three arms built once and timed in alternating rounds:

  a  ``FusedGradientAllReduceAlgorithm`` + ``make_sharded_fused_adam(max_grad_norm=1.0)``          no loss scaling
  b  the same with ``loss_scaling=True``, driven by ``ShardedGradScaler``                          unscale, vote and skip on the device
  c  ``GradientAllReduceAlgorithm`` + ``FusedAdam`` + ``torch.amp.GradScaler`` + ``clip_grad_norm_``   the path without the sharded optimizer:
     fp32 weights and gradients, fp16 compute under ``torch.autocast`` (torch's scaler refuses fp16 parameters)

Prints one JSON object: device-timed milliseconds per step (CUDA events around ``--steps`` steps; median, minimum and maximum over
``--rounds``), native kernel launches per step, how many of arm b's timed steps were skipped, and the card's name and power limit.
Writes ``--out`` when given.

    python scripts/loss_scale_overhead.py --steps 20 --rounds 5 --out results/loss_scale_overhead.json
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=5)
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
        raise SystemExit("loss_scale_overhead.py measures on a GPU; none is visible")
    from bagua_b200.env import find_free_network_port

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(find_free_network_port()))
    import bagua_b200 as bagua
    from bagua_b200 import models
    from bagua_b200.amp import ShardedGradScaler
    from bagua_b200.core import native
    from bagua_b200.ops.optim import FusedAdam
    from bagua_b200.parallel.algorithms.gradient_allreduce import (FusedGradientAllReduceAlgorithm, GradientAllReduceAlgorithm,
                                                                    make_sharded_fused_adam)

    bagua.init_process_group()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bs, seq = args.batch_size, args.seq_len
    cfg = models.bert_large_config()

    def build(arm):
        torch.manual_seed(4321)
        model = models.BertForQuestionAnswering(cfg).to(dev)
        if arm != "c":
            model = model.to(torch.float16)
        if arm == "c":   # torch's scaler refuses fp16 parameters: fp32 weights, fp16 compute under autocast
            opt = FusedAdam(model.parameters(), lr=3e-5, adamw=True, weight_decay=0.01)
            return model.with_bagua([opt], GradientAllReduceAlgorithm()), opt, torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
        opt = make_sharded_fused_adam(model.parameters(), lr=3e-5, adamw=True, weight_decay=0.01, max_grad_norm=1.0, loss_scaling=arm == "b")
        return model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt)), opt, ShardedGradScaler(init_scale=2.0 ** 12) if arm == "b" else None

    torch.manual_seed(99)
    batch = (torch.randint(0, cfg.vocab_size, (bs, seq), device=dev), torch.randint(0, 2, (bs, seq), device=dev),
             torch.ones(bs, seq, dtype=torch.int64, device=dev), torch.randint(0, seq, (bs,), device=dev), torch.randint(0, seq, (bs,), device=dev))

    arms = {}
    for arm in "abc":
        model, opt, scaler = build(arm)
        skipped = torch.zeros((), device=dev)

        def step(model=model, opt=opt, arm=arm, scaler=scaler, skipped=skipped):
            opt.zero_grad()
            ids, tt, mask, sp, ep = batch
            with torch.autocast("cuda", dtype=torch.float16, enabled=arm == "c"):
                loss = model(ids, token_type_ids=tt, attention_mask=mask, start_positions=sp, end_positions=ep)[0]
            if arm == "a":
                loss.backward()
                opt.step()
                return
            scaler.scale(loss).backward()
            if arm == "c":
                model.bagua_ddp.wait_pending_comm_ops()
                scaler.unscale_(opt)
                opt.clip_grad_norm_(1.0)
            scaler.step(opt)
            if arm == "b":
                skipped.add_(opt.last_step_skipped)   # on the device: no synchronisation in the timed loop
            scaler.update()

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        arms[arm] = {"step": step, "model": model, "ms": [], "skipped": skipped, "variants": sorted({b.allreduce_variant for b in model.bagua_buckets})}

    C = native()
    for arm in "abc":   # launches per step: the library's own kernel counter over one step
        n0 = C.launch_count()
        arms[arm]["step"]()
        torch.cuda.synchronize()
        arms[arm]["launches_per_step"] = C.launch_count() - n0

    arms["b"]["skipped"].zero_()
    for _ in range(args.rounds):
        for arm in "abc":
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            for _ in range(args.steps):
                arms[arm]["step"]()
            end.record()
            torch.cuda.synchronize()
            arms[arm]["ms"].append(start.elapsed_time(end) / args.steps)

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "workload": f"BERT-large fp16 seq {seq} batch {bs}, self-peer world 1",
           "steps_per_round": args.steps, "rounds": args.rounds,
           "skipped_steps_in_b": int(arms["b"]["skipped"].item()),
           "arms": {k: {"median_ms_per_step": sorted(v["ms"])[len(v["ms"]) // 2], "min_ms_per_step": min(v["ms"]), "max_ms_per_step": max(v["ms"]),
                        "ms_per_step_rounds": [round(x, 3) for x in v["ms"]],
                        "native_launches_per_step": v["launches_per_step"], "bucket_variants": v["variants"]} for k, v in arms.items()},
           "legend": {"a": "sharded in-bucket AdamW, max_grad_norm=1.0, no loss scaling",
                      "b": "sharded in-bucket AdamW, max_grad_norm=1.0, loss_scaling=True + ShardedGradScaler",
                      "c": "fp32 weights under torch.autocast(fp16): GradientAllReduceAlgorithm + FusedAdam + torch.amp.GradScaler + clip_grad_norm_(1.0)"}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
