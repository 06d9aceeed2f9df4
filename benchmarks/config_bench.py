"""Benchmarks of the other BASELINE.json configurations (one JSON line per run, device-timed, max over ranks):

  bert_bytegrad           BERT-large, SQuAD-shaped synthetic batches (seq 384), ByteGrad
  resnet50_decentralized  ResNet-50, DecentralizedAlgorithm(peer_selection_mode=all)
  resnet50_async          ResNet-50, AsyncModelAverageAlgorithm
  gpt2_moe                GPT-2 medium MoE-8, expert all-to-all (peer dispatch/combine + wgmma expert GEMMs)

``BAGUA_ALLREDUCE_VARIANT=nccl BAGUA_MOE_PEER=0`` runs the same schedule on NCCL/cuBLAS only (the baseline arm)."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

p = argparse.ArgumentParser()
p.add_argument("--config", required=True)
p.add_argument("--steps", type=int, default=15)
p.add_argument("--warmup", type=int, default=5)
p.add_argument("--batch-size", type=int, default=0)
p.add_argument("--tiny", action="store_true", help="shrunken models for CPU smoke tests")
p.add_argument("--cpu", action="store_true")
p.add_argument("--force-bf16", action="store_true", help="bf16 parameters even on the CPU smoke path (exercises the same python code as the GPU run)")
p.add_argument("--comm-report", action="store_true", help="per-bucket device time / GB/s of the communication programs (adds 2 event records per bucket)")
p.add_argument("--arm", choices=["peer", "nccl"], default="peer", help="nccl = same schedule on NCCL collectives / cuBLAS experts only (baseline arm)")
args = p.parse_args()
if os.environ.get("WORLD_SIZE", "1") == "1" and args.arm == "peer" and not args.cpu:
    os.environ.setdefault("BAGUA_SELF_PEER", "1")   # one GPU: same kernels with this GPU as the only peer (see bench.py)
if args.arm == "nccl":
    os.environ["BAGUA_ALLREDUCE_VARIANT"] = "nccl"
    os.environ["BAGUA_MOE_PEER"] = "0"
    os.environ["BAGUA_DISABLE_GROUPED_GEMM"] = "1"

import bagua_b200 as bagua  # noqa: E402
from bagua_b200 import models  # noqa: E402
from bagua_b200.ops.optim import FusedAdam  # noqa: E402
from bagua_b200.parallel.algorithms import async_model_average, bytegrad, decentralized, gradient_allreduce  # noqa: E402

cuda = torch.cuda.is_available() and not args.cpu
if cuda:
    torch.cuda.set_device(bagua.get_local_rank())
if "MASTER_PORT" not in os.environ:
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(bagua.env.find_free_network_port())
bagua.init_process_group()
rank, world = bagua.get_rank(), bagua.get_world_size()
dev = torch.device("cuda", bagua.get_local_rank()) if cuda else torch.device("cpu")
dtype = torch.bfloat16 if (cuda or args.force_bf16) else torch.float32
torch.manual_seed(1 + rank)
torch.backends.cudnn.benchmark = True
cfg = args.config

if cfg == "bert_bytegrad":
    c = models.bert_large_config() if not args.tiny else models.BertConfig(vocab_size=500, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128)
    bs, seq = args.batch_size or 8, 384 if not args.tiny else 32
    model = models.BertForQuestionAnswering(c).to(dev).to(dtype)
    opt = FusedAdam(model.parameters(), lr=3e-5, adamw=True, weight_decay=0.01) if cuda else torch.optim.AdamW(model.parameters(), lr=3e-5)
    model = model.with_bagua([opt], bytegrad.ByteGradAlgorithm())
    ids = torch.randint(0, c.vocab_size, (bs, seq), device=dev)
    sp, ep = torch.randint(0, seq, (bs,), device=dev), torch.randint(0, seq, (bs,), device=dev)
    unit, per_step = "samples/s", bs

    def step():
        opt.zero_grad()
        loss = model(ids, start_positions=sp, end_positions=ep)[0]
        loss.backward()
        opt.step()
        return loss

elif cfg in ("resnet50_decentralized", "resnet50_async"):
    bs = args.batch_size or 32
    res = 224 if not args.tiny else 32
    model = models.resnet50(num_classes=1000 if not args.tiny else 10).to(dev).to(dtype)
    if cuda:
        model = model.to(memory_format=torch.channels_last)
    # --tiny (CPU smoke test): batch 2 on 32x32 inputs leaves BatchNorm with degenerate statistics, the benchmark learning rate blows the
    # bf16 loss up to 1e6 and now and then past the finite range — the smoke test is about wiring, so it steps gently
    opt = torch.optim.SGD(model.parameters(), lr=0.01 * world if not args.tiny else 1e-4, momentum=0.9)
    algo = decentralized.DecentralizedAlgorithm(peer_selection_mode="all") if cfg == "resnet50_decentralized" else async_model_average.AsyncModelAverageAlgorithm(sync_interval_ms=100)
    model = model.with_bagua([opt], algo)
    x = torch.randn(bs, 3, res, res, device=dev).to(dtype)
    if cuda:
        x = x.contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (bs,), device=dev)
    unit, per_step = "images/s", bs

    def step():
        opt.zero_grad()
        loss = F.cross_entropy(model(x).float(), y)
        loss.backward()
        opt.step()
        return loss

elif cfg == "gpt2_moe":
    c = models.gpt2_medium_moe8_config() if not args.tiny else models.GPT2MoEConfig(vocab_size=512, n_positions=64, n_embd=64, n_layer=2, n_head=4, num_experts=world * 2)
    bs, seq = args.batch_size or 8, 1024 if not args.tiny else 64
    model = models.GPT2MoE(c, world_size=world).to(dev).to(dtype)
    opt = FusedAdam(model.parameters(), lr=1e-4, adamw=True) if cuda else torch.optim.AdamW(model.parameters(), lr=1e-4)
    model = model.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
    idx = torch.randint(0, c.vocab_size, (bs, seq), device=dev)
    tgt = torch.randint(0, c.vocab_size, (bs, seq), device=dev)
    unit, per_step = "tokens/s", bs * seq

    def step():
        opt.zero_grad()
        loss, _ = model(idx, tgt)
        loss.backward()
        opt.step()
        return loss

else:
    raise SystemExit(f"unknown config {cfg}")


def sync():
    if world > 1:
        dist.barrier()
    if cuda:
        torch.cuda.synchronize()


sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler  # noqa: E402

sampler = ClockSampler(bagua.get_local_rank()).start() if (cuda and rank == 0) else None
for _ in range(max(args.warmup, 3)):
    loss = step()
sync()
if args.comm_report:
    model.bagua_ddp.comm_profile(True)
t_begin = ClockSampler.now()
if cuda:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(args.steps):
        loss = step()
    e.record()
    torch.cuda.synchronize()
    ms = torch.tensor([s.elapsed_time(e)], device=dev)
else:
    import time

    t0 = time.time()
    for _ in range(args.steps):
        loss = step()
    ms = torch.tensor([(time.time() - t0) * 1e3])
t_end = ClockSampler.now()
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
if cfg == "resnet50_async":
    model.bagua_algorithm.abort(model)
finite = bool(torch.isfinite(loss.detach().float()).item())
if args.comm_report and rank == 0:
    if cuda:
        torch.cuda.synchronize()
    for r in model.bagua_ddp.comm_report():
        print("[comm]", json.dumps(r), file=sys.stderr)
if rank == 0:
    print(json.dumps({
        "config": cfg, "arm": args.arm, "moe_fused_combine": os.environ.get("BAGUA_MOE_FUSED_COMBINE", "0"), "n_gpus": world, "value": per_step * world * args.steps / (ms.item() / 1e3), "unit": unit, "ms_per_step": ms.item() / args.steps,
        "per_gpu_batch": bs, "dtype": str(dtype), "loss_finite": finite,
        "arm": "nccl-only" if os.environ.get("BAGUA_ALLREDUCE_VARIANT") == "nccl" else "peer-kernels",
        "moe_peer": os.environ.get("BAGUA_MOE_PEER", "1"), "steps": args.steps, "warmup": max(args.warmup, 3),
        "clocks": sampler.stop(t_begin, t_end) if sampler is not None else None, "final_loss": float(loss.detach().float().item()),
        "timing": "CUDA events around the K steps on the launching stream, max over ranks; synthetic data, random-init weights",
    }))
if world > 1:
    dist.barrier()
