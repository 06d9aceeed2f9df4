"""Microbenchmark of the NVSwitch allreduce kernels against NCCL (torchrun, one rank per GPU).

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 benchmarks/collective_bench.py --out profiles/allreduce_n8.json

Times each call with CUDA events on the launching stream after warm-up, takes the max over ranks, reports algorithm
bandwidth (bytes / time) and bus bandwidth (algbw * 2(N-1)/N) per variant, message size and CTA count."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

p = argparse.ArgumentParser()
p.add_argument("--out", default="")
p.add_argument("--dtype", default="bf16")
p.add_argument("--iters", type=int, default=20)
p.add_argument("--sizes", default="65536,1048576,16777216,134217728,268435456")
p.add_argument("--blocks", default="4,8,16,32,64")
p.add_argument("--rs-ag", action="store_true", help="also time the split reduce-scatter / all-gather kernels (hierarchical path, blocking API) vs NCCL")
args = p.parse_args()

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
import bagua_b200 as bagua  # noqa: E402
from bagua_b200.core import native  # noqa: E402

bagua.init_process_group()
pg = bagua.communication._get_default_group()
eng = pg.peer_engine()
assert eng is not None
C = native()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import ClockSampler  # noqa: E402

sampler = ClockSampler(local).start() if rank == 0 else None
dtype = {"bf16": torch.bfloat16, "f32": torch.float32}[args.dtype]
dev = torch.device("cuda", local)
stream = torch.cuda.current_stream().cuda_stream
results = []


def timeit(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


for nbytes in [int(x) for x in args.sizes.split(",")]:
    numel = nbytes // torch.empty(0, dtype=dtype).element_size()
    sl = eng.alloc(nbytes)
    sl.view(dtype, numel).normal_()
    x = torch.randn(numel, device=dev).to(dtype)
    ms = timeit(lambda: dist.all_reduce(x), args.iters)
    row = {"bytes": nbytes, "variant": "nccl", "blocks": 0, "ms": ms}
    results.append(row)
    variants = (["one_shot"] if nbytes <= 256 * 1024 else []) + ["two_shot"] + (["multimem"] if eng.has_multicast else [])
    for v in variants:
        for nb in [int(b) for b in args.blocks.split(",")]:
            if v == "one_shot" and nb > 8:
                continue
            op, chosen = eng.make_allreduce_op(sl, sl, nbytes, dtype, True, v, blocks=nb)
            ms = timeit(lambda: C.run_op(op, stream, local), args.iters)
            results.append({"bytes": nbytes, "variant": chosen, "blocks": nb, "ms": ms})
    if args.rs_ag and nbytes % (16 * world) == 0:
        from bagua_b200.core import dtype_code

        shard = torch.empty(numel // world, dtype=dtype, device=dev)
        for name, fn in (("nccl_reduce_scatter", lambda: dist.reduce_scatter_tensor(shard, x)), ("nccl_all_gather", lambda: dist.all_gather_into_tensor(x, shard))):
            results.append({"bytes": nbytes, "variant": name, "blocks": 0, "ms": timeit(fn, args.iters), "half": True})
        use_mc = bool(sl.has_multicast and eng.has_multicast)
        for nb in [int(b) for b in args.blocks.split(",")]:
            cfg = eng.launch_cfg("multimem" if use_mc else "two_shot", nbytes, blocks=nb)
            rs = C.ReduceScatterOp(eng.comm, sl.buf, sl.offset, nbytes, dtype_code(dtype), 1.0 / world, use_mc, cfg)
            ag = C.AllGatherOp(eng.comm, sl.buf, sl.offset, nbytes, dtype_code(dtype), use_mc, cfg)
            suffix = "_multimem" if use_mc else "_peer"
            results.append({"bytes": nbytes, "variant": "reduce_scatter" + suffix, "blocks": nb, "ms": timeit(lambda: C.run_op(rs, stream, local), args.iters), "half": True})
            results.append({"bytes": nbytes, "variant": "all_gather" + suffix, "blocks": nb, "ms": timeit(lambda: C.run_op(ag, stream, local), args.iters), "half": True})
    sl.free()

if rank == 0:
    for r in results:
        r["algbw_GBs"] = r["bytes"] / r["ms"] / 1e6
        r["busbw_GBs"] = r["algbw_GBs"] * (1 if r.get("half") else 2) * (world - 1) / world
    print(f"{'bytes':>12} {'variant':>24} {'blocks':>6} {'ms':>9} {'algbw GB/s':>11} {'busbw GB/s':>11}")
    for r in results:
        print(f"{r['bytes']:>12} {r['variant']:>24} {r['blocks']:>6} {r['ms']:>9.4f} {r['algbw_GBs']:>11.1f} {r['busbw_GBs']:>11.1f}")
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"world": world, "dtype": args.dtype, "multicast": eng.has_multicast, "clocks": sampler.stop(),
                       "roofline_note": "an all-reduce moves ~bytes in and ~bytes out of every GPU: the NVLink bound is ALGBW <= 450 GB/s nominal per direction on H100 (NVLink 4); busbw is reported for comparison with nccl-tests only",
                       "results": results}, f, indent=1)
assert eng.comm.error_code() == 0
dist.barrier()
