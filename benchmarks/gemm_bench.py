"""wgmma grouped GEMM vs cuBLAS (torch.bmm) on MoE expert shapes; CUDA-event timing after warm-up, L2 flushed between calls."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bagua_b200.ops.gemm import grouped_gemm_tn  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--out", default="")
args = p.parse_args()
dev = torch.device("cuda", 0)
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
rows = []
for (G, M, N, K) in [(1, 8192, 4096, 1024), (1, 8192, 1024, 4096), (2, 8192, 4096, 1024), (4, 4096, 4096, 1024), (1, 8192, 8192, 8192)]:
    a = torch.randn(G, M, K, device=dev).to(torch.bfloat16)
    b = torch.randn(G, N, K, device=dev).to(torch.bfloat16)
    bias = torch.randn(G, N, device=dev).to(torch.bfloat16)

    def bench(fn, iters=10):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(iters):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e))
        return sorted(ts)[len(ts) // 2]

    flops = 2.0 * G * M * N * K
    t_ours = bench(lambda: grouped_gemm_tn(a, b, bias))
    t_cublas = bench(lambda: torch.baddbmm(bias.unsqueeze(1), a, b.transpose(1, 2)))
    rows.append({"G": G, "M": M, "N": N, "K": K, "wgmma_ms": t_ours, "wgmma_tflops": flops / t_ours / 1e9, "cublas_ms": t_cublas,
                 "cublas_tflops": flops / t_cublas / 1e9})
    print(rows[-1])
if args.out:
    json.dump(rows, open(args.out, "w"), indent=1)
