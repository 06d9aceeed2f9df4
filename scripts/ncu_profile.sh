#!/usr/bin/env bash
# ncu captures of the top kernels (run under gpurun on ONE GPU; never wrap a multi-rank command in ncu).
#   gpurun --timeout 900 -- 'bash scripts/ncu_profile.sh'
# Reports land in gpurun_out/*.ncu-rep; summarise them offline (no GPU needed) into the tracked profiles/ directory with
#   python scripts/ncu_summary.py gpurun_out/ncu_*.ncu-rep --launches gpurun_out/launches_step.csv > profiles/ncu_summary.md
# or read single metrics with
#   ncu -i gpurun_out/<name>.ncu-rep --page raw --csv | grep -E 'dram__bytes_(read|write).sum|gpu__dram_throughput|sm__pipe_tensor_cycles_active|launch__registers_per_thread'
set -euo pipefail
mkdir -p gpurun_out
NCU="ncu --set full --clock-control none --import-source on"
# 1. fused optimizer + NHWC epilogues inside the flagship step
$NCU -k regex:flat_sgd_kernel -s 3 -c 1 -o gpurun_out/ncu_flat_sgd python bench.py --steps 2 --warmup 3 --no-e2e > gpurun_out/ncu_flat_sgd.log 2>&1 || true
$NCU -k regex:bias_relu_bwd_kernel -s 8 -c 1 -o gpurun_out/ncu_bias_relu_bwd python bench.py --steps 2 --warmup 3 --no-e2e > gpurun_out/ncu_bias_relu_bwd.log 2>&1 || true
# 2. wgmma grouped GEMM
$NCU -k regex:grouped_gemm_tn_kernel -s 3 -c 1 -o gpurun_out/ncu_gemm python benchmarks/gemm_bench.py > gpurun_out/ncu_gemm.log 2>&1 || true
# 3. every launch of one flagship step with its device time
ncu --metrics gpu__time_duration.sum --clock-control none -s 3000 -c 400 --csv --log-file gpurun_out/launches_step.csv python bench.py --steps 2 --warmup 3 --no-e2e > gpurun_out/launches_step.log 2>&1 || true
