#!/usr/bin/env bash
# ncu --set full over one launch of every hand-written kernel (scripts/kernel_zoo.py, world = 1). The .ncu-rep stays on the box when it is
# large (gpurun brings back at most 64 MiB): the raw and details pages are exported to CSV there; profiles/ncu_summary.md is built from them here.
set -uo pipefail
out=${1:-gpurun_out/ncu}
mkdir -p "$out"
K='regex:allreduce_|all_gather_k|reduce_scatter_k|peer_average|bytegrad|lpdec|async_average|flat_sgd|flat_adam|minmax_uint8|bias_relu|moe_|grouped_gemm'
ZOO_NCU=1 timeout 1200 ncu --set full --clock-control none -k "$K" -o /tmp/ncu_zoo -f python scripts/kernel_zoo.py > "$out/ncu_zoo.log" 2>&1
echo "ncu rc=$?" >> "$out/ncu_zoo.log"
ncu -i /tmp/ncu_zoo.ncu-rep --page raw --csv > "$out/ncu_zoo_raw.csv" 2>> "$out/ncu_zoo.log"
ncu -i /tmp/ncu_zoo.ncu-rep --page details --csv > "$out/ncu_zoo_details.csv" 2>> "$out/ncu_zoo.log"
sz=$(stat -c %s /tmp/ncu_zoo.ncu-rep 2>/dev/null || echo 0)
if [ "$sz" -lt 30000000 ] && [ "$sz" -gt 0 ]; then cp /tmp/ncu_zoo.ncu-rep "$out/"; fi
# source-level capture (SASS + source lines, stall reasons) of the three headline kernels only
for k in allreduce_update_kernel bytegrad_kernel grouped_gemm_tn_kernel; do
  ZOO_NCU=1 timeout 600 ncu --set full --clock-control none --import-source on -k "regex:$k" -c 1 -o /tmp/ncu_$k -f python scripts/kernel_zoo.py >> "$out/ncu_zoo.log" 2>&1
  ncu -i /tmp/ncu_$k.ncu-rep --page source --csv > "$out/ncu_${k}_source.csv" 2>> "$out/ncu_zoo.log"
  s2=$(stat -c %s /tmp/ncu_$k.ncu-rep 2>/dev/null || echo 0)
  if [ "$s2" -lt 12000000 ] && [ "$s2" -gt 0 ]; then cp /tmp/ncu_$k.ncu-rep "$out/"; fi
done
ls -la "$out"
