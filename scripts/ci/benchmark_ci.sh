#!/usr/bin/env bash
# CI benchmark gate: the six algorithms on the synthetic benchmark (throughput floor + finite, reproducible final loss) and the MoE
# example with and without a checkpoint round trip — the role of the reference's .buildkite/scripts/benchmark_master.sh:82-151 and
# benchmark.sh:14-37, on ONE node (NVSwitch) through this repo's launchers.
#
#   bash scripts/ci/benchmark_ci.sh [NGPUS]            # GPUs of this node (default: all visible)
#   BAGUA_CI_CPU=1 bash scripts/ci/benchmark_ci.sh 2   # plumbing run on the host (gloo, MNIST-sized model, no floors)
#
# Floors are per-GPU img/s for ResNet-50 bs 32 bf16; they are 0 (throughput unchecked, the final loss still is) until they can be
# derived from a measured H100 run (the reference's floors — 185/180/150/115/190/165 on an unnamed 2019 GPU in fp32 — are kept
# below for context).
set -uo pipefail
cd "$(dirname "$0")/../.."
N=${1:-$(python -c "import torch; print(max(torch.cuda.device_count(), 1))")}
CPU=${BAGUA_CI_CPU:-0}
algorithms=(gradient_allreduce bytegrad decentralized low_precision_decentralized async qadam)
floors=(0 0 0 0 0 0)                           # not measured on H100 yet
ref_floors=(185.0 180.0 150.0 115.0 190 165)    # reference CI (context)
fail=()
port=29610
for i in "${!algorithms[@]}"; do
  a=${algorithms[$i]}
  log=$(mktemp /tmp/bagua_b200_ci_${a}.XXXXXX.log)
  port=$((port + 1))
  if [ "$CPU" = "1" ]; then
    extra="--cpu --model mnist --num-iters 3 --num-batches-per-iter 3 --num-warmup-batches 2 --async-warmup-steps 2"
  else
    extra="--bf16 --num-iters 20"
  fi
  timeout 900 python -m bagua_b200.distributed.launch --nproc_per_node "$N" --master_port $port examples/benchmark/synthetic_benchmark.py \
      --algorithm "$a" --deterministic --async-sync-interval 100 $extra > "$log" 2>&1
  rc=$?
  speed=$(grep "Img/sec per GPU" "$log" | tail -n 1 | awk '{print $4}')
  loss=$(grep "Final loss" "$log" | tail -n 1 | awk '{print $NF}')
  echo "[$a] rc=$rc img/s/GPU=${speed:-?} final_loss=${loss:-?} (floor ${floors[$i]}; reference CI floor ${ref_floors[$i]})"
  [ "$CPU" != "1" ] && [ "${floors[$i]}" = "0" ] && echo "[$a] WARNING: no H100 throughput floor set yet: throughput is NOT checked, only the final loss"
  [ "$rc" -ne 0 ] && fail+=("$a: exit code $rc (log $log)")
  python - "$speed" "$loss" "${floors[$i]}" "$CPU" <<'PY' || fail+=("$a: throughput / loss check failed")
import math, sys
speed, loss, floor, cpu = sys.argv[1:5]
ok = loss not in ("", "?") and math.isfinite(float(loss))
if cpu != "1":
    ok = ok and speed not in ("", "?") and float(speed) >= float(floor)
sys.exit(0 if ok else 1)
PY
done
# MoE example: same final loss with and without a checkpoint save/load in the middle (reference: exact 0.000071 on its CI hardware)
moe_flags="--epochs 2 --num-local-experts 2 --set-deterministic"
[ "$CPU" = "1" ] && moe_flags="$moe_flags --cpu"
for variant in "" "--save-model"; do
  log=$(mktemp /tmp/bagua_b200_ci_moe.XXXXXX.log)
  port=$((port + 1))
  timeout 900 python -m bagua_b200.distributed.launch --nproc_per_node "$N" --master_port $port examples/moe/mnist_main.py --algorithm gradient_allreduce $moe_flags $variant > "$log" 2>&1
  rc=$?
  l=$(grep "Loss" "$log" | tail -n 1 | awk '{print $NF}')
  echo "[moe $variant] rc=$rc final_loss=${l:-?}"
  [ "$rc" -ne 0 ] && fail+=("moe $variant: exit code $rc (log $log)")
  moe_losses+=("${l:-nan}")
done
if [ "${moe_losses[0]}" != "${moe_losses[1]}" ]; then fail+=("moe: final loss differs with checkpointing: ${moe_losses[*]}"); fi
if [ ${#fail[@]} -gt 0 ]; then printf '%s\n' "${fail[@]}"; exit 1; fi
echo "benchmark CI passed"
