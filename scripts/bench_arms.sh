#!/usr/bin/env bash
# The three arms of bench.py on N GPUs of one node, one torchrun each, every command under its own timeout:
#   bash scripts/bench_arms.sh N
set -uo pipefail
N=${1:-1}
out=gpurun_out/arms_n$N
mkdir -p "$out"
port=29800
for impl in ours nccl_baseline ddp; do
  port=$((port + 1))
  if [ "$N" = "1" ]; then
    timeout 400 python bench.py --gpus 1 --steps 20 --warmup 5 --impl $impl > "$out/bench_$impl.json" 2> "$out/bench_$impl.err"
  else
    timeout 400 python -m torch.distributed.run --nnodes=1 --nproc-per-node "$N" --master-addr 127.0.0.1 --master-port $port bench.py --gpus "$N" --steps 20 --warmup 5 \
        --impl $impl > "$out/bench_$impl.json" 2> "$out/bench_$impl.err"
  fi
  echo "bench $impl rc=$?" >> "$out/bench_$impl.err"
  python - "$out/bench_$impl.json" "$impl" "$N" <<'PY'
import json, sys
path, impl, n = sys.argv[1:4]
try:
    d = json.load(open(path))
    b = d.get("bert_large_bytegrad", {})
    print(f"{impl} N={n}: vgg16 {d['value']:.0f} img/s (e2e {d['e2e']['value']:.0f}), bert {b.get('value', 0):.1f} samples/s (e2e {(b.get('e2e') or {}).get('value', 0):.1f}), "
          f"verify {d.get('verify', {}).get('fraction_outside_tolerance')}, clocks {d['clocks']}")
except Exception as e:  # noqa: BLE001
    print(f"{impl} N={n}: no result ({e}); see {path.replace('.json', '.err')}")
PY
done
