#!/usr/bin/env bash
# The GPU work that is queued behind the CPU-only development of round 1, in the order it should be spent
# (each block is one gpurun call; budgets in GPU-minutes = wall minutes x GPUs).
#
#   1 GPU  (~20 min):  gpurun --timeout 1500 -- 'bash scripts/gpu_validation_plan.sh one'
#   2 GPUs (~2x10 min): gpurun --gpus 2 --timeout 900 -- 'bash scripts/gpu_validation_plan.sh two'
#   8 GPUs (~8x6 min):  gpurun --gpus 8 --timeout 600 -- 'bash scripts/gpu_validation_plan.sh eight'
set -uo pipefail
mkdir -p gpurun_out
case "${1:-one}" in
one)
  timeout 120 python -m bagua_b200.script.bagua_doctor --json > gpurun_out/doctor_1.json 2> gpurun_out/doctor_1.err; echo "doctor exit=$?" | tee gpurun_out/plan_one.txt
  timeout 600 python -m pytest tests -m "gpu and not multigpu" -x -q > gpurun_out/pytest_gpu_1.log 2>&1; echo "pytest1 exit=$?" | tee -a gpurun_out/plan_one.txt
  timeout 600 bash scripts/ncu_profile.sh; echo "ncu exit=$?" | tee -a gpurun_out/plan_one.txt
  BAGUA_EXPERIMENTAL=1 timeout 400 python -m pytest tests/test_zz_new_kernels_gpu.py -x -q > gpurun_out/pytest_new_kernels.log 2>&1; echo "new kernels exit=$?" | tee -a gpurun_out/plan_one.txt
  timeout 120 python benchmarks/torch_ddp_baseline.py --steps 30 --warmup 5 > gpurun_out/torch_ddp_n1.json 2> gpurun_out/torch_ddp_n1.err; echo "torch ddp baseline exit=$?" | tee -a gpurun_out/plan_one.txt
  timeout 120 python bench.py --steps 30 --warmup 5 > gpurun_out/bench1.json 2> gpurun_out/bench1.err; echo "bench exit=$?" | tee -a gpurun_out/plan_one.txt
  # A/B of the host-overhead experiment (only meaningful if the gated test above passed)
  BAGUA_NHWC_FINALIZE=1 timeout 120 python bench.py --steps 30 --warmup 5 > gpurun_out/bench1_nhwc_finalize.json 2> gpurun_out/bench1_nhwc_finalize.err
  echo "bench (nhwc finalize) exit=$?" | tee -a gpurun_out/plan_one.txt
  BAGUA_NATIVE_HOOKS=1 timeout 120 python bench.py --steps 30 --warmup 5 > gpurun_out/bench1_native_hooks.json 2> gpurun_out/bench1_native_hooks.err
  echo "bench (native hooks) exit=$?" | tee -a gpurun_out/plan_one.txt
  BAGUA_NATIVE_NHWC=1 timeout 120 python bench.py --steps 30 --warmup 5 > gpurun_out/bench1_native_nhwc.json 2> gpurun_out/bench1_native_nhwc.err
  echo "bench (C++ nhwc functions) exit=$?" | tee -a gpurun_out/plan_one.txt
  BAGUA_NATIVE_HOOKS=1 BAGUA_NATIVE_NHWC=1 BAGUA_NHWC_FINALIZE=1 timeout 120 python bench.py --steps 30 --warmup 5 > gpurun_out/bench1_all_host_opts.json 2> gpurun_out/bench1_all_host_opts.err
  echo "bench (native hooks + C++ nhwc functions + in-kernel finish) exit=$?" | tee -a gpurun_out/plan_one.txt
  # whole step replayed from a CUDA graph (gated test test_graphed_train_step_matches_eager_steps must have passed above)
  timeout 180 python bench.py --steps 30 --warmup 5 --cuda-graph > gpurun_out/bench1_cuda_graph.json 2> gpurun_out/bench1_cuda_graph.err
  echo "bench (cuda graph) exit=$?" | tee -a gpurun_out/plan_one.txt
  ;;
two)
  timeout 180 python -m bagua_b200.distributed.launch --nproc_per_node=2 --master_port=29605 -m bagua_b200.script.bagua_doctor > gpurun_out/doctor_2.log 2>&1
  echo "doctor(2) exit=$?" | tee gpurun_out/plan_two.txt
  # opt-in kernels written without hardware access in round 1: fused GEMM+combine, fused allreduce+Adam, mixed-precision Adam
  BAGUA_EXPERIMENTAL=1 timeout 400 python -m pytest tests/test_peer_gpu.py -q -k "fused or abort or sync_batchnorm or peer_allgather or graphed or sharded" > gpurun_out/pytest_experimental_2.log 2>&1
  echo "experimental exit=$?" | tee -a gpurun_out/plan_two.txt
  timeout 400 python -m pytest tests/test_peer_gpu.py -x -q > gpurun_out/pytest_peer_2.log 2>&1; echo "peer exit=$?" | tee -a gpurun_out/plan_two.txt
  # the shipped examples on real GPUs (each asserts its own results)
  for ex in "communication_primitives/main.py" "mnist/main.py --algorithm bytegrad --epochs 1 --steps-per-epoch 20" "moe/mnist_main.py --epochs 1 --steps-per-epoch 20 --num-local-experts 2" \
            "squad/main.py --tiny --epochs 1 --num-synthetic 64 --max_seq_length 128 --doc_stride 64 --algorithm qadam --output_dir /tmp/squad_plan --overwrite_output_dir" \
            "imagenet/main.py --arch vgg16 --synthetic --epochs 1 --steps-per-epoch 10 --fused-shard"; do
    timeout 240 python -m bagua_b200.distributed.launch --nproc_per_node=2 --master_port=$((29640 + RANDOM % 50)) examples/$ex > gpurun_out/example_$(echo $ex | cut -d/ -f1).log 2>&1
    echo "example $ex exit=$?" | tee -a gpurun_out/plan_two.txt
  done
  # inline issue of the bucket kernels (no worker-thread hand-off) — A/B on the 2-GPU point
  for inl in 0 1; do
    BAGUA_INLINE_COMM=$inl timeout 200 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port $((29630 + inl)) \
      bench.py --gpus 2 --steps 30 --warmup 5 > gpurun_out/bench2_inline$inl.json 2> gpurun_out/bench2_inline$inl.err
    echo "bench2 inline=$inl exit=$?" | tee -a gpurun_out/plan_two.txt
  done
  timeout 240 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29637 \
    bench.py --gpus 2 --steps 30 --warmup 5 --cuda-graph > gpurun_out/bench2_cuda_graph.json 2> gpurun_out/bench2_cuda_graph.err
  echo "bench2 cuda graph exit=$?" | tee -a gpurun_out/plan_two.txt
  for fused in 0 1; do
    BAGUA_MOE_FUSED_COMBINE=$fused timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port $((29610 + fused)) \
      benchmarks/config_bench.py --config gpt2_moe --steps 10 --warmup 3 >> gpurun_out/config_bench_n2.jsonl 2>> gpurun_out/config_bench_n2.err
    echo "gpt2_moe fused=$fused exit=$?" | tee -a gpurun_out/plan_two.txt
  done
  ;;
eight)
  BAGUA_EXPERIMENTAL=1 timeout 300 python -m pytest tests/test_peer_gpu.py -x -q -k "hierarchical or fused" > gpurun_out/pytest_experimental_8.log 2>&1
  echo "experimental(8) exit=$?" | tee gpurun_out/plan_eight.txt
  timeout 200 python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29690 benchmarks/torch_ddp_baseline.py \
    --steps 30 --warmup 5 > gpurun_out/torch_ddp_n8.json 2> gpurun_out/torch_ddp_n8.err; echo "torch ddp baseline(8) exit=$?" | tee -a gpurun_out/plan_eight.txt
  port=29700
  for cfg in gpt2_moe bert_bytegrad resnet50_decentralized; do
    for arm in peer nccl; do
      port=$((port + 1))
      timeout 240 python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port $port \
        benchmarks/config_bench.py --config $cfg --arm $arm --steps 10 --warmup 3 >> gpurun_out/config_bench_n8.jsonl 2>> gpurun_out/config_bench_n8.err
      echo "$cfg $arm exit=$?" | tee -a gpurun_out/plan_eight.txt
    done
  done
  ;;
esac
