#!/usr/bin/env bash
# Race / sync / memory checks of the CUDA kernels (SURVEY §5.2: the reference wires up none). One GPU, under gpurun:
#   gpurun --timeout 1200 -- 'bash scripts/sanitize.sh'
set -uo pipefail
mkdir -p gpurun_out
for tool in memcheck racecheck synccheck; do
  compute-sanitizer --tool $tool --error-exitcode 1 python -m pytest tests/test_kernels_gpu.py -q -x -k "sgd or adam or minmax or nhwc or elementwise" \
      > gpurun_out/sanitizer_$tool.log 2>&1
  echo "$tool exit=$?" | tee -a gpurun_out/sanitizer_summary.txt
done
# the peer / quantised / MoE kernels among virtual ranks on this one GPU (memcheck + synccheck; racecheck only tracks shared memory and
# does not model wgmma / mbarrier / cross-stream global traffic). P = 1 cases keep the run short; spinning multi-stream cases are slow under
# the sanitizer, so their in-kernel time-out is raised.
for tool in memcheck synccheck; do
  BAGUA_PEER_TIMEOUT_S=600 compute-sanitizer --tool $tool --error-exitcode 1 python -m pytest tests/test_virtual_peer_gpu.py -q -x -k "1-" \
      > gpurun_out/sanitizer_${tool}_peer_kernels.log 2>&1
  echo "$tool(peer kernels, P=1) exit=$?" | tee -a gpurun_out/sanitizer_summary.txt
done
compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_zz_new_kernels_gpu.py -q -x \
    > gpurun_out/sanitizer_memcheck_new_kernels.log 2>&1
echo "memcheck(new kernels) exit=$?" | tee -a gpurun_out/sanitizer_summary.txt
# host side: the C++ scheduler under TSAN/ASAN runs in the CPU suite (tests/test_scheduler_tsan.py)
