#!/bin/bash
# Runs the GPU parity suites one process per file (a device fault in one cannot poison the next).
# Usage (under gpurun): bash scripts/gpu_tests.sh
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw --format=csv > gpurun_out/nvsmi.txt 2>&1
for f in tests/test_gpu_gemm.py tests/test_gpu_forward.py tests/test_gpu_sampler.py tests/test_gpu_mdn_sample.py \
         tests/test_gpu_backward_stages.py tests/test_gpu_forward_stages.py tests/test_gpu_langevin.py tests/test_gpu_latent_stats.py \
         tests/test_gpu_coverage_metrics.py tests/test_gpu_snapshot_sampling.py tests/test_gpu_ddim.py tests/test_gpu_ddim_encode.py tests/test_gpu_dpm.py \
         tests/test_gpu_ssm_backward_stages.py tests/test_gpu_ssm.py tests/test_gpu_bench_stages.py "$@"; do
  n=$(basename $f .py)
  echo "=== $f"
  timeout 420 python -m pytest $f -m gpu -q -x --timeout=240 -p no:cacheprovider > gpurun_out/$n.log 2>&1
  echo "exit=$?" >> gpurun_out/$n.log
  tail -n 25 gpurun_out/$n.log
done
