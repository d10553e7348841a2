#!/bin/bash
# Developer script: GPU tests, profile, quick timings, checks build and scheduler bench on one GPU, for the current tree.
mkdir -p gpurun_out
timeout 2400 python -m pytest tests -m gpu -x -q > gpurun_out/pytest_gpu.log 2>&1
bash tools/gpu_profile.sh > gpurun_out/gpu_profile.out 2>&1
timeout 300 python tools/quick_bench.py 2 3 4 5 > gpurun_out/quick.log 2>&1
NHD_B200_LIB=$PWD/nhd_b200/libnhd_b200_chk.so timeout 300 python tools/chk_run.py 4 0 > gpurun_out/chk.log 2>&1
timeout 900 python tools/scheduler_bench.py 65536 4096 > gpurun_out/scheduler_bench.log 2>&1
tail -n 3 gpurun_out/pytest_gpu.log; tail -n 4 gpurun_out/sanitizer_*.log; cat gpurun_out/phase.log gpurun_out/quick.log gpurun_out/chk.log; tail -n 1 gpurun_out/scheduler_bench.log | cut -c1-700; cut -c1-900 gpurun_out/bench.log
