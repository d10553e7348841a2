#!/bin/bash
# Developer script: sanitizers + ncu captures + bench line.
mkdir -p gpurun_out
for tool in racecheck synccheck memcheck; do
  timeout 900 compute-sanitizer --tool $tool --print-limit 20 python tools/sanitizer_run.py > gpurun_out/sanitizer_$tool.log 2>&1
done
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/launches.csv \
    python bench.py --steps 3 --warmup 3 > gpurun_out/bench_under_ncu.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:'sweep_kernel|filter_kernel' -s 4 -c 2 -f -o gpurun_out/prof \
    python tools/profile_run.py 4 3 > gpurun_out/ncu_full.log 2>&1
NHD_B200_LIB=$PWD/nhd_b200/libnhd_b200_prof.so timeout 300 python tools/phase_profile.py 4 > gpurun_out/phase.log 2>&1
timeout 600 python bench.py > gpurun_out/bench.log 2>&1
timeout 600 python bench.py --impl reference --steps 3 --warmup 1 > gpurun_out/bench_ref.log 2>&1
tail -n 4 gpurun_out/sanitizer_*.log; tail -n 3 gpurun_out/ncu_full.log; cat gpurun_out/phase.log; cut -c1-1200 gpurun_out/bench.log
