#!/bin/bash
# Round-2 profiling pass (run under gpurun on ONE GPU): per-launch durations of the small paths and one full capture of the
# dominant kernel.  Outputs under gpurun_out/; the summaries worth keeping are copied into profiles/ by hand.
mkdir -p gpurun_out
M="--metrics gpu__time_duration.sum --clock-control none --csv"
ncu $M --log-file gpurun_out/r02_launches_mc.csv python tools/prof_r2.py mc > /dev/null 2>&1
ncu $M --log-file gpurun_out/r02_launches_train.csv python tools/prof_r2.py train 16384 > /dev/null 2>&1
ncu $M --log-file gpurun_out/r02_launches_c2f.csv python tools/prof_r2.py c2f > /dev/null 2>&1
ncu $M -c 600 --log-file gpurun_out/r02_launches_bench.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-secondary > gpurun_out/r02_bench_under_ncu.log 2>&1
ncu --set full --clock-control none --import-source on -k regex:sdf_tc_kernel --launch-skip 1 -c 1 -f -o gpurun_out/r02_tc3_full python tools/prof_r2.py render > /dev/null 2>&1
ls -la gpurun_out/*.ncu-rep gpurun_out/r02_launches_*.csv
