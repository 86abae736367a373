#!/bin/bash
# Round-2 profile collection on the GPU box (run under gpurun; everything lands in gpurun_out/, summarised here by
# scripts/summarize_profiles.py 2).  Never a bench value: numbers printed under ncu are discarded.
set -x
B="python bench.py --no-cpu-baseline --no-batch --no-microbench"
# (1) the bench line of this box, not under a profiler
$B --steps 20 --warmup 3 > gpurun_out/bench_line.json 2> gpurun_out/bench_line.err
# (2) every launch with its device time (cold-cache, serialised: shares only)
ncu --metrics gpu__time_duration.sum --clock-control none -s 300 -c 400 --csv --log-file gpurun_out/launches.csv $B --steps 4 --warmup 3 > gpurun_out/b_under_ncu.log 2>&1
# (3) the dominant kernels, --set full (default search: k_knn_box)
ncu --set full --clock-control none --import-source on -k regex:"k_knn_box|k_plane_fit|k_eval_unary" -s 18 -c 6 -o gpurun_out/prof_top $B --steps 2 --warmup 3 > gpurun_out/ncu_top.log 2>&1
