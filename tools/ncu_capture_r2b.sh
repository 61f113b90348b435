#!/bin/bash
# Round-2 ncu evidence, second pass: the kernels that changed after tools/ncu_capture_r2.sh ran (integrate with the frustum box and the
# fused z sums) and the slice post-processing kernels.   tools/ncu_capture_r2b.sh <tag>
set -u
TAG=${1:-r2v2}
export KT_BENCH_FRAMES=8
mkdir -p prof_out
B0="python bench.py --steps 4 --warmup 3 --no-cpu-baseline --no-shared-volume --odometry 0"
B1024="python bench.py --steps 4 --warmup 3 --no-cpu-baseline --no-shared-volume --odometry 0 --vol 1024"
ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file prof_out/launches_${TAG}_odo0.csv $B0 > prof_out/ncu_${TAG}_l0.log 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -c 500 --csv --log-file prof_out/launches_${TAG}_shift.csv python tools/prof_shift.py > prof_out/ncu_${TAG}_ls.log 2>&1
cap() {  # name, kernel regex, skip, command...
  local name=$1 k=$2 skip=$3; shift 3
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:$k -s $skip -c 1 -f -o prof_out/prof_${TAG}_$name "$@" > prof_out/ncu_${TAG}_$name.log 2>&1
  tail -1 prof_out/ncu_${TAG}_$name.log | cut -c1-200
}
cap integrate_kernel integrate_kernel 3 $B0
cap integrate_kernel_1024 integrate_kernel 3 $B1024
cap slice_normals_kernel slice_normals_kernel 1 python tools/prof_shift.py
cap slice_accumulate_kernel slice_accumulate_kernel 1 python tools/prof_shift.py
cap slice_mark_kernel slice_mark_kernel 1 python tools/prof_shift.py
cap extract_kernel extract_kernel 1 python tools/prof_shift.py
cap ztable_kernel ztable_kernel 3 $B0
