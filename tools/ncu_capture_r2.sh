#!/bin/bash
# Round-2 ncu evidence: one launch list per configuration and one `--set full` capture per product kernel at the shipped configuration.
#   tools/ncu_capture_r2.sh <tag>        (run from the repository root; reports land in prof_out/, export with tools/ncu_export.sh)
set -u
TAG=${1:-r2}
export KT_BENCH_FRAMES=8
mkdir -p prof_out
B0="python bench.py --steps 4 --warmup 3 --no-cpu-baseline --no-shared-volume --odometry 0"
B2="python bench.py --steps 4 --warmup 3 --no-cpu-baseline --no-shared-volume --odometry 2"
B1024="python bench.py --steps 4 --warmup 3 --no-cpu-baseline --no-shared-volume --odometry 0 --vol 1024"
ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file prof_out/launches_${TAG}_odo0.csv $B0 > prof_out/ncu_${TAG}_l0.log 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file prof_out/launches_${TAG}_odo2.csv $B2 > prof_out/ncu_${TAG}_l2.log 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file prof_out/launches_${TAG}_shift.csv python tools/prof_shift.py > prof_out/ncu_${TAG}_ls.log 2>&1
cap() {  # name, kernel regex, skip, command...
  local name=$1 k=$2 skip=$3; shift 3
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:$k -s $skip -c 1 -f -o prof_out/prof_${TAG}_$name "$@" > prof_out/ncu_${TAG}_$name.log 2>&1
  tail -1 prof_out/ncu_${TAG}_$name.log | cut -c1-200
}
cap icp_frame_kernel icp_frame_kernel 3 $B0
cap integrate_kernel integrate_kernel 3 $B0
cap raycast_kernel raycast_kernel 3 $B0
cap bilateral_scale_kernel bilateral_scale_kernel 3 $B0
cap frontend_pyramid_kernel frontend_pyramid_kernel 3 $B0
cap rgbd_frame_kernel rgbd_frame_kernel 3 $B2
cap frontend_pyramid_kernel_rgbd frontend_pyramid_kernel 3 $B2
cap integrate_kernel_1024 integrate_kernel 3 $B1024
cap raycast_kernel_1024 raycast_kernel 3 $B1024
cap extract_kernel extract_kernel 1 python tools/prof_shift.py
cap clear_planes_x_kernel clear_planes_x_kernel 1 python tools/prof_shift.py
cap views_kernel views_kernel 0 python tools/prof_shift.py
cap fill_zero_u4 fill_zero_u4 0 python tools/prof_shift.py
cap transform_maps_kernel transform_maps_kernel 0 python tools/prof_shift.py
