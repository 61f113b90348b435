#!/bin/bash
# Round-2 ncu evidence, third pass: the kernels off the default tracker path -- the small slice-processing kernels, the y/z slab clear,
# and the per-iteration odometry kernels of the operator API / large-image fallback (KT_FORCE_PER_ITERATION).   tools/ncu_capture_r2c.sh <tag>
set -u
TAG=${1:-r2v3}
mkdir -p prof_out
cap() {  # name, kernel regex, skip, command...
  local name=$1 k=$2 skip=$3; shift 3
  timeout 600 ncu --set full --clock-control none --import-source on -k regex:$k -s $skip -c 1 -f -o prof_out/prof_${TAG}_$name "$@" > prof_out/ncu_${TAG}_$name.log 2>&1
  tail -1 prof_out/ncu_${TAG}_$name.log | cut -c1-160
}
cap slice_bounds_kernel slice_bounds_kernel 0 python tools/prof_shift.py
cap slice_mark_kernel slice_mark_kernel 0 python tools/prof_shift.py
cap scan_final_kernel scan_final_kernel 0 python tools/prof_shift.py
cap slice_centroid_kernel slice_centroid_kernel 0 python tools/prof_shift.py
cap slice_normals_kernel slice_normals_kernel 0 python tools/prof_shift.py
cap clear_planes_yz_kernel clear_planes_yz_kernel 0 python tools/prof_shift.py
export KT_FORCE_PER_ITERATION=1
cap icp_kernel "icp_kernel" 40 python tools/stage_ab.py 8 512 0
cap residual_kernel residual_kernel 40 python tools/stage_ab.py 8 512 2
cap rgb_step_kernel rgb_step_kernel 40 python tools/stage_ab.py 8 512 2
