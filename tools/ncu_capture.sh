#!/bin/bash
# ncu evidence: one launch list of a short bench run plus one `--set full` capture per hot kernel.
# Run on the GPU machine from the repository root; reports land in prof_out/ (git-ignored) and are exported to CSV with tools/ncu_export.sh.
#   tools/ncu_capture.sh <tag> [odometry] [kernel ...]
set -u
TAG=${1:-r1}; ODO=${2:-0}; shift 2 || true
KERNELS=${@:-icp_frame_kernel integrate_kernel raycast_kernel bilateral_scale_kernel frontend_pyramid_kernel}
export KT_BENCH_FRAMES=8
mkdir -p prof_out
BENCH="python bench.py --steps 4 --warmup 3 --no-cpu-baseline --odometry $ODO"
ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file prof_out/launches_${TAG}_odo${ODO}.csv $BENCH > prof_out/ncu_bench_${TAG}.log 2>&1
for k in $KERNELS; do
    timeout 600 ncu --set full --clock-control none --import-source on -k regex:$k -s 3 -c 1 -f -o prof_out/prof_${TAG}_$k $BENCH > prof_out/ncu_${TAG}_$k.log 2>&1
    tail -2 prof_out/ncu_${TAG}_$k.log
done
