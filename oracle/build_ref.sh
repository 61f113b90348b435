#!/bin/bash
# TEST INFRASTRUCTURE ONLY. Builds oracle/_ref/libkt_ref_<VOL>.so: the reference's own CUDA operators
# ($KT_REFERENCE_ROOT/src/frontend/cuda/*.cu + containers/*.cpp, compiled from where they lie) plus
# oracle/ref_harness.cu. The reference sources are copied to a TEMPORARY directory only because two files
# need mechanical patches to compile for sm_90 (SURVEY.md D7) and VOL must become a -D macro (D5):
#   reduce.cu : __shfl_down(x, offset)  -> __shfl_down_sync(0xffffffff, x, offset)
#   extract.cu: __all(..)/__ballot(..)  -> *_sync(0xffffffff, ..)
#   internal.h: #define VOL 512         -> #ifndef VOL / #define VOL 512 / #endif
# Nothing but the .so lands in the repo tree (oracle/_ref/ is git-ignored). Flags are the reference's own
# (CMakeLists.txt:47): --ftz=true --prec-div=false --prec-sqrt=false, arch retargeted to sm_90.
# usage: oracle/build_ref.sh [VOL ...]   (default: 256 512)
set -euo pipefail
REF=${KT_REFERENCE_ROOT:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
if [ ! -d "$REF/src/frontend/cuda" ]; then echo "build_ref: $REF not present, keeping prebuilt $OUT"; exit 0; fi
mkdir -p "$OUT"
VOLS=${@:-256 512}
TMP=$(mktemp -d /tmp/ktref_build.XXXXXX)
trap 'rm -rf "$TMP"' EXIT
cp -r "$REF/src/frontend/cuda" "$TMP/cuda"
sed -i -E 's/__shfl_down\(([^,]+), offset\)/__shfl_down_sync(0xffffffffu, \1, offset)/g' "$TMP/cuda/reduce.cu"
sed -i -E 's/__all \(/__all_sync (0xffffffffu, /g; s/__ballot \(/__ballot_sync (0xffffffffu, /g' "$TMP/cuda/extract.cu"
sed -i 's/^#define VOL 512/#ifndef VOL\n#define VOL 512\n#endif/' "$TMP/cuda/internal.h"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-std=c++14 -O3 -gencode arch=compute_90,code=sm_90 --ftz=true --prec-div=false --prec-sqrt=false -Xcompiler -fPIC -w"
for V in $VOLS; do
  B=$TMP/build_$V; mkdir -p $B
  pids=()
  for f in bilateral_pyrdown maps reduce tsdf_volume ray_caster extract image_generator; do
    $NVCC $FLAGS -DVOL=$V -I"$TMP/cuda" -c "$TMP/cuda/$f.cu" -o $B/$f.o & pids+=($!)
  done
  $NVCC $FLAGS -DVOL=$V -I"$TMP/cuda" -I"$HERE" -Xcompiler -ffp-contract=off -c "$HERE/ref_harness.cu" -o $B/ref_harness.o & pids+=($!)
  for f in device_memory initialization; do
    g++ -O3 -fPIC -w -I/usr/local/cuda/include -I"$TMP/cuda/containers" -c "$TMP/cuda/containers/$f.cpp" -o $B/$f.o & pids+=($!)
  done
  for p in "${pids[@]}"; do wait $p; done
  $NVCC -shared -o "$OUT/libkt_ref_$V.so" $B/*.o -lcudart
  echo "built $OUT/libkt_ref_$V.so"
done
