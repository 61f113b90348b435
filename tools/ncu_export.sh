#!/bin/bash
# Export the captures tools/ncu_capture.sh brought back (prof_out/prof_<tag>_<kernel>.ncu-rep) to CSVs beside them (prof_out/ is git-ignored).
#   tools/ncu_export.sh <tag> <profiles-prefix>      e.g. tools/ncu_export.sh r1v9 r1_ncu_full_v9
set -u
TAG=$1; PREFIX=$2
for rep in prof_out/prof_${TAG}_*.ncu-rep; do
    k=$(basename $rep .ncu-rep); k=${k#prof_${TAG}_}
    ncu -i $rep --page raw --csv > prof_out/${PREFIX}_$k.csv
    ncu -i $rep --page source --csv --print-source cuda,sass > /tmp/${PREFIX}_${k}_source.csv 2>/dev/null
    echo "$k -> prof_out/${PREFIX}_$k.csv (source page: /tmp/${PREFIX}_${k}_source.csv)"
done
