#!/bin/bash
# usage: tools/ncu_capture.sh <name> <regex on the demangled kernel name> <workload> [launch-count]   (needs a GPU)
# Captures the matching launches with ncu --set full, exports the raw / source (SASS and CUDA-C views) /
# details pages into $NCU_OUT (default ncu_out/) and leaves the large .ncu-rep in /tmp/ncu.
set -e
name=$1; rx=$2; wl=$3; cnt=${4:-1}
out=${NCU_OUT:-ncu_out}
mkdir -p "$out" /tmp/ncu
ncu --set full --clock-control none --import-source on --kernel-name-base demangled -k "regex:$rx" --launch-count $cnt -f \
    -o /tmp/ncu/$name python tools/profile_run.py $wl 1 | tail -1
ncu -i /tmp/ncu/$name.ncu-rep --page raw --csv > "$out"/${name}_raw.csv
ncu -i /tmp/ncu/$name.ncu-rep --page source --csv > "$out"/${name}_source.csv 2>/dev/null || true
ncu -i /tmp/ncu/$name.ncu-rep --page details > "$out"/${name}_details.txt
ls -la "$out"/${name}_*
