#!/bin/bash
# Source-level `ncu --set full` of ONE launch per tensor-core kernel variant at its bench shape (tools/layer_prof.py), on the GPU:
#     bash tools/ncu_layers.sh <tag> layer[:kernel-regex] ...      e.g.  r2 conv6:conv3d_tcdc conv1s2:conv3d_tcs2 bb64:conv3d_tcg
# -> gpurun_out/<tag>_<layer>.ncu-rep (with -lineinfo source correlation; read here with `ncu -i ... --page source --csv`)
set -u
TAG=$1; shift
mkdir -p gpurun_out
for spec in "$@"; do
  L=${spec%%:*}; K=${spec#*:}; [ "$K" = "$spec" ] && K=conv3d
  ncu --set full --clock-control none --import-source on --kernel-name-base demangled -k regex:$K -s 3 -c 1 -f \
      -o gpurun_out/${TAG}_${L} python tools/layer_prof.py $L 8 2 > /dev/null 2>&1
  ls -la gpurun_out/${TAG}_${L}.ncu-rep
done
