#!/bin/bash
# Debug-counter build of the library (RMD_DEBUG_COUNTERS=1) for tools/timeline_probe.py:
#   RMD_B200_LIB=tools/build/librmd_b200_dbg.so python tools/timeline_probe.py
set -e
cd "$(dirname "$0")/.."
mkdir -p tools/build/dbg
SRC=rpg_open_remode_b200/csrc
FLAGS="-std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -use_fast_math -Xcompiler -fPIC -DRMD_DEBUG_COUNTERS=1"
for f in $SRC/*.cu; do
  nvcc $FLAGS -c $f -o tools/build/dbg/$(basename $f .cu).o &
done
wait
nvcc -shared -o tools/build/librmd_b200_dbg.so tools/build/dbg/*.o -gencode arch=compute_90a,code=sm_90a -lpthread -ldl
ls -la tools/build/librmd_b200_dbg.so
