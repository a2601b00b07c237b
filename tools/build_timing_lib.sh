#!/bin/bash
# debug build of the C-ABI library with the ba_schur_tc_kernel timeline stamps (-DDBA_TC_TIMING); used by tools/tc_timeline.py
set -e
cd "$(dirname "$0")/.."
mkdir -p /tmp/dba_dbg tools/bin
for f in common corr_index altcorr geom ba chol corr_volume; do
  nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -DDBA_TC_TIMING -c droid_slam_b200/csrc/$f.cu -o /tmp/dba_dbg/$f.o -Idroid_slam_b200/csrc -Iinclude &
done
wait
nvcc -shared -o tools/bin/libdroid_b200_timing.so /tmp/dba_dbg/*.o -lcudart
