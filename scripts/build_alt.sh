#!/bin/bash
# Development aid: link libfmb200 with an alternative fm_ordered.{cu,cuh} (A/B timing of kernel variants on one box).
#   scripts/build_alt.sh <tag> <dir holding fm_ordered.cu + fm_ordered.cuh>
set -e
tag=$1; dir=$2
root=$(cd "$(dirname "$0")/.." && pwd)
mkdir -p $root/libfm_b200/lib/alt
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -I $root/include -I $root/libfm_b200/csrc \
  -c $dir/fm_ordered.cu -o /tmp/fm_ordered_$tag.o
objs=$(ls $root/build/obj/*.o | grep -v fm_ordered.o)
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o $root/libfm_b200/lib/alt/libfmb200_$tag.so $objs /tmp/fm_ordered_$tag.o
echo built $root/libfm_b200/lib/alt/libfmb200_$tag.so
