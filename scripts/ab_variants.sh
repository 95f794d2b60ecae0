#!/bin/bash
# Build one libtsgpu per compile-time setting (here, no GPU needed) into ab/ — then `scripts/ab_run.sh` times them on the GPU in one run.
# usage: scripts/ab_variants.sh name1 "-DFLAG=..." name2 "-DFLAG=..." ...
set -e
cd "$(dirname "$0")/.."
D=${AB_DIR:-ab}; mkdir -p $D
PKG=tiered-storage-for-apache-kafka_b200
while [ $# -ge 2 ]; do
  name=$1; flags=$2; shift 2
  nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr $flags -shared -o $D/libtsgpu_$name.so $PKG/csrc/tsgpu.cu -lcudart 2>/dev/null &
done
wait
ls -la $D/
