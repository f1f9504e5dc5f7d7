#!/bin/bash
# Builds libfav_b200.so (sm_90a, H100) in-tree.  nvcc cross-compiles without a GPU.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=libfav_b200.so
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden -Xptxas -v"
mkdir -p build
objs=""
for f in common front consistency vr net_kernels conv_tc net session video_pipeline; do
  if [ ! -f build/$f.o ] || [ csrc/$f.cu -nt build/$f.o ] || [ -n "$(find csrc include ../include -name '*.cuh' -newer build/$f.o -o -name '*.hpp' -newer build/$f.o -o -name '*.h' -newer build/$f.o 2>/dev/null | head -1)" ]; then
    echo "nvcc $f.cu"
    $NVCC $FLAGS -c csrc/$f.cu -o build/$f.o 2> build/$f.ptxas.log || { cat build/$f.ptxas.log; exit 1; }
  fi
  objs="$objs build/$f.o"
done
g++ -O2 -fPIC -fvisibility=hidden -std=c++17 -c csrc/flo_io.cpp -o build/flo_io.o
$NVCC -shared -o $OUT $objs build/flo_io.o -gencode arch=compute_90a,code=sm_90a -lcudart -lz
echo "built $(pwd)/$OUT"
