#!/bin/bash
# Builds dragonfly_b200/libdfb200.so for sm_90a (H100) in-tree.  Used by __graft_entry__.build().
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v"
mkdir -p build
for f in kernels api ubench; do
  $NVCC $FLAGS -c $f.cu -o build/$f.o 2> build/$f.ptxas.log || { cat build/$f.ptxas.log; exit 1; }
done
$NVCC $ARCH -shared -o ../libdfb200.so build/kernels.o build/api.o build/ubench.o -lcudart
echo "built $(cd .. && pwd)/libdfb200.so"
