#!/bin/bash
# Builds libdip.so (sm_90a) in-tree. Usage: deep-image-prior_b200/build.sh
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr"
mkdir -p build
for f in conv_tc kernels_mem downsample conv_simt engine; do
  if [ ! -f build/$f.o ] || [ csrc/$f.cu -nt build/$f.o ] || [ -n "$(find csrc include ../include -name '*.h' -newer build/$f.o -o -name '*.cuh' -newer build/$f.o 2>/dev/null)" ]; then
    echo "[nvcc] $f.cu"
    $NVCC $FLAGS ${PTXAS_V:+-Xptxas -v} -c csrc/$f.cu -o build/$f.o &
  fi
done
wait
$NVCC -shared -o libdip.so build/conv_tc.o build/kernels_mem.o build/downsample.o build/conv_simt.o build/engine.o -cudart static
echo "built $(pwd)/libdip.so"
