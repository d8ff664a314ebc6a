#!/bin/bash
# Builds libaab200.so (all sm_90a kernels + the C-ABI) in-tree. nvcc cross-compiles without a GPU.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC --use_fast_math"
FLAGS_EXACT="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC"
mkdir -p ../_build
pids=()
for f in igemm attention norm elementwise clip_image; do
  if [ ../_build/$f.o -nt $f.cu ] && [ ../_build/$f.o -nt common.cuh ] && [ ../_build/$f.o -nt igemm.h ] && [ ../_build/$f.o -nt wgmma.cuh ]; then continue; fi
  $NVCC $FLAGS_EXACT -c $f.cu -o ../_build/$f.o &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
# link under a temporary name and rename: a reader (dlopen, a repository snapshot) never sees a half-written library
$NVCC -arch=sm_90a -shared -o ../libaab200.so.tmp ../_build/igemm.o ../_build/attention.o ../_build/norm.o ../_build/elementwise.o ../_build/clip_image.o -lcudart
mv -f ../libaab200.so.tmp ../libaab200.so
echo "built $(realpath ../libaab200.so)"
