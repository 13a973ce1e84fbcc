#!/bin/sh
# Build a tuning variant of the library next to the default one:
#   tools/build_variant.sh NAME "-DDNG_NT=384 -DDNG_CTAS_PER_SM=2"
# -> dragnet_b200/libdragnet_gpu_NAME.so  (use with DNG_LIB=...)
# (the flags reach api.cu and compressed.cu, the decoders' policies included:
# the run-time linked F kernel is built by the Makefile's JITFLAGS)
set -e
cd "$(dirname "$0")/../dragnet_b200/csrc"
mkdir -p build/var_$1
NVCC="/usr/local/cuda/bin/nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-Wall $2"
$NVCC -Xptxas -v -c -o build/var_$1/api.o api.cu 2> build/var_$1/api.log
grep -A2 "scan_kernelENS" build/var_$1/api.log | grep -E "registers|spill" || true
$NVCC -c -o build/var_$1/compressed.o compressed.cu
make -s build/merge.o build/plan.o build/result.o build/tmpl.o build/fast.o build/jit.o build/jit_load.o build/jit_cache.o build/jit_blob.o
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared \
    -o ../libdragnet_gpu_$1.so build/var_$1/api.o build/var_$1/compressed.o build/merge.o build/plan.o \
    build/result.o build/tmpl.o build/fast.o build/jit.o build/jit_load.o build/jit_cache.o build/jit_blob.o -ldl
