#!/bin/bash
# tools/build_variant.sh NAME -DFLAG=... : variants/lib_NAME.so = the library with extra nvcc flags (for tools/ab_variants.sh; SMR_LIB_PATH selects it)
set -e
name=$1; shift
cd "$(dirname "$0")/../sortmerna_b200/csrc"
make -s smr_index.o smr_build.o smr_blob.o
mkdir -p ../../variants
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xptxas -v "$@" -c smr_capi.cu -o /tmp/smr_capi_$name.o 2> ../../variants/ptxas_$name.txt
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../variants/lib_$name.so /tmp/smr_capi_$name.o smr_index.o smr_build.o smr_blob.o -lcudart
grep -A2 "lis_kernel" ../../variants/ptxas_$name.txt | grep -E "stack frame|Used" | head -2
