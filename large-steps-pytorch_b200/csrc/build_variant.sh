#!/bin/bash
# ./build_variant.sh <suffix> <extra nvcc flags...>: builds ../largesteps_b200/libls_b200_<suffix>.so with the fused TUs recompiled under the flags (A/B builds)
SUF=$1; shift
NVCC=${NVCC:-nvcc}
NV="$NVCC -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC --expt-relaxed-constexpr"
FUSED="ls_pcg ls_fused_a ls_fused_b ls_fused_c ls_fused_batch"   # every TU that includes ls_pcg_fused.cuh
mkdir -p build_$SUF
for f in $FUSED; do $NV "$@" -c $f.cu -o build_$SUF/$f.o 2> build_$SUF/$f.log & done; wait
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../largesteps_b200/libls_b200_$SUF.so build/ls_capi.o build/ls_assemble.o build/ls_order.o build/ls_spmm.o build/ls_adam.o build/ls_glue.o $(for f in $FUSED; do echo build_$SUF/$f.o; done) -lcudart_static -lpthread -ldl -lrt && echo built $SUF
