#!/bin/bash
# ./build_variant.sh <suffix> <extra nvcc flags...>: builds ../largesteps_b200/libls_b200_<suffix>.so, every source compiled under
# the flags into build_<suffix>/ (A/B builds; the Makefile lists the sources)
set -e
SUF=$1; shift
cd "$(dirname "$0")"
make -j8 BUILD=build_$SUF OUT=../largesteps_b200/libls_b200_$SUF.so EXTRA="$*"
echo built $SUF
