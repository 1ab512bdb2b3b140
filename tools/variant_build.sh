#!/bin/bash
# Builds a variant of the library with extra -D flags next to the product library (measuring aid; tools/tick_probe.py
# loads it when HQS_LIB names it).  Usage: tools/variant_build.sh <suffix> [-DFLAG ...]
set -e
cd "$(dirname "$0")/.."
sfx=$1; shift
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 "$@" -Xcompiler -fPIC,-Wall,-Wno-subobject-linkage \
     --shared -cudart shared -Iinclude -o hyperqueue_b200/libhqsched_b200_$sfx.so hyperqueue_b200/csrc/hqsched.cu
