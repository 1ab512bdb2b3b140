#!/bin/bash
# Measuring build of the library: -DHQS_TRACE replaces the phase stamps of hqs_debug_read by cycle sums of the sections
# of the lean first-fit loop (tools/trace_probe.py reads them) or of the wide loop (tools/trace_wide.py), and adds
# %globaltimer stamps of the emit tail (tools/trace_emit.py).  The product library is not touched.
set -e
cd "$(dirname "$0")/.."
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -DHQS_TRACE -Xcompiler -fPIC,-Wall,-Wno-subobject-linkage \
     --shared -cudart shared -Iinclude -o hyperqueue_b200/libhqsched_b200_trace.so hyperqueue_b200/csrc/hqsched.cu
