#!/bin/bash
# Debug variant of the CUDA library with clock64 stamps at the phase boundaries of k_match / k_terms / the IESKF update (IM_STAMP in the
# sources; empty in the product build).  Read with tools/debug/lio_stamps.py.
cd "$(dirname "$0")/../.."
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -fmad=false -Xcompiler -fPIC -shared -DIM_DEBUG_STAMPS \
     -ccbin /usr/bin/g++ -o tools/debug/libimmesh_stamps.so immesh_b200/csrc/*.cu
