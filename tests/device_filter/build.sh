#!/bin/sh
# TEST TOOL: compiles devfilter.cu as a user's translation unit would be compiled -- sm_90a, nvcc's default floating-point
# flags, the public headers through -I include only -- into _build/libdevfilter.so (ptxas report in _build/devfilter.ptxas.log)
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
mkdir -p _build
$NVCC -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I ../../include -Xcompiler -fPIC -Xptxas -v -shared \
    -o _build/libdevfilter.so devfilter.cu 2> _build/devfilter.ptxas.log || { cat _build/devfilter.ptxas.log; exit 1; }
