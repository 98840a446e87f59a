#!/bin/sh
# TEST TOOL: compiles devshade.cu as a user's translation unit would be compiled -- sm_90a, nvcc's default floating-point
# flags, the public headers through -I include only -- into _build/libdevshade.so (ptxas report in _build/devshade.ptxas.log)
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
mkdir -p _build
$NVCC -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I ../../include -Xcompiler -fPIC -Xptxas -v -shared \
    -o _build/libdevshade.so devshade.cu 2> _build/devshade.ptxas.log || { cat _build/devshade.ptxas.log; exit 1; }
