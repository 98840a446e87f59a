#!/bin/sh
# TEST TOOL: host instantiation of embree_b200/csrc/interp.cuh (see interp_emu.cpp header comment); same flags as tests/emu
set -e
cd "$(dirname "$0")"
mkdir -p _build
g++ -O2 -g -std=c++17 -fPIC -shared -mfma -ffp-contract=off -o _build/libinterp_emu.so interp_emu.cpp
