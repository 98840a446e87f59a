// interp_emu.cpp -- TEST TOOL ONLY: the host instantiation of embree_b200/csrc/interp.cuh, the arithmetic rtcInterpolate and the
// batched interpolation kernel share, so that tests/test_interpolate_curves.py can hold it to the reference's answers on a machine
// without a GPU.  Compiled by tests/interp_emu/build.sh into tests/interp_emu/_build/libinterp_emu.so; never loaded by the product.
#include <stdint.h>

#include "../../embree_b200/csrc/interp.cuh"

using namespace rtk;

// rtcInterpolateN through interp.cuh: n queries (primIDs, u, v) of one geometry, `kind` an rtk::InterpKind; idx / data / tang are
// the index, requested and tangent buffers with their byte strides; outputs value j of query i at [j * n + i] (NULL = not wanted)
extern "C" void emu_interpolate(unsigned kind, unsigned basis, const void* idx, uint64_t istride, const void* data, uint64_t dstride,
                                const void* tang, uint64_t tstride, const uint32_t* primIDs, const float* u, const float* v, uint64_t n,
                                unsigned valueCount, float* P, float* dPdu, float* dPdv, float* ddPdudu, float* ddPdvdv, float* ddPdudv) {
  for (uint64_t i = 0; i < n; ++i) {
    float* const out[6] = {P ? P + i : nullptr, dPdu ? dPdu + i : nullptr, dPdv ? dPdv + i : nullptr,
                           ddPdudu ? ddPdudu + i : nullptr, ddPdvdv ? ddPdvdv + i : nullptr, ddPdudv ? ddPdudv + i : nullptr};
    interpolate_prim(kind, basis, reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(idx) + primIDs[i] * istride),
                     static_cast<const uint8_t*>(data), dstride, static_cast<const uint8_t*>(tang), tstride, u[i], v[i], valueCount, out, n);
  }
}
