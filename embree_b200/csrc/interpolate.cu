// interpolate.cu -- batched rtcInterpolate of the hits of a traced batch (rtcb200InterpolateHits*), sm_90a.
//
// One thread per hit, grid-stride, 64-bit indices throughout (value j of hit i lives at j * M + i, which passes 2^32 at
// realistic sizes).  A thread reads the hit's u, v, primID, geomID and instID[0] and runs interp.cuh's interpolate_hit, the body
// rtcb200Interpolate1 runs in the caller's kernels: it resolves the hit's interpolation table entry (two lookups through an
// instance), gathers the primitive's indices and then the control values of each requested component: four at a time with
// 16-byte loads where the buffers' strides allow it, one at a time otherwise.  The arithmetic is interp.cuh's, the host
// rtcInterpolate's.  Consecutive threads are consecutive hits, so the stores of one value coalesce.  The kernel is a gather:
// no shared memory, no tensor cores.
#include "interp.cuh"
#include "rtk_device.h"

namespace rtk {

namespace {

__device__ __forceinline__ void store_value(const InterpParams& p, uint64_t at, const float o[6]) {
#pragma unroll
  for (int c = 0; c < 6; ++c)
    if (p.out[c]) p.out[c][at] = o[c];
}

__global__ void __launch_bounds__(128) interpolate_hits(const InterpParams p) {
  const uint64_t M = p.M;
  const unsigned V = p.valueCount;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* h = static_cast<const uint8_t*>(p.hits) + i * 96 + 60;   // RTCRayHit: hit.u at byte 60
    const float u = __ldg(reinterpret_cast<const float*>(h));
    const float v = __ldg(reinterpret_cast<const float*>(h + 4));
    const uint32_t primID = __ldg(reinterpret_cast<const uint32_t*>(h + 8));
    const uint32_t geomID = __ldg(reinterpret_cast<const uint32_t*>(h + 12));
    const uint32_t instID = __ldg(reinterpret_cast<const uint32_t*>(h + 16));
    if (geomID == kInvalidID) continue;   // a miss: its outputs stay as they are
    interpolate_hit(p.table, p.nentries, geomID, instID, primID, u, v, V,
                    [&](unsigned k, const float o[6]) { store_value(p, (uint64_t)k * M + i, o); });
  }
}

}  // namespace

int launch_interpolate(const InterpParams& p, cudaStream_t stream) {
  if (p.M == 0) return 0;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const uint64_t blocks = (p.M + 127) / 128;
  const unsigned grid = (unsigned)(blocks < (uint64_t)sms * 16 ? blocks : (uint64_t)sms * 16);
  interpolate_hits<<<grid, 128, 0, stream>>>(p);
  count_launch();
  return (int)cudaGetLastError();
}

}  // namespace rtk
