// interpolate.cu -- batched rtcInterpolate of the hits of a traced batch (rtcb200InterpolateHits*), sm_90a.
//
// One thread per hit, grid-stride, 64-bit indices throughout (value j of hit i lives at j * M + i, which passes 2^32 at
// realistic sizes).  A thread reads the hit's u, v, primID, geomID and instID[0], resolves its interpolation table entry (two
// lookups through an instance), gathers the primitive's indices and then the control values of each requested component: four
// at a time with 16-byte loads where the buffers' strides allow it, one at a time otherwise.  The arithmetic is interp.cuh's, the
// host rtcInterpolate's.  Consecutive threads are consecutive hits, so the stores of one value coalesce.  The kernel is a gather:
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
    // resolve the entry: the scene's own geometry, or geometry geomID of the scene instance instID instantiates
    InterpEntry e;
    e.kind = INTERP_NONE;
    uint32_t slot = geomID, end = p.nentries;
    bool ok = true;
    if (instID != kInvalidID) {
      ok = instID < p.nentries && p.table[instID].kind == INTERP_INSTANCE;
      if (ok) { slot = p.table[instID].sub + geomID; end = p.table[instID].sub + p.table[instID].nprims; ok = geomID < p.table[instID].nprims; }
    }
    if (ok && slot < end) e = p.table[slot];
    const uint32_t kind = e.kind;
    InterpPrim s;
    bool valid = kind != INTERP_NONE && kind != INTERP_INSTANCE && primID < e.nprims;
    if (valid) {
      uint32_t idx[4] = {0, 0, 0, 0};
      const uint32_t* ip = reinterpret_cast<const uint32_t*>(e.idx + (uint64_t)primID * e.istride);
      const int ni = interp_index_count(kind);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k < ni) idx[k] = __ldg(ip + k);
      s = interp_prim(kind, e.basis, idx, u, v);
      // every element read must lie in its buffer
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (r < s.nrows) valid = valid && (uint64_t)s.row[r] < ((kind == INTERP_HERMITE && r >= 2) ? e.ntang : e.nelems);
    }
    if (!valid) {
      const float o[6] = {__int_as_float(0x7FC00000), __int_as_float(0x7FC00000), __int_as_float(0x7FC00000),
                          __int_as_float(0x7FC00000), __int_as_float(0x7FC00000), __int_as_float(0x7FC00000)};
      for (unsigned k = 0; k < V; ++k) store_value(p, (uint64_t)k * M + i, o);
      continue;
    }
    const uint8_t* rows[4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
      rows[r] = (kind == INTERP_HERMITE && r >= 2) ? e.tang + (uint64_t)s.row[r] * e.tstride : e.data + (uint64_t)s.row[r] * e.dstride;
    unsigned k = 0;
    // 16-byte loads where every row is 16-byte aligned
    const bool vec = ((reinterpret_cast<uintptr_t>(e.data) | e.dstride) & 15) == 0 &&
                     (kind != INTERP_HERMITE || ((reinterpret_cast<uintptr_t>(e.tang) | e.tstride) & 15) == 0);
    if (vec) {
      for (; k + 4 <= V; k += 4) {
        float4 q[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) q[r] = r < s.nrows ? __ldg(reinterpret_cast<const float4*>(rows[r] + 4ull * k)) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float c0[4] = {q[0].x, q[1].x, q[2].x, q[3].x}, c1[4] = {q[0].y, q[1].y, q[2].y, q[3].y};
        const float c2[4] = {q[0].z, q[1].z, q[2].z, q[3].z}, c3[4] = {q[0].w, q[1].w, q[2].w, q[3].w};
        float o[6];
        interp_value(kind, s, c0, o); store_value(p, (uint64_t)k * M + i, o);
        interp_value(kind, s, c1, o); store_value(p, (uint64_t)(k + 1) * M + i, o);
        interp_value(kind, s, c2, o); store_value(p, (uint64_t)(k + 2) * M + i, o);
        interp_value(kind, s, c3, o); store_value(p, (uint64_t)(k + 3) * M + i, o);
      }
    }
    for (; k < V; ++k) {
      float c[4] = {0.f, 0.f, 0.f, 0.f}, o[6];
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (r < s.nrows) c[r] = __ldg(reinterpret_cast<const float*>(rows[r]) + k);
      interp_value(kind, s, c, o);
      store_value(p, (uint64_t)k * M + i, o);
    }
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
