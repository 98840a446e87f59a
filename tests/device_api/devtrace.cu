// TEST TOOL: kernels that trace from device code through include/embree4_b200_device.cuh, compiled as a user would
// (build.sh: nvcc for sm_90a, default floating-point flags, -I include only).  tests/test_device_traversal.py drives the
// extern "C" launchers with ctypes and compares their records with the batched entry points'.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "embree4_b200.h"
#include "embree4_b200_device.cuh"

namespace {

constexpr int kThreads = 128;

// (a) one thread per ray, straight on the caller's global records
__global__ void intersect_kernel(const RTCB200DeviceTraversable t, RTCRayHit* rh, size_t n, const RTCIntersectArguments* args) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rtcb200TraversableIntersect1(t, rh + i, args);
}
__global__ void occluded_kernel(const RTCB200DeviceTraversable t, RTCRay* r, size_t n, const RTCOccludedArguments* args) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rtcb200TraversableOccluded1(t, r + i, args);
}

__device__ uint32_t hash32(uint32_t x) {   // lowbias32
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__device__ float unit(uint32_t h) { return (float)(h >> 8) * (1.0f / 16777216.0f); }

// (b) two queries per thread on a copy of the ray in the thread's own memory: trace, form a secondary ray at the hit point
// (P = org + tfar * dir; from the origin on a miss) in a hashed direction, write it out, trace it, write its result
__global__ void two_query_kernel(const RTCB200DeviceTraversable t, RTCRayHit* rh, RTCRayHit* sec_in, RTCRayHit* sec_out, size_t n,
                                 uint32_t seed, float eps) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RTCRayHit q = rh[i];
  rtcb200TraversableIntersect1(t, &q);
  rh[i] = q;
  const bool hit = q.hit.geomID != RTC_INVALID_GEOMETRY_ID;
  const float s = hit ? q.ray.tfar : 0.0f;
  RTCRayHit b;
  memset(&b, 0, sizeof b);   // the record's padding too: it is compared byte for byte
  b.ray.org_x = __fmaf_rn(s, q.ray.dir_x, q.ray.org_x);
  b.ray.org_y = __fmaf_rn(s, q.ray.dir_y, q.ray.org_y);
  b.ray.org_z = __fmaf_rn(s, q.ray.dir_z, q.ray.org_z);
  const uint32_t h = hash32(seed ^ hash32((uint32_t)i));
  b.ray.dir_x = __fsub_rn(2.0f * unit(hash32(h + 1u)), 1.0f);
  b.ray.dir_y = __fsub_rn(2.0f * unit(hash32(h + 2u)), 1.0f);
  b.ray.dir_z = __fsub_rn(2.0f * unit(hash32(h + 3u)), 1.0f);
  b.ray.tnear = eps; b.ray.time = 0.0f; b.ray.tfar = INFINITY;
  b.ray.mask = 0xFFFFFFFFu; b.ray.id = (unsigned)i; b.ray.flags = 0u;
  b.hit.Ng_x = b.hit.Ng_y = b.hit.Ng_z = 0.0f; b.hit.u = b.hit.v = 0.0f;
  b.hit.primID = b.hit.geomID = RTC_INVALID_GEOMETRY_ID;
  b.hit.instID[0] = b.hit.instPrimID[0] = RTC_INVALID_GEOMETRY_ID;
  sec_in[i] = b;
  rtcb200TraversableIntersect1(t, &b);
  sec_out[i] = b;
}

// (c) even lanes intersect, odd lanes test occlusion, in the same warp, on records staged in shared memory
__global__ void mixed_kernel(const RTCB200DeviceTraversable t, RTCRayHit* rh, size_t n) {
  __shared__ RTCRayHit s[kThreads];
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  s[threadIdx.x] = rh[i];
  if (i & 1) rtcb200TraversableOccluded1(t, &s[threadIdx.x].ray);
  else rtcb200TraversableIntersect1(t, &s[threadIdx.x]);
  rh[i] = s[threadIdx.x];
}

unsigned blocks_for(size_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

extern "C" {

int devtrace_intersect(const RTCB200DeviceTraversable* t, RTCRayHit* d_rh, size_t n, const RTCIntersectArguments* d_args, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  intersect_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_rh, n, d_args);
  return (int)cudaGetLastError();
}
int devtrace_occluded(const RTCB200DeviceTraversable* t, RTCRay* d_r, size_t n, const RTCOccludedArguments* d_args, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  occluded_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_r, n, d_args);
  return (int)cudaGetLastError();
}
int devtrace_two_query(const RTCB200DeviceTraversable* t, RTCRayHit* d_rh, RTCRayHit* d_sec_in, RTCRayHit* d_sec_out, size_t n, unsigned seed,
                       float eps, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  two_query_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_rh, d_sec_in, d_sec_out, n, seed, eps);
  return (int)cudaGetLastError();
}
int devtrace_mixed(const RTCB200DeviceTraversable* t, RTCRayHit* d_rh, size_t n, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  mixed_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_rh, n);
  return (int)cudaGetLastError();
}

}  // extern "C"
