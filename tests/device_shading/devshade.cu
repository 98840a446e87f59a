// TEST TOOL: kernels that shade from device code through include/embree4_b200_device.cuh -- user data, instance transforms and
// rtcb200Interpolate1 -- compiled as a user would (build.sh: nvcc for sm_90a, default floating-point flags, -I include only).
// tests/test_device_shading.py and scripts/device_shading_bench.py drive the extern "C" launchers with ctypes.
#include <cuda_runtime.h>
#include <stdint.h>

#include "embree4_b200.h"
#include "embree4_b200_device.cuh"

namespace {

constexpr int kThreads = 128;

// rtcb200Interpolate1 of hit i, value k of output c at out[c][i * vc + k] (NULL outputs skipped)
__device__ void interpolate_record(const RTCB200DeviceInterpolator& ip, const RTCRayHit& rh, size_t i, unsigned vc, float* const* out) {
  RTCB200DeviceInterpolateArguments a;
  a.geomID = rh.hit.geomID; a.instID = rh.hit.instID[0]; a.primID = rh.hit.primID; a.u = rh.hit.u; a.v = rh.hit.v;
  float** o[6] = {&a.P, &a.dPdu, &a.dPdv, &a.ddPdudu, &a.ddPdvdv, &a.ddPdudv};
  for (int c = 0; c < 6; ++c) *o[c] = out[c] ? out[c] + i * vc : nullptr;
  a.valueCount = vc;
  rtcb200Interpolate1(ip, &a);
}

struct Outputs { float* p[6]; };

// (a) one thread per traced hit
__global__ void interpolate_kernel(const RTCB200DeviceInterpolator ip, const RTCRayHit* rh, size_t n, unsigned vc, Outputs out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) interpolate_record(ip, rh[i], i, vc, out.p);
}

// (b) trace and interpolate in one thread
__global__ void trace_interpolate_kernel(const RTCB200DeviceTraversable t, const RTCB200DeviceInterpolator ip, RTCRayHit* rh, size_t n,
                                         unsigned vc, Outputs out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RTCRayHit q = rh[i];
  rtcb200TraversableIntersect1(t, &q);
  rh[i] = q;
  interpolate_record(ip, q, i, vc, out.p);
}

__global__ void user_data_kernel(const RTCB200DeviceTraversable t, const unsigned* ids, size_t n, unsigned long long* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (unsigned long long)(uintptr_t)rtcb200GetGeometryUserDataFromTraversable(t, ids[i]);
}

__global__ void transform_kernel(const RTCB200DeviceTraversable t, const unsigned* ids, size_t n, unsigned format, float* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rtcb200GetGeometryTransformFromTraversable(t, ids[i], 0.5f, (RTCFormat)format, out + 16 * i);
}

// ---- the shading workload of scripts/device_shading_bench.py ---------------------------------------------------------------
// object-space normal n of a hit to world space through instance instID (identity when it is not instanced), normalised;
// the one definition both paths use, so their outputs can be compared bit for bit
__device__ __forceinline__ void world_normal(const RTCB200DeviceTraversable& t, unsigned instID, const float n[3], float* w) {
  float x[12];
  rtcb200GetGeometryTransformFromTraversable(t, instID, 0.0f, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, x);
  float r[3];
  for (int k = 0; k < 3; ++k) r[k] = __fmaf_rn(x[k], n[0], __fmaf_rn(x[3 + k], n[1], __fmul_rn(x[6 + k], n[2])));
  const float s = rsqrtf(__fmaf_rn(r[0], r[0], __fmaf_rn(r[1], r[1], __fmul_rn(r[2], r[2]))));
  for (int k = 0; k < 3; ++k) w[k] = __fmul_rn(r[k], s);
}

// megakernel: trace, interpolate the normal from attribute slot `ip`, bring it to world space, write it (misses: zero)
__global__ void shade_kernel(const RTCB200DeviceTraversable t, const RTCB200DeviceInterpolator ip, const RTCRayHit* rh, size_t n, float* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RTCRayHit q = rh[i];
  rtcb200TraversableIntersect1(t, &q);
  float w[3] = {0.0f, 0.0f, 0.0f};
  if (q.hit.geomID != RTC_INVALID_GEOMETRY_ID) {
    float nrm[3];
    RTCB200DeviceInterpolateArguments a = {};
    a.geomID = q.hit.geomID; a.instID = q.hit.instID[0]; a.primID = q.hit.primID; a.u = q.hit.u; a.v = q.hit.v;
    a.P = nrm; a.valueCount = 3;
    rtcb200Interpolate1(ip, &a);
    world_normal(t, q.hit.instID[0], nrm, w);
  }
  for (int k = 0; k < 3; ++k) out[3 * i + k] = w[k];
}

// the batched path's last step: normals interpolated by rtcb200InterpolateHitsDevice ([3][n]) to world space
__global__ void transform_normals_kernel(const RTCB200DeviceTraversable t, const RTCRayHit* rh, const float* P, size_t n, float* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned geomID = rh[i].hit.geomID, instID = rh[i].hit.instID[0];
  float w[3] = {0.0f, 0.0f, 0.0f};
  if (geomID != RTC_INVALID_GEOMETRY_ID) {
    const float nrm[3] = {P[i], P[n + i], P[2 * n + i]};
    world_normal(t, instID, nrm, w);
  }
  for (int k = 0; k < 3; ++k) out[3 * i + k] = w[k];
}

unsigned blocks_for(size_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

extern "C" {

int devshade_interpolate(const RTCB200DeviceInterpolator* ip, int device, const RTCRayHit* d_rh, size_t n, unsigned vc, float* const out[6],
                         void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(device);
  Outputs o;
  for (int c = 0; c < 6; ++c) o.p[c] = out[c];
  interpolate_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*ip, d_rh, n, vc, o);
  return (int)cudaGetLastError();
}
int devshade_trace_interpolate(const RTCB200DeviceTraversable* t, const RTCB200DeviceInterpolator* ip, RTCRayHit* d_rh, size_t n, unsigned vc,
                               float* const out[6], void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  Outputs o;
  for (int c = 0; c < 6; ++c) o.p[c] = out[c];
  trace_interpolate_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, *ip, d_rh, n, vc, o);
  return (int)cudaGetLastError();
}
int devshade_user_data(const RTCB200DeviceTraversable* t, const unsigned* d_ids, size_t n, unsigned long long* d_out, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  user_data_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_ids, n, d_out);
  return (int)cudaGetLastError();
}
int devshade_transform(const RTCB200DeviceTraversable* t, const unsigned* d_ids, size_t n, unsigned format, float* d_out, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  transform_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_ids, n, format, d_out);
  return (int)cudaGetLastError();
}
int devshade_shade(const RTCB200DeviceTraversable* t, const RTCB200DeviceInterpolator* ip, const RTCRayHit* d_rh, size_t n, float* d_out, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  shade_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, *ip, d_rh, n, d_out);
  return (int)cudaGetLastError();
}
int devshade_transform_normals(const RTCB200DeviceTraversable* t, const RTCRayHit* d_rh, const float* d_P, size_t n, float* d_out, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  transform_normals_kernel<<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_rh, d_P, n, d_out);
  return (int)cudaGetLastError();
}

}  // extern "C"
