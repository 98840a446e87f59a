// transform_format.cuh -- how an instance transform is written out in each RTCFormat (storeTransform, kernels/common/rtcore.h:125-155).
// One definition for the host entry points (rtcGetGeometryTransform*, rtcore_shim.cpp) and the device-side
// rtcb200GetGeometryTransformFromTraversable (include/embree4_b200_device.cuh), so both give the same bytes.  Plain C++ with no
// other include: the public device header reaches it by relative path, and a host compiler can instantiate it on its own.
#pragma once

#if defined(__CUDACC__)
#define RTK_TF_HD __host__ __device__ __forceinline__
#else
#define RTK_TF_HD inline
#endif

namespace rtk {

// m = the local-to-world columns vx | vy | vz | p (AffineSpace3fa).  Writes 12 floats (FLOAT3X4_ROW_MAJOR 0x9134,
// FLOAT3X4_COLUMN_MAJOR 0x9234) or 16 (FLOAT4X4_COLUMN_MAJOR 0x9244) to x; any other format writes nothing and returns false.
RTK_TF_HD bool store_transform(const float m[12], unsigned format, float* x) {
  switch (format) {
    case 0x9134:
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) x[4 * r + c] = m[3 * c + r];
      return true;
    case 0x9234:
      for (int k = 0; k < 12; ++k) x[k] = m[k];
      return true;
    case 0x9244:
      for (int c = 0; c < 4; ++c) {
        for (int r = 0; r < 3; ++r) x[4 * c + r] = m[3 * c + r];
        x[4 * c + 3] = c == 3 ? 1.0f : 0.0f;
      }
      return true;
    default:
      return false;
  }
}

}  // namespace rtk
