// record_tests.cuh -- the per-record pieces of the trace kernel that the device-side query functions
// (include/embree4_b200_device.cuh) share with it: the ray setup's reciprocal, the instance transform of the ray and the
// curve / point record tests.  Both include this one copy, so a record is tested by the same code whichever entry point
// traces it.
//
// The __noinline__ functions are also `inline`: a caller that compiles several translation units with -rdc=true gets one
// definition of each, not a duplicate symbol per unit.
#pragma once
#include "rtk_device.h"

namespace rtk {

// rcp_safe with the reference's own recipe: hardware approximation + one Newton step (common/simd/vfloat4_sse2.h:304-323)
// instead of an IEEE division: __frcp_rn is correctly rounded, the 1/dir error that node_hitmask's pads are derived for.
__device__ __forceinline__ float rcp_safe_fast(float d) {
  const float x = fabsf(d) < kMinRcpInput ? kMinRcpInput : d;
  const float r = __frcp_rn(x);
  return r;
}

// instanced scenes (kernels/geometry/instance_intersector.cpp:15-38): the records of an instance hold the OBJECT-space
// triangle; the ray is taken into that space with the instance's world2local exactly as the reference does before it
// traces the instanced scene (xfmPoint / xfmVector, affinespace.h:102-103) -- t is unchanged by the affine map, so the
// world-space BVH above and the object-space triangle test below share one parametrisation.
__device__ __forceinline__ void to_object_space(const GeomDesc& d, Ray& r) {
  const float ox = r.ox, oy = r.oy, oz = r.oz, dx = r.dx, dy = r.dy, dz = r.dz;
  r.ox = fma_rn(ox, d.w2l[0], fma_rn(oy, d.w2l[3], fma_rn(oz, d.w2l[6], d.w2l[9])));
  r.oy = fma_rn(ox, d.w2l[1], fma_rn(oy, d.w2l[4], fma_rn(oz, d.w2l[7], d.w2l[10])));
  r.oz = fma_rn(ox, d.w2l[2], fma_rn(oy, d.w2l[5], fma_rn(oz, d.w2l[8], d.w2l[11])));
  r.dx = fma_rn(dx, d.w2l[0], fma_rn(dy, d.w2l[3], mul_rn(dz, d.w2l[6])));
  r.dy = fma_rn(dx, d.w2l[1], fma_rn(dy, d.w2l[4], mul_rn(dz, d.w2l[7])));
  r.dz = fma_rn(dx, d.w2l[2], fma_rn(dy, d.w2l[5], mul_rn(dz, d.w2l[8])));
}

// round linear curve record (build.cu leaf_pack): a = (p0.xyz, primID), b = (p1.xyz, descriptor), c = (r0, r1, first vertex | flags << 30,
// mask).  The neighbour vertices -- needed to cut away what lies inside the adjacent segments -- come from the geometry's
// resident float4 vertex buffer (LineSegments::gather, scene_line_segments.h:270-276).
// round cubic curve (sweep intersector): its own function, so that its arrays and register needs stay out of the other curve tests
inline __device__ __noinline__ bool round_record_test(const GeomDesc& d, const Ray& r, float tfar, uint32_t vid, int lane, CurveHit& h) {
  CurveVtx cp[4];
  load_cubic_cp(d, vid, cp);
  return round_cubic_test(r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, r.tnear, tfar, cp, d.basis, h, lane);
}
inline __device__ __noinline__ bool curve_record_test(const GeomDesc& d, const Ray& r, float tfar, const uint4& a, const uint4& b, const uint4& c, CurveHit& h) {
  if (d.kind >= PRIM_SPHERE)   // point primitives (sphere / ray-facing disc / oriented disc): the record holds everything (build.cu leaf_pack)
    return point_test(r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, r.tnear, tfar, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z),
                      __uint_as_float(c.x), __uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z), (int)(d.kind - PRIM_SPHERE), h);
  if (d.kind == PRIM_ROUND_CUBIC) return round_record_test(d, r, tfar, c.z, (int)c.x, h);   // c.x: this record's first-level sub-segment
  if (d.kind == PRIM_FLAT_CUBIC) {   // flat cubic curve (Bezier / B-spline / Catmull-Rom / Hermite): control points from the resident vertex buffer
    CurveVtx cp[4];
    load_cubic_cp(d, c.z, cp);
    return flat_cubic_test(r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, r.tnear, tfar, cp, d.basis, (int)d.tess, d.basis_tab, h, (int)c.x);   // c.x: this record's segment
  }
  const CurveVtx v0{__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(c.x)};
  const CurveVtx v1{__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(c.y)};
  if (d.kind == PRIM_FLAT_LINEAR)   // RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE: ray-facing ribbon, no neighbours involved
    return flat_curve_test(r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, r.tnear, tfar, v0, v1, h);
  const uint32_t vid = c.z & 0x3FFFFFFFu;
  const bool hasL = (c.z >> 30) & 1u, hasR = (c.z >> 31) & 1u;
  CurveVtx vL = v0, vR = v1;
  if (hasL) { const float4 q = __ldg(reinterpret_cast<const float4*>(d.verts + (size_t)(vid - 1) * d.vstride)); vL = CurveVtx{q.x, q.y, q.z, q.w}; }
  if (hasR) { const float4 q = __ldg(reinterpret_cast<const float4*>(d.verts + (size_t)(vid + 2) * d.vstride)); vR = CurveVtx{q.x, q.y, q.z, q.w}; }
  return curve_test(r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, r.tnear, tfar, v0, v1, hasL, vL, hasR, vR, h);
}

}  // namespace rtk
