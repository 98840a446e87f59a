// interp.cuh -- vertex-data interpolation at (primID, u, v): rtcInterpolate's arithmetic, shared by the host entry points
// (rtcore_shim.cpp), the batched interpolation kernel (interpolate.cu) and the CPU emulator (tests/emu).
//
// Every operation is rounded explicitly (rt_core.cuh fma_rn / mul_rn / sub_rn / add_rn), so the host and the device
// instantiations give the same bits.  Reference semantics restated here (paths relative to the reference tree):
//   triangle / quad     kernels/common/scene_triangle_mesh.h:49-105, scene_quad_mesh.h interpolate_impl
//   linear curves       kernels/common/scene_line_segments.h:39-75
//   cubic curves        kernels/common/scene_curves.h:535-579 (Bezier / B-spline / Catmull-Rom), :699-761 (Hermite)
//   curve bases         kernels/subdiv/bezier_curve.h:12-51, :375-405; bspline_curve.h:11-50, :115-131;
//                       catmullrom_curve.h:20-58, :123-139; hermite_curve.h:19-20
// Triangle and quad meshes and linear curves are interpolated by code of the reference without FMA: their products and sums
// stay unfused.  Cubic curve geometries come from its AVX2 / AVX-512 builds (rtcore.cpp:1619-1622), where `madd` is a fused
// multiply-add: it is fma_rn here.  tests/test_interpolate_curves.py holds all of this to the reference's answers bit for bit.
#pragma once
#include "rt_core.cuh"

namespace rtk {

// what a geometry interpolates as (the kind of an interpolation table entry, InterpEntry below)
enum InterpKind : uint32_t {
  INTERP_NONE = 0,            // nothing to interpolate (points, missing buffer or slot): quiet NaN
  INTERP_TRIANGLE = 1,
  INTERP_QUAD = 2,
  INTERP_LINEAR = 3,          // round / flat linear curves
  INTERP_CUBIC = 4,           // Bezier / B-spline / Catmull-Rom curves, round or flat (`basis`)
  INTERP_HERMITE = 5,         // Hermite curve, RTC_BUFFER_TYPE_VERTEX: cubic Hermite of (p0, t0, p1, t1)
  INTERP_HERMITE_ATTRIB = 6,  // Hermite curve, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE: linear between index and index + 1
  INTERP_INSTANCE = 7,        // device table only: the hit's geomID indexes the instanced scene's sub-table
};
RT_HD constexpr bool interp_curve(uint32_t kind) { return kind >= INTERP_LINEAR && kind <= INTERP_HERMITE_ATTRIB; }
RT_HD constexpr int interp_index_count(uint32_t kind) { return kind == INTERP_TRIANGLE ? 3 : kind == INTERP_QUAD ? 4 : 1; }

// One entry of a scene's device interpolation table (rtcb200InterpolateHits*, rtcb200GetSceneDeviceInterpolator): one entry per
// geomID of the scene, then one block of entries per instanced scene: an INTERP_INSTANCE entry's `sub` is the first entry of its
// scene's block and `nprims` the block's length, so a hit resolves in at most two lookups.  Buffers are device copies (stride honoured).
struct InterpEntry {
  uint32_t kind = 0;             // InterpKind
  uint32_t basis = 0;            // INTERP_CUBIC: CurveBasis
  uint32_t nprims = 0;           // primitives (INTERP_INSTANCE: entries of the sub-table)
  uint32_t sub = 0;              // INTERP_INSTANCE: first entry of the sub-table
  const uint8_t* idx = nullptr;  // index buffer
  const uint8_t* data = nullptr; // the requested vertex / attribute buffer
  const uint8_t* tang = nullptr; // INTERP_HERMITE: the tangent buffer
  uint64_t istride = 0, dstride = 0, tstride = 0;
  uint64_t nelems = 0, ntang = 0;   // elements of the data / tangent buffer: an index beyond them gives NaN, not a wild read
};

// One primitive at (u, v): the buffer elements its control values come from and the weights they are combined with.
// row[0..3]: element indices into the requested buffer, except for INTERP_HERMITE, whose row[2], row[3] index the tangent
// buffer (t0, t1).  nrows: how many of them are read.
struct InterpPrim {
  uint32_t row[4];
  int nrows;
  float u, v, w;              // triangle / quad: barycentrics of the half the point lies in; curves: u
  bool left;                  // quad: the point lies in the (v0, v1, v3) half
  float b[4], d[4], dd[4];    // cubic curves: basis, first and second derivative weights at u
};

// Basis, first and second derivative weights at u (BezierBasis / BSplineBasis / CatmullRomBasis ::eval, ::derivative, ::derivative2)
// as the reference's AVX2 build of the curve geometries evaluates them: its compiler contracts a product into the sum that is its only
// use, so the B-spline and Catmull-Rom weights below carry exactly those fused multiply-adds.  The Bezier weights and the B-spline
// derivatives are rt_core.cuh's, where no contraction changes a result (products by 2 and 4 are exact).
RT_HD void interp_basis(uint32_t basis, float u, float b[4], float d[4], float dd[4]) {
  const float t = u, s = sub_rn(1.0f, u);
  if (basis == BASIS_BEZIER) {
    float unused[4];
    curve_basis_table_entry(basis, u, b, unused);
    curve_basis_derivative(basis, u, d);
    curve_basis_derivative2(basis, u, dd);
  } else if (basis == BASIS_BSPLINE) {
    const float sss = mul_rn(mul_rn(s, s), s), ttt = mul_rn(mul_rn(t, t), t), st = mul_rn(s, t), sts = mul_rn(st, s), tst = mul_rn(st, t);
    const float k = 1.0f / 6.0f;
    b[0] = mul_rn(k, sss);
    b[1] = mul_rn(k, add_rn(fma_rn(4.0f, sss, ttt), fma_rn(12.0f, sts, mul_rn(6.0f, tst))));
    b[2] = mul_rn(k, add_rn(fma_rn(4.0f, ttt, sss), fma_rn(12.0f, tst, mul_rn(6.0f, sts))));
    b[3] = mul_rn(k, ttt);
    curve_basis_derivative(basis, u, d);
    curve_basis_derivative2(basis, u, dd);
  } else {
    // P and the derivatives are evaluated in one function there, which shares 3t, 3s, t*t and s*s between the three sets of
    // weights: a shared product is not fused.  (When a call asks for the derivatives without P, the reference fuses the derivative
    // weights differently and its last bits can differ from these.)
    const float t3 = mul_rn(3.0f, t), s3 = mul_rn(3.0f, s), tt = mul_rn(t, t), ss = mul_rn(s, s), s2 = add_rn(s, s), t2 = add_rn(t, t);
    b[0] = mul_rn(0.5f, mul_rn(mul_rn(-t, s), s));
    b[1] = mul_rn(0.5f, fma_rn(tt, sub_rn(t3, 5.0f), 2.0f));
    b[2] = mul_rn(0.5f, fma_rn(ss, sub_rn(s3, 5.0f), 2.0f));
    b[3] = mul_rn(0.5f, mul_rn(mul_rn(-s, t), t));
    d[0] = mul_rn(0.5f, fma_rn(s2, t, -ss));
    d[1] = mul_rn(0.5f, fma_rn(t2, sub_rn(t3, 5.0f), mul_rn(t, t3)));
    d[2] = mul_rn(0.5f, fma_rn(s2, add_rn(t3, 2.0f), -mul_rn(s, s3)));
    d[3] = mul_rn(0.5f, fma_rn(-s2, t, tt));
    dd[0] = sub_rn(2.0f, t3); dd[1] = fma_rn(9.0f, t, -5.0f); dd[2] = fma_rn(-9.0f, t, 4.0f); dd[3] = sub_rn(t3, 1.0f);
  }
}

// `idx` points at the primitive's entry of the index buffer (3, 4 or 1 unsigned ints, interp_index_count).
RT_HD InterpPrim interp_prim(uint32_t kind, uint32_t basis, const uint32_t* idx, float u, float v) {
  InterpPrim s;
  s.u = u; s.v = v; s.w = 0.0f; s.left = true;
  for (int k = 0; k < 4; ++k) { s.row[k] = 0; s.b[k] = s.d[k] = s.dd[k] = 0.0f; }
  if (kind == INTERP_TRIANGLE || kind == INTERP_QUAD) {
    s.nrows = 3;
    s.row[0] = idx[0]; s.row[1] = idx[1]; s.row[2] = idx[2];
    if (kind == INTERP_QUAD) {   // the (v0,v1,v3) half, or the (v2,v3,v1) half with (1-u, 1-v)
      s.left = add_rn(u, v) <= 1.0f;
      s.row[0] = s.left ? idx[0] : idx[2]; s.row[1] = s.left ? idx[1] : idx[3]; s.row[2] = s.left ? idx[3] : idx[1];
      if (!s.left) { s.u = sub_rn(1.0f, u); s.v = sub_rn(1.0f, v); }
    }
    s.w = sub_rn(sub_rn(1.0f, s.u), s.v);
    return s;
  }
  const uint32_t i = idx[0];
  if (kind == INTERP_CUBIC) {
    s.nrows = 4;
    for (int k = 0; k < 4; ++k) s.row[k] = i + k;
  } else {
    s.nrows = kind == INTERP_HERMITE ? 4 : 2;
    s.row[0] = i; s.row[1] = i + 1; s.row[2] = i; s.row[3] = i + 1;
  }
  if (kind == INTERP_CUBIC || kind == INTERP_HERMITE)   // a Hermite curve is evaluated as its Bezier control points
    interp_basis(kind == INTERP_HERMITE ? (uint32_t)BASIS_BEZIER : basis, u, s.b, s.d, s.dd);
  return s;
}

// madd(b.x, v0, madd(b.y, v1, madd(b.z, v2, b.w * v3))) (bezier_curve.h:393-405 and the B-spline / Catmull-Rom twins)
RT_HD float interp_blend(const float w[4], float p0, float p1, float p2, float p3) {
  return fma_rn(w[0], p0, fma_rn(w[1], p1, fma_rn(w[2], p2, mul_rn(w[3], p3))));
}

// One component.  p[r] = the component of element row[r] (INTERP_HERMITE: p0, p1, t0, t1).  o = P, dPdu, dPdv, ddPdudu,
// ddPdvdv, ddPdudv; a curve's v-derivatives are 0.
RT_HD void interp_value(uint32_t kind, const InterpPrim& s, const float p[4], float o[6]) {
  o[2] = o[4] = o[5] = 0.0f;
  if (kind == INTERP_TRIANGLE || kind == INTERP_QUAD) {
    // madd(w, p0, madd(u, p1, v * p2)) of the AVX build: unfused
    o[0] = add_rn(mul_rn(s.w, p[0]), add_rn(mul_rn(s.u, p[1]), mul_rn(s.v, p[2])));
    o[1] = s.left ? sub_rn(p[1], p[0]) : sub_rn(p[0], p[1]);
    o[2] = s.left ? sub_rn(p[2], p[0]) : sub_rn(p[0], p[2]);
    o[3] = 0.0f;
    return;
  }
  if (kind == INTERP_LINEAR) {   // lerp(p0, p1, u) = madd(u, p1 - p0, p0) (vfloat4_sse2.h:543-545), of a build without FMA: unfused
    const float e = sub_rn(p[1], p[0]);
    o[0] = add_rn(mul_rn(s.u, e), p[0]); o[1] = e;
    // The reference writes this zero into dPdu instead (scene_line_segments.h:73), which loses dPdu whenever ddPdudu is
    // requested and leaves ddPdudu unwritten.  The second derivative of a line is zero, and that is what ddPdudu gets here.
    o[3] = 0.0f;
    return;
  }
  if (kind == INTERP_HERMITE_ATTRIB) {   // madd(1-u, p0, u*p1) (scene_curves.h:721)
    o[0] = fma_rn(sub_rn(1.0f, s.u), p[0], mul_rn(s.u, p[1])); o[1] = sub_rn(p[1], p[0]); o[3] = 0.0f;
    return;
  }
  float c0 = p[0], c1 = p[1], c2 = p[2], c3 = p[3];
  if (kind == INTERP_HERMITE) {   // Bezier control points (v0, madd(1/3, t0, v0), nmadd(1/3, t1, v1), v1) (hermite_curve.h:19-20)
    const float k = 1.0f / 3.0f;
    c0 = p[0]; c1 = fma_rn(k, p[2], p[0]); c2 = fma_rn(-k, p[3], p[1]); c3 = p[1];
  }
  o[0] = interp_blend(s.b, c0, c1, c2, c3);
  o[1] = interp_blend(s.d, c0, c1, c2, c3);
  o[3] = interp_blend(s.dd, c0, c1, c2, c3);
}

// rtcInterpolate of one primitive from host-visible buffers: `data` / `dstride` the requested buffer, `tang` / `tstride` the
// tangent buffer of a Hermite curve (its own stride: the reference reads tangents with the vertex buffer's stride,
// scene_curves.h:739, which is out of bounds when the two differ).  out[c] (P, dPdu, dPdv, ddPdudu, ddPdvdv, ddPdudv; NULL =
// not wanted) receives value k at out[c][k * ostride].
RT_HD void interpolate_prim(uint32_t kind, uint32_t basis, const uint32_t* idx, const uint8_t* data, uint64_t dstride, const uint8_t* tang,
                            uint64_t tstride, float u, float v, unsigned valueCount, float* const out[6], uint64_t ostride) {
  const InterpPrim s = interp_prim(kind, basis, idx, u, v);
  const uint8_t* rows[4];
  for (int r = 0; r < 4; ++r)
    rows[r] = (kind == INTERP_HERMITE && r >= 2) ? tang + (uint64_t)s.row[r] * tstride : data + (uint64_t)s.row[r] * dstride;
  for (unsigned k = 0; k < valueCount; ++k) {
    float p[4] = {0.0f, 0.0f, 0.0f, 0.0f}, o[6];
    for (int r = 0; r < s.nrows; ++r) p[r] = reinterpret_cast<const float*>(rows[r])[k];
    interp_value(kind, s, p, o);
    for (int c = 0; c < 6; ++c)
      if (out[c]) out[c][(uint64_t)k * ostride] = o[c];
  }
}

#if defined(__CUDACC__)
// One hit of the device interpolation: the batched kernel (interpolate.cu) and rtcb200Interpolate1 (include/embree4_b200_device.cuh)
// both run this body; only where value k goes differs, so `store(k, o)` writes the six outputs o (P, dPdu, dPdv, ddPdudu, ddPdvdv,
// ddPdudv) of value k.  The hit is geometry geomID of the table's scene, or, with instID valid, geometry geomID of the scene
// instance instID instantiates.  Points, instances, a missing buffer or slot and an index beyond a buffer store quiet NaN.
template <typename Store>
__device__ __forceinline__ void interpolate_hit(const InterpEntry* table,uint32_t nentries, uint32_t geomID, uint32_t instID,
                                                uint32_t primID, float u, float v, unsigned V, Store store) {
  // resolve the entry: the scene's own geometry, or geometry geomID of the scene instance instID instantiates
  InterpEntry e;
  e.kind = INTERP_NONE;
  uint32_t slot = geomID, end = nentries;
  bool ok = true;
  if (instID != kInvalidID) {
    ok = instID < nentries && table[instID].kind == INTERP_INSTANCE;
    if (ok) { slot = table[instID].sub + geomID; end = table[instID].sub + table[instID].nprims; ok = geomID < table[instID].nprims; }
  }
  if (ok && slot < end) e = table[slot];
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
    for (unsigned k = 0; k < V; ++k) store(k, o);
    return;
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
      interp_value(kind, s, c0, o); store(k, o);
      interp_value(kind, s, c1, o); store(k + 1, o);
      interp_value(kind, s, c2, o); store(k + 2, o);
      interp_value(kind, s, c3, o); store(k + 3, o);
    }
  }
  for (; k < V; ++k) {
    float c[4] = {0.f, 0.f, 0.f, 0.f}, o[6];
#pragma unroll
    for (int r = 0; r < 4; ++r)
      if (r < s.nrows) c[r] = __ldg(reinterpret_cast<const float*>(rows[r]) + k);
    interp_value(kind, s, c, o);
    store(k, o);
  }
}
#endif

}  // namespace rtk
