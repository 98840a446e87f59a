// record_tests.cuh -- the per-record rules of every ray query, shared by the trace kernel (trace.cu) and the device-side
// query functions (include/embree4_b200_device.cuh): the ray setup's reciprocal, the instance transform of the ray, the
// record test (masks, curve / point and triangle tests, finalize, the SPREAD acceptance rule), the hit write-back and which
// GENERAL specialisation a scene runs.  Both include this one copy, so a record is tested and reported by the same code
// whichever entry point traces it; the one exception is the trace kernel's warp-wide SPREAD step, which writes
// spread_record_test out for speed.
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
// `d` is a GeomDesc, or the InstRec of instance traversal (trace.cu, INST), which applies the same map when a ray enters an instance.
template <typename Xfm>
__device__ __forceinline__ void to_object_space(const Xfm& d, Ray& r) {
  const float ox = r.ox, oy = r.oy, oz = r.oz, dx = r.dx, dy = r.dy, dz = r.dz;
  r.ox = fma_rn(ox, d.w2l[0], fma_rn(oy, d.w2l[3], fma_rn(oz, d.w2l[6], d.w2l[9])));
  r.oy = fma_rn(ox, d.w2l[1], fma_rn(oy, d.w2l[4], fma_rn(oz, d.w2l[7], d.w2l[10])));
  r.oz = fma_rn(ox, d.w2l[2], fma_rn(oy, d.w2l[5], fma_rn(oz, d.w2l[8], d.w2l[11])));
  r.dx = fma_rn(dx, d.w2l[0], fma_rn(dy, d.w2l[3], mul_rn(dz, d.w2l[6])));
  r.dy = fma_rn(dx, d.w2l[1], fma_rn(dy, d.w2l[4], mul_rn(dz, d.w2l[7])));
  r.dz = fma_rn(dx, d.w2l[2], fma_rn(dy, d.w2l[5], mul_rn(dz, d.w2l[8])));
}

// Record layouts: build.cu pack_triangle / pack_linear / pack_cubic / pack_point.  A round linear curve's neighbour vertices -- needed
// to cut away what lies inside the adjacent segments -- come from the geometry's resident float4 vertex buffer (LineSegments::gather,
// scene_line_segments.h:270-276).
// round cubic curve (sweep intersector): its own function, so that its arrays and register needs stay out of the other curve tests
inline __device__ __noinline__ bool round_record_test(const GeomDesc& d, const Ray& r, float tfar, uint32_t vid, int lane, CurveHit& h) {
  CurveVtx cp[4];
  load_cubic_cp(d, vid, cp);
  return round_cubic_test(r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, r.tnear, tfar, cp, d.basis, h, lane);
}
inline __device__ __noinline__ bool curve_record_test(const GeomDesc& d, const Ray& r, float tfar, const uint4& a, const uint4& b, const uint4& c, CurveHit& h) {
  if (d.kind >= PRIM_SPHERE)   // point primitives (sphere / ray-facing disc / oriented disc): the record holds everything (build.cu pack_point)
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

// Which specialisation a scene's records take: 0 = triangle records with geomIDs, 1 = records through descriptors (instances,
// quads), 2 = with curve or point records among them (kept apart: the curve tests cost registers).
__host__ __device__ constexpr int general_of(const void* descs, unsigned curves) { return !descs ? 0 : (curves ? 2 : 1); }

// The SPREAD rule for one Moeller-Trumbore triangle record (a, b, c) of a GENERAL 0 scene: the ray mask, the test against the ray's
// own tfar `own_tfar` (not the hit so far), then finalize() -- t, u, v = T, U, V * rcp(absDen) -- and acceptance when t <= `best`,
// the hit so far.  The winner is then the smallest t over all tested records, whatever order or batches they are tested in, which
// is what lets the SPREAD kernel's warp test the records of several rays together (its warp-wide step in trace.cu writes this
// rule out: called from there, it slows that kernel).  An accepted record writes u, v, calls commit(t) and returns true, all where
// it was accepted (see record_test).  HIT = false: the verdict of the mask and the test only; u, v are not written and commit gets 0.
template <bool HIT, typename Commit>
__device__ __forceinline__ bool spread_record_test(const Ray& r, uint32_t mask, float own_tfar, const uint4& a, const uint4& b, const uint4& c,
                                                   float best, float& u, float& v, const Commit& commit) {
  TriHit th;
  if (!((c.w & mask) != 0 &&
        tri_test(r, own_tfar, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(b.x), __uint_as_float(b.y),
                 __uint_as_float(b.z), __uint_as_float(c.x), __uint_as_float(c.y), __uint_as_float(c.z), th)))
    return false;
  if (!HIT) {
    commit(0.0f);
    return true;
  }
  const float rcpAbsDen = 1.0f / th.absDen;
  const float t = th.T * rcpAbsDen;
  if (!(t <= best)) return false;
  u = th.U * rcpAbsDen; v = th.V * rcpAbsDen;
  commit(t);
  return true;
}

// An accepted record's candidate besides its u, v: t and, for a curve / point record (curve = true), the normal its test found.
// The round cubic test is an iteration whose result depends on the tfar it started from, so that normal is kept from the winning
// test instead of being recomputed at write-back.
struct RecordHit { float t, ngx, ngy, ngz; bool curve; };

// One leaf record (a, b, c) against the world-space ray r, `tfar` being the current hit distance.  In order: the ray mask
// (intersector_epilog.h:256-262); GENERAL: b.w is a descriptor index -- the instance mask (instance_intersector.cpp:19-22), the
// object-space ray (t is unchanged), and for GENERAL == 2 the curve / point tests; then the triangle test, Pluecker (ROBUST) or
// Moeller-Trumbore, its finalize and the quad's second-half u / v swap.
// An accepted record writes its u, v to `u`, `v`, is then handed to `commit(const RecordHit&)`, and record_test returns true.  Both
// happen where the record was accepted: committing after a merged return makes the compiler select between the old and the new hit
// state, which costs the callers registers, and u, v are stored as they are computed, as the trace kernel's shared-memory copies of
// them want.
//  - HIT = false (any hit without a filter): only the verdict; u, v are not written and commit's argument holds nothing.
//  - SPREAD (Moeller-Trumbore closest hit over GENERAL 0 records): spread_record_test with the ray's own r.tfar and `tfar` as the
//    hit so far.  Without it the test runs against tfar and nothing is checked after the division; folding the two rules together
//    would change results.
template <bool ROBUST, int GENERAL, bool HIT, bool SPREAD, typename Commit>
__device__ __forceinline__ bool record_test(const GeomDesc* __restrict__ descs, const uint4& a, const uint4& b, const uint4& c, Ray r,
                                            float tfar, float& u, float& v, const Commit& commit) {
  static_assert(!SPREAD || (!ROBUST && GENERAL == 0), "the SPREAD rule is that of Moeller-Trumbore triangle scenes");
  RecordHit h;
  if (SPREAD) return spread_record_test<HIT>(r, r.mask, r.tfar, a, b, c, tfar, u, v, [&](float t) { h.t = t; h.curve = false; commit(h); });
  bool visible = (c.w & r.mask) != 0;
  if (GENERAL) {
    const GeomDesc& d = descs[b.w];
    visible = visible && (d.inst_mask & r.mask) != 0;
    if (d.has_xfm) to_object_space(d, r);
    if (GENERAL == 2 && d.kind != PRIM_TRIANGLE) {
      CurveHit ch;
      if (!(visible && curve_record_test(d, r, tfar, a, b, c, ch))) return false;
      if (HIT) { h.t = ch.t; u = ch.u; v = ch.v; h.ngx = ch.ngx; h.ngy = ch.ngy; h.ngz = ch.ngz; h.curve = true; }
      commit(h);
      return true;
    }
  }
  if (!visible) return false;
  h.curve = false;
  if (ROBUST) {   // RTC_SCENE_FLAG_ROBUST: the record holds v0, v1, v2; watertight Pluecker test
    PlueckerHit ph;
    if (!tri_test_pluecker(r, tfar, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(b.x),
                           __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(c.x), __uint_as_float(c.y), __uint_as_float(c.z), ph))
      return false;
    if (HIT) {
      h.t = ph.t; pluecker_uv(ph, u, v);
      if (GENERAL && (a.w >> 31)) {   // second half of a quad (QuadHitPlueckerM::finalize, AVX form)
        const float u1 = sub_rn(1.0f, u), v1 = sub_rn(1.0f, v);
        u = v1; v = u1;
      }
    }
    commit(h);
    return true;
  }
  TriHit th;
  if (!tri_test(r, tfar, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(b.x),
                __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(c.x), __uint_as_float(c.y), __uint_as_float(c.z), th))
    return false;
  if (HIT) {
    const float rcpAbsDen = 1.0f / th.absDen;   // finalize(): t,u,v = T,U,V * rcp(absDen)
    h.t = th.T * rcpAbsDen;
    if (GENERAL && (a.w >> 31)) {   // second half of a quad: U' = absDen - V, V' = absDen - U (quad_intersector_moeller.h:196-198)
      u = sub_rn(th.absDen, th.V) * rcpAbsDen; v = sub_rn(th.absDen, th.U) * rcpAbsDen;
    } else { u = th.U * rcpAbsDen; v = th.V * rcpAbsDen; }
  }
  commit(h);
  return true;
}

// The hit that winning record ti reports at (u, v) (intersector_epilog.h:285-299; hit.t is the caller's): primID and geomID, through
// the descriptor for GENERAL; Ng in OBJECT space, as in the reference -- Moeller-Trumbore: cross(e2, e1) of the record, ROBUST: the
// stable normal of the origin-relative edges exactly as tri_test_pluecker computes it, a curve / point record: `curve_normal()`, the
// normal its test kept; a quad's second half reports the quad's primID with flipped winding.  instID / instPrimID come in as the
// caller's and become the instance's for an instanced record.
// `world_ray()` returns the world-space ray and `curve_normal()` a float3.  Only their branches call them for more than the ray's
// origin, so a caller that parks the ray's direction or the normal in memory loads it only when it is needed; u and v are taken by
// reference for the same reason, and read after the record.
template <bool ROBUST, int GENERAL, typename WorldRay, typename CurveNormal>
__device__ __forceinline__ void record_write_back(const uint4* __restrict__ recs, const GeomDesc* __restrict__ descs, uint32_t ti,
                                                  const WorldRay& world_ray, const CurveNormal& curve_normal, const float& u, const float& v, Hit& hit,
                                                  uint32_t& instID, uint32_t& instPrimID) {
  const uint4* tp = recs + (size_t)ti * 3;
  const uint4 a = __ldg(tp), b = __ldg(tp + 1), c = __ldg(tp + 2);
  hit.u = u; hit.v = v;
  hit.primID = a.w; hit.geomID = b.w;
  float lox = world_ray().ox, loy = world_ray().oy, loz = world_ray().oz;   // ray origin in the space the record's triangle lives in
  bool curve_hit = false;
  if (GENERAL) {
    const GeomDesc& d = descs[b.w];
    hit.geomID = d.geomID;
    if (GENERAL == 2 && d.kind != PRIM_TRIANGLE) {
      const float3 n = curve_normal();
      hit.ngx = n.x; hit.ngy = n.y; hit.ngz = n.z;
      curve_hit = true;
    }
    if (d.has_xfm) {
      instID = d.instID; instPrimID = 0u;   // instance_id_stack::push(context, instID, 0)
      if (ROBUST) { Ray lr = world_ray(); to_object_space(d, lr); lox = lr.ox; loy = lr.oy; loz = lr.oz; }
    }
  }
  if (curve_hit) {
  } else if (ROBUST) {
    const float v0x = sub_rn(__uint_as_float(a.x), lox), v0y = sub_rn(__uint_as_float(a.y), loy), v0z = sub_rn(__uint_as_float(a.z), loz);
    const float v1x = sub_rn(__uint_as_float(b.x), lox), v1y = sub_rn(__uint_as_float(b.y), loy), v1z = sub_rn(__uint_as_float(b.z), loz);
    const float v2x = sub_rn(__uint_as_float(c.x), lox), v2y = sub_rn(__uint_as_float(c.y), loy), v2z = sub_rn(__uint_as_float(c.z), loz);
    stable_normal(sub_rn(v2x, v0x), sub_rn(v2y, v0y), sub_rn(v2z, v0z), sub_rn(v0x, v1x), sub_rn(v0y, v1y), sub_rn(v0z, v1z),
                  sub_rn(v1x, v2x), sub_rn(v1y, v2y), sub_rn(v1z, v2z), hit.ngx, hit.ngy, hit.ngz);
  } else {
    const float e1x = __uint_as_float(b.x), e1y = __uint_as_float(b.y), e1z = __uint_as_float(b.z);
    const float e2x = __uint_as_float(c.x), e2y = __uint_as_float(c.y), e2z = __uint_as_float(c.z);
    hit.ngx = msub(e2y, e1z, mul_rn(e2z, e1y));
    hit.ngy = msub(e2z, e1x, mul_rn(e2x, e1z));
    hit.ngz = msub(e2x, e1y, mul_rn(e2y, e1x));
  }
  if (GENERAL && !curve_hit && (a.w >> 31)) {   // quad halves share the quad's primID; the second one has flipped winding
    hit.primID = a.w & 0x7FFFFFFFu;
    hit.ngx = -hit.ngx; hit.ngy = -hit.ngy; hit.ngz = -hit.ngz;
  }
}

}  // namespace rtk
