// embree4_b200_device.cuh -- ray queries from the caller's own CUDA kernels (Embree 4's rtcTraversableIntersect1 /
// rtcTraversableOccluded1 in device code, rtcore_scene.h:266,304).
//
// Include it from a .cu file compiled with `-I <this directory>`; it reaches the library's core headers by relative path.
// The host takes a committed scene's RTCB200DeviceTraversable (rtcb200GetSceneDeviceTraversable, embree4_b200.h Section B)
// and passes it to the kernel by value; every thread may then trace its own rays:
//
//   __global__ void shade(RTCB200DeviceTraversable t, ...) {
//     RTCRayHit rh = ...;                      // registers, local, shared or global memory
//     rtcb200TraversableIntersect1(t, &rh);
//     if (rh.hit.geomID != RTC_INVALID_GEOMETRY_ID) { RTCRay shadow = ...; rtcb200TraversableOccluded1(t, &shadow); }
//   }
//
// Results are those of rtcb200Intersect1MDevice / rtcb200Occluded1MDevice for the same ray, bit for bit, when this file is
// compiled with nvcc's default floating-point flags (-use_fast_math, -prec-div=false or -ftz=true void that): the same fields
// are written (tfar, Ng, u, v, primID, geomID, instID[0], instPrimID[0]; occluded: tfar = -inf), a miss leaves the record
// untouched, a ray with tfar < 0 counts as already occluded and an empty scene returns at once.
//
// `args` may be NULL or point to memory the calling thread can read.  Only args->context is read: its instID[0] and
// instPrimID[0] seed a hit's instance ids, as on the host.  args->filter, flags and feature_mask are ignored -- no filter runs
// on the device, and the scene's statistics counters do not count these queries.
#pragma once
#include "embree4_b200.h"
#include "../embree_b200/csrc/record_tests.cuh"

namespace rtk {

// One query of one thread, specialised as the batched kernel is (trace.cu launch_k): GENERAL 0 = triangle records with
// geomIDs, 1 = records through descriptors (instances, quads), 2 = with curve or point records; ROBUST = Pluecker test.
// The record test and the write-back restate trace.cu's test_tri and write_back for one lane (the tests of
// tests/test_device_traversal.py compare both bit for bit); closest-hit triangle scenes follow the SPREAD instantiation's
// acceptance rule, which is what the batched entry points run there.
template <bool OCCLUDED, bool ROBUST, int GENERAL>
__device__ __noinline__ void device_query1(const RTCB200DeviceTraversable t, RTCRay* ray, RTCHit* hitrec, uint32_t instID, uint32_t instPrimID) {
  const Node8* __restrict__ nodes = static_cast<const Node8*>(t.nodes);
  const uint4* __restrict__ recs = static_cast<const uint4*>(t.records);
  const GeomDesc* __restrict__ descs = static_cast<const GeomDesc*>(t.descs);
  Ray r;
  r.ox = ray->org_x; r.oy = ray->org_y; r.oz = ray->org_z; r.tnear = ray->tnear;
  r.dx = ray->dir_x; r.dy = ray->dir_y; r.dz = ray->dir_z; r.time = ray->time;
  r.tfar = ray->tfar; r.mask = ray->mask; r.id = ray->id; r.flags = ray->flags;
  const float tfar0 = r.tfar;   // the ray's own tfar: the SPREAD rule tests every triangle against it
  float hit_u = 0.0f, hit_v = 0.0f, cngx = 0.0f, cngy = 0.0f, cngz = 0.0f;
  uint32_t hit_rec = 0;

  auto load_node = [&](uint32_t i) -> NodeW {
    const uint4* p = reinterpret_cast<const uint4*>(nodes + i);
    NodeW nw;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const uint4 q = __ldg(p + k);
      nw.w[4 * k] = q.x; nw.w[4 * k + 1] = q.y; nw.w[4 * k + 2] = q.z; nw.w[4 * k + 3] = q.w;
    }
    return nw;
  };
  // trace.cu test_tri: ray mask, then the descriptor's instance mask and object-space ray, then the record's own test
  auto test = [&](uint32_t ti, float& tfar) -> bool {
    const uint4* tp = recs + (size_t)ti * 3;
    const uint4 a = __ldg(tp), b = __ldg(tp + 1), c = __ldg(tp + 2);
    Ray lr = r;
    bool visible = (c.w & lr.mask) != 0;
    if (GENERAL) {
      const GeomDesc& d = descs[b.w];
      visible = visible && (d.inst_mask & lr.mask) != 0;
      if (d.has_xfm) to_object_space(d, lr);
      if (GENERAL == 2 && d.kind != PRIM_TRIANGLE) {   // curve / point record: the winning test's normal is kept
        CurveHit ch;
        if (!(visible && curve_record_test(d, lr, tfar, a, b, c, ch))) return false;
        if (!OCCLUDED) { tfar = ch.t; hit_u = ch.u; hit_v = ch.v; hit_rec = ti; cngx = ch.ngx; cngy = ch.ngy; cngz = ch.ngz; }
        return true;
      }
    }
    if (!visible) return false;
    if (ROBUST) {
      PlueckerHit ph;
      if (!tri_test_pluecker(lr, tfar, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(b.x),
                             __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(c.x), __uint_as_float(c.y), __uint_as_float(c.z), ph))
        return false;
      if (OCCLUDED) return true;
      tfar = ph.t; pluecker_uv(ph, hit_u, hit_v); hit_rec = ti;
      if (GENERAL && (a.w >> 31)) {   // second half of a quad (QuadHitPlueckerM::finalize, AVX form)
        const float u1 = sub_rn(1.0f, hit_u), v1 = sub_rn(1.0f, hit_v);
        hit_u = v1; hit_v = u1;
      }
      return true;
    }
    // SPREAD (GENERAL 0 closest hit): a candidate passes the test against the ray's own tfar and its t is <= the hit so far
    constexpr bool kSpread = GENERAL == 0 && !OCCLUDED;
    TriHit th;
    if (!tri_test(lr, kSpread ? tfar0 : tfar, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(b.x),
                  __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(c.x), __uint_as_float(c.y), __uint_as_float(c.z), th))
      return false;
    if (OCCLUDED) return true;
    const float rcpAbsDen = 1.0f / th.absDen;   // finalize(): t,u,v = T,U,V * rcp(absDen)
    const float tt = th.T * rcpAbsDen;
    if (kSpread && !(tt <= tfar)) return false;
    tfar = tt;
    if (GENERAL && (a.w >> 31)) {   // second half of a quad: U' = absDen - V, V' = absDen - U (quad_intersector_moeller.h:196-198)
      hit_u = sub_rn(th.absDen, th.V) * rcpAbsDen; hit_v = sub_rn(th.absDen, th.U) * rcpAbsDen;
    } else { hit_u = th.U * rcpAbsDen; hit_v = th.V * rcpAbsDen; }
    hit_rec = ti;
    return true;
  };
  const Ray r0 = r;   // the world-space ray: traverse_records shrinks r.tfar
  if (!traverse_records<OCCLUDED, false>(r, rcp_safe_fast(r.dx), rcp_safe_fast(r.dy), rcp_safe_fast(r.dz), load_node, test, t.root_valid, nullptr))
    return;
  if (OCCLUDED) { ray->tfar = -INFINITY; return; }

  // trace.cu write_back: Ng and the ids from the winning record; Ng stays in object space
  const uint4* tp = recs + (size_t)hit_rec * 3;
  const uint4 a = __ldg(tp), b = __ldg(tp + 1), c = __ldg(tp + 2);
  float ngx, ngy, ngz;
  uint32_t primID = a.w, geomID = b.w;
  float lox = r0.ox, loy = r0.oy, loz = r0.oz;   // ray origin in the space the record's triangle lives in
  bool curve_hit = false;
  if (GENERAL) {
    const GeomDesc& d = descs[b.w];
    geomID = d.geomID;
    if (GENERAL == 2 && d.kind != PRIM_TRIANGLE) { ngx = cngx; ngy = cngy; ngz = cngz; curve_hit = true; }
    if (d.has_xfm) {
      instID = d.instID; instPrimID = 0u;   // instance_id_stack::push(context, instID, 0)
      if (ROBUST) { Ray lr = r0; to_object_space(d, lr); lox = lr.ox; loy = lr.oy; loz = lr.oz; }
    }
  }
  if (curve_hit) {
  } else if (ROBUST) {   // stable_triangle_normal of the origin-relative edges, exactly as in tri_test_pluecker
    const float v0x = sub_rn(__uint_as_float(a.x), lox), v0y = sub_rn(__uint_as_float(a.y), loy), v0z = sub_rn(__uint_as_float(a.z), loz);
    const float v1x = sub_rn(__uint_as_float(b.x), lox), v1y = sub_rn(__uint_as_float(b.y), loy), v1z = sub_rn(__uint_as_float(b.z), loz);
    const float v2x = sub_rn(__uint_as_float(c.x), lox), v2y = sub_rn(__uint_as_float(c.y), loy), v2z = sub_rn(__uint_as_float(c.z), loz);
    stable_normal(sub_rn(v2x, v0x), sub_rn(v2y, v0y), sub_rn(v2z, v0z), sub_rn(v0x, v1x), sub_rn(v0y, v1y), sub_rn(v0z, v1z),
                  sub_rn(v1x, v2x), sub_rn(v1y, v2y), sub_rn(v1z, v2z), ngx, ngy, ngz);
  } else {
    const float e1x = __uint_as_float(b.x), e1y = __uint_as_float(b.y), e1z = __uint_as_float(b.z);
    const float e2x = __uint_as_float(c.x), e2y = __uint_as_float(c.y), e2z = __uint_as_float(c.z);
    ngx = msub(e2y, e1z, mul_rn(e2z, e1y));
    ngy = msub(e2z, e1x, mul_rn(e2x, e1z));
    ngz = msub(e2x, e1y, mul_rn(e2y, e1x));
  }
  if (GENERAL && !curve_hit && (a.w >> 31)) {   // quad halves share the quad's primID; the second one has flipped winding
    primID = a.w & 0x7FFFFFFFu;
    ngx = -ngx; ngy = -ngy; ngz = -ngz;
  }
  ray->tfar = r.tfar;
  hitrec->Ng_x = ngx; hitrec->Ng_y = ngy; hitrec->Ng_z = ngz; hitrec->u = hit_u; hitrec->v = hit_v;
  hitrec->primID = primID; hitrec->geomID = geomID; hitrec->instID[0] = instID; hitrec->instPrimID[0] = instPrimID;
}

// the specialisation the batched kernel would run for this scene (trace.cu launch_k)
template <bool OCCLUDED>
__device__ __forceinline__ void device_query1_dispatch(const RTCB200DeviceTraversable& t, RTCRay* ray, RTCHit* hit, const RTCRayQueryContext* ctx) {
  if (!t.root_valid) return;   // empty scene
  uint32_t instID = RTC_INVALID_GEOMETRY_ID, instPrimID = RTC_INVALID_GEOMETRY_ID;
  if (ctx) { instID = ctx->instID[0]; instPrimID = ctx->instPrimID[0]; }
  const int g = !t.descs ? 0 : (t.curves ? 2 : 1);
  switch (g * 2 + (t.robust ? 1 : 0)) {
    case 0: device_query1<OCCLUDED, false, 0>(t, ray, hit, instID, instPrimID); break;
    case 1: device_query1<OCCLUDED, true, 0>(t, ray, hit, instID, instPrimID); break;
    case 2: device_query1<OCCLUDED, false, 1>(t, ray, hit, instID, instPrimID); break;
    case 3: device_query1<OCCLUDED, true, 1>(t, ray, hit, instID, instPrimID); break;
    case 4: device_query1<OCCLUDED, false, 2>(t, ray, hit, instID, instPrimID); break;
    default: device_query1<OCCLUDED, true, 2>(t, ray, hit, instID, instPrimID); break;
  }
}

}  // namespace rtk

// Closest hit of one ray: as one record of rtcb200Intersect1MDevice.
__device__ __forceinline__ void rtcb200TraversableIntersect1(const RTCB200DeviceTraversable& t, RTCRayHit* rayhit,
                                                             const RTCIntersectArguments* args = nullptr) {
  rtk::device_query1_dispatch<false>(t, &rayhit->ray, &rayhit->hit, args ? args->context : nullptr);
}
// Any hit of one ray: as one record of rtcb200Occluded1MDevice (tfar = -inf on a hit).
__device__ __forceinline__ void rtcb200TraversableOccluded1(const RTCB200DeviceTraversable& t, RTCRay* ray,
                                                            const RTCOccludedArguments* args = nullptr) {
  rtk::device_query1_dispatch<true>(t, ray, nullptr, args ? args->context : nullptr);
}
