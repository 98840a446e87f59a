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
// untouched, a ray with tfar < 0 counts as already occluded and an empty scene returns at once.  The records are tested and
// written back by the code the batched kernel uses (record_tests.cuh; only its warp-wide SPREAD step writes that rule out);
// the traversal loop is per thread.
//
// `args` may be NULL or point to memory the calling thread can read.  args->context's instID[0] and instPrimID[0] seed a hit's
// instance ids, as on the host.  The scene's statistics counters do not count these queries.
//
// Argument filters (Embree 4's filter_sycl.h: on a GPU only the filter passed in the arguments runs).  A kernel opts in at compile
// time, as Embree 4's SYCL feature-mask specialisation does: rtcb200TraversableIntersect1<FEATURES> / Occluded1<FEATURES> with
// RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS in FEATURES.  The calls without a template argument compile no filter code, ignore
// args->filter and cost a kernel nothing.  In an opted-in call, when args->filter is set and args->feature_mask has
// RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS, every candidate that passes the primitive test is offered to the filter if its
// geometry -- the instanced child, through an instance -- enabled it with rtcSetGeometryEnableFilterFunctionFromArguments, or if
// args->flags has RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER:
//
//   __device__ void cutout(const RTCFilterFunctionNArguments* a) {      // N == 1
//     const RTCHit* h = (const RTCHit*)a->hit;
//     if (alpha(a->geometryUserPtr, h->primID, h->u, h->v) < 0.5f) a->valid[0] = 0;
//   }
//   __global__ void shade(RTCB200DeviceTraversable t, ...) {
//     RTCIntersectArguments args; rtcInitIntersectArguments(&args);
//     args.filter = cutout;                    // the address is taken in DEVICE code (or read from a __device__ variable)
//     rtcb200TraversableIntersect1<RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS>(t, &rh, &args);
//   }
//
//  - The opted-in kernel holds both the filtered and the unfiltered variants: more registers, whether a filter runs or not.
//  - The filter must be a __device__ function: a host function's address cannot be called here.  Without -rdc it has to live in
//    the translation unit of the kernel; with -rdc=true anywhere in the device link.
//  - Each call gets N = 1, valid[0] = -1, the geometry's user data (as rtcb200GetSceneDeviceTraversable snapshot it), `context` =
//    args->context (a default one in the thread's memory when NULL), `ray` = a copy of the caller's world-space RTCRay with tfar =
//    the candidate's t, and `hit` = the RTCHit the candidate would be written as.  During the call context->instID[0] /
//    instPrimID[0] hold the candidate's instance ids; they are restored afterwards, so a context shared by several threads races.
//  - Accepted (valid[0] != 0): closest hit -- the candidate becomes the hit, written as the filter left `hit`, and the `ray.tfar`
//    it left is the distance further candidates are culled against; any hit -- the query writes tfar = -inf and returns.
//    Rejected: nothing changes and traversal goes on; that record is not offered to this ray again.
//  - Candidates come in traversal order, one per leaf record (a sphere point's back hit, or a second root of a curve segment,
//    is not offered after its front hit is rejected).  Geometry filter callbacks never run on the device.
//  - The scene flag RTC_SCENE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS is not required, as on the host.
//
// Shading at a hit, in the same kernel (Embree 4's rtcGetGeometryUserDataFromTraversable / rtcGetGeometryTransformFromTraversable
// in SYCL device code, rtcore_scene.h:247,250, and rtcInterpolate through a table of the scene's buffers):
//
//   __global__ void shade(RTCB200DeviceTraversable t, RTCB200DeviceInterpolator normals, ...) {   // normals: VERTEX_ATTRIBUTE slot
//     rtcb200TraversableIntersect1(t, &rh);
//     if (rh.hit.geomID == RTC_INVALID_GEOMETRY_ID) return;
//     float n[3];
//     RTCB200DeviceInterpolateArguments ia = {rh.hit.geomID, rh.hit.instID[0], rh.hit.primID, rh.hit.u, rh.hit.v, n};
//     ia.valueCount = 3;
//     rtcb200Interpolate1(normals, &ia);                  // object space
//     float x[12];
//     rtcb200GetGeometryTransformFromTraversable(t, rh.hit.instID[0], 0.0f, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR, x);   // identity when
//     ...                                                  // the hit is not instanced
//   }
//
//  - rtcb200GetGeometryUserDataFromTraversable(t, geomID): the user data of geometry geomID of the traversable's own scene (an
//    instance's own pointer for an instance); NULL for an id beyond the scene's geometries or an empty slot.
//  - rtcb200GetGeometryTransformFromTraversable: an instance's local-to-world transform, in the bytes the host
//    rtcGetGeometryTransformFromScene writes for RTC_FORMAT_FLOAT3X4_ROW_MAJOR, _FLOAT3X4_COLUMN_MAJOR or _FLOAT4X4_COLUMN_MAJOR;
//    identity for any other geometry or an invalid id; `time` is ignored (one time step); another format leaves xfm untouched.
//  - Both read the snapshot rtcb200GetSceneDeviceTraversable took: user data and transforms as they were at that call.
//  - rtcb200Interpolate1: see RTCB200DeviceInterpolateArguments (embree4_b200.h).  Points, instances, a missing buffer or slot, and
//    a primitive or element beyond its buffer write quiet NaN, as the batched call does.
#pragma once
#include "embree4_b200.h"
#include "../embree_b200/csrc/record_tests.cuh"
#include "../embree_b200/csrc/interp.cuh"
#include "../embree_b200/csrc/transform_format.cuh"

namespace rtk {


// One query of one thread, specialised as the batched kernel is (trace.cu launch_k): GENERAL as general_of, ROBUST = Pluecker
// test.  The record test and the write-back are the kernel's own (record_tests.cuh record_test / record_write_back), so both
// entry points share the record code; closest-hit triangle scenes follow the SPREAD instantiation's acceptance rule, which
// is what the batched entry points run there.
// The RTCHit of winning record `ti` hit at (u, v) by the world-space ray r0 -- a curve / point record with the normal its test
// kept (cng*).
template <bool ROBUST, int GENERAL>
__device__ __forceinline__ void rtc_hit(const uint4* __restrict__ recs, const GeomDesc* __restrict__ descs, uint32_t ti, const Ray& r0, float u,
                                        float v, float cngx, float cngy, float cngz, uint32_t instID, uint32_t instPrimID, RTCHit& h) {
  Hit hit;
  record_write_back<ROBUST, GENERAL>(recs, descs, ti, [&] { return r0; }, [&] { return make_float3(cngx, cngy, cngz); }, u, v, hit, instID,
                                     instPrimID);
  h.Ng_x = hit.ngx; h.Ng_y = hit.ngy; h.Ng_z = hit.ngz; h.u = hit.u; h.v = hit.v;
  h.primID = hit.primID; h.geomID = hit.geomID; h.instID[0] = instID; h.instPrimID[0] = instPrimID;
}

// A filtered query's state in the thread's local memory: the traversal loop keeps only its address, so the filtered variants
// hold about as many registers as the others and the caller's kernel keeps its occupancy.
struct FilterQuery {
  const uint4* recs; const GeomDesc* descs; const RTCB200DeviceGeometry* geoms;
  Ray r;                                  // the caller's world-space ray
  RTCFilterFunctionN filter; RTCRayQueryContext* fctx; uint32_t instID, instPrimID; bool enforce;
  float tfar;                             // out: the distance an accepting call left in ray.tfar
  RTCHit best;                            // out: the hit of the last accepted candidate (closest hit)
};

// runIntersectionFilter1SYCL / runOcclusionFilter1SYCL (filter_sycl.h:83-108) for the candidate record ti at distance t; true =
// accepted.  A candidate whose geometry does not enable the filter is accepted without a call.
template <bool OCCLUDED, bool ROBUST, int GENERAL>
__device__ __noinline__ bool offer_candidate(FilterQuery* q, uint32_t ti, float t, float u, float v, float cngx, float cngy, float cngz) {
  const RTCB200DeviceGeometry& geom = q->geoms[__ldg(q->recs + (size_t)ti * 3 + 1).w];   // b.w: geomID or descriptor index
  q->tfar = t;
  if (!(q->enforce || geom.argFilterEnabled)) {   // the candidate is the hit: kept now, a later candidate overwrites u, v ...
    if (!OCCLUDED) rtc_hit<ROBUST, GENERAL>(q->recs, q->descs, ti, q->r, u, v, cngx, cngy, cngz, q->instID, q->instPrimID, q->best);
    return true;
  }
  RTCHit h;
  rtc_hit<ROBUST, GENERAL>(q->recs, q->descs, ti, q->r, u, v, cngx, cngy, cngz, q->instID, q->instPrimID, h);
  RTCRay fr;   // the caller's world-space ray, tfar = the candidate's t
  fr.org_x = q->r.ox; fr.org_y = q->r.oy; fr.org_z = q->r.oz; fr.tnear = q->r.tnear;
  fr.dir_x = q->r.dx; fr.dir_y = q->r.dy; fr.dir_z = q->r.dz; fr.time = q->r.time;
  fr.tfar = t; fr.mask = q->r.mask; fr.id = q->r.id; fr.flags = q->r.flags;
  RTCRayQueryContext fallback;
  rtcInitRayQueryContext(&fallback);
  RTCRayQueryContext* ctx = q->fctx ? q->fctx : &fallback;
  const unsigned saveI = ctx->instID[0], saveP = ctx->instPrimID[0];
  ctx->instID[0] = h.instID[0]; ctx->instPrimID[0] = h.instPrimID[0];   // instance_id_stack::push during an instanced traversal
  int valid = -1;
  RTCFilterFunctionNArguments fa;
  fa.valid = &valid; fa.geometryUserPtr = geom.userPtr; fa.context = ctx;
  fa.ray = reinterpret_cast<RTCRayN*>(&fr); fa.hit = reinterpret_cast<RTCHitN*>(&h); fa.N = 1;
  q->filter(&fa);
  ctx->instID[0] = saveI; ctx->instPrimID[0] = saveP;
  if (valid == 0) return false;
  if (!OCCLUDED) { q->best = h; q->tfar = fr.tfar; }   // copyHitToRay, and the distance the filter left
  return true;
}

// FILTER: the arguments' filter `filter` runs on every candidate whose geometry enables it (`enforce`:
// RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER), as runIntersectionFilter1SYCL / runOcclusionFilter1SYCL do (filter_sycl.h:83-108);
// geoms is the traversable's snapshot, fctx args->context.  Without FILTER the last four parameters are unused.
template <bool OCCLUDED, bool ROBUST, int GENERAL, bool FILTER>
__device__ __forceinline__ void query1(const RTCB200DeviceTraversable t, RTCRay* ray, RTCHit* hitrec, uint32_t instID, uint32_t instPrimID,
                                       const RTCB200DeviceGeometry* geoms, RTCFilterFunctionN filter, RTCRayQueryContext* fctx, bool enforce) {
  const Node8* __restrict__ nodes = static_cast<const Node8*>(t.nodes);
  const uint4* __restrict__ recs = static_cast<const uint4*>(t.records);
  const GeomDesc* __restrict__ descs = static_cast<const GeomDesc*>(t.descs);
  Ray r;
  r.ox = ray->org_x; r.oy = ray->org_y; r.oz = ray->org_z; r.tnear = ray->tnear;
  r.dx = ray->dir_x; r.dy = ray->dir_y; r.dz = ray->dir_z; r.time = ray->time;
  r.tfar = ray->tfar; r.mask = ray->mask; r.id = ray->id; r.flags = ray->flags;
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
  // record_test against the world-space ray; r.tfar stays the ray's own until traverse_records returns.  An occlusion filter is
  // handed the candidate's hit too.  Closest-hit GENERAL 0 Moeller-Trumbore scenes take the SPREAD rule.
  auto test = [&](uint32_t ti, float& tfar) -> bool {
    const uint4* tp = recs + (size_t)ti * 3;
    const uint4 a = __ldg(tp), b = __ldg(tp + 1), c = __ldg(tp + 2);
    return record_test<ROBUST, GENERAL, !OCCLUDED || FILTER, GENERAL == 0 && !OCCLUDED && !ROBUST>(descs, a, b, c, r, tfar, hit_u, hit_v,
                                                                                                    [&](const RecordHit& h) {
      if (OCCLUDED && !FILTER) return;
      tfar = h.t; hit_rec = ti;
      if (GENERAL == 2 && h.curve) { cngx = h.ngx; cngy = h.ngy; cngz = h.ngz; }
    });
  };
  // FILTER: a candidate the primitive test accepted is offered to the arguments' filter (offer_candidate); a rejected one leaves
  // `tfar` as it was
  FilterQuery q;
  if (FILTER) {
    q.recs = recs; q.descs = descs; q.geoms = geoms; q.r = r; q.filter = filter; q.fctx = fctx;
    q.instID = instID; q.instPrimID = instPrimID; q.enforce = enforce;
  }
  auto ftest = [&](uint32_t ti, float& tfar) -> bool {
    const float tprev = tfar;
    if (!test(ti, tfar)) return false;
    if (offer_candidate<OCCLUDED, ROBUST, GENERAL>(&q, ti, tfar, hit_u, hit_v, cngx, cngy, cngz)) { tfar = q.tfar; return true; }
    tfar = tprev;
    return false;
  };
  bool found;
  if (FILTER) found = traverse_records<OCCLUDED, false>(r, rcp_safe_fast(r.dx), rcp_safe_fast(r.dy), rcp_safe_fast(r.dz), load_node, ftest, t.root_valid, nullptr);
  else found = traverse_records<OCCLUDED, false>(r, rcp_safe_fast(r.dx), rcp_safe_fast(r.dy), rcp_safe_fast(r.dz), load_node, test, t.root_valid, nullptr);
  if (!found) return;
  if (OCCLUDED) { ray->tfar = -INFINITY; return; }
  if (FILTER) {
    ray->tfar = r.tfar;
    const RTCHit& b = q.best;
    hitrec->Ng_x = b.Ng_x; hitrec->Ng_y = b.Ng_y; hitrec->Ng_z = b.Ng_z; hitrec->u = b.u; hitrec->v = b.v;
    hitrec->primID = b.primID; hitrec->geomID = b.geomID; hitrec->instID[0] = b.instID[0]; hitrec->instPrimID[0] = b.instPrimID[0];
    return;
  }
  RTCHit h;   // (only r's tfar has changed: the write-back reads its origin and direction)
  rtc_hit<ROBUST, GENERAL>(recs, descs, hit_rec, r, hit_u, hit_v, cngx, cngy, cngz, instID, instPrimID, h);
  ray->tfar = r.tfar;
  hitrec->Ng_x = h.Ng_x; hitrec->Ng_y = h.Ng_y; hitrec->Ng_z = h.Ng_z; hitrec->u = h.u; hitrec->v = h.v;
  hitrec->primID = h.primID; hitrec->geomID = h.geomID; hitrec->instID[0] = h.instID[0]; hitrec->instPrimID[0] = h.instPrimID[0];
}

// One query of one thread, as its own function: the six variants without a filter and the six with one.
template <bool OCCLUDED, bool ROBUST, int GENERAL>
__device__ __noinline__ void device_query1(const RTCB200DeviceTraversable t, RTCRay* ray, RTCHit* hitrec, uint32_t instID, uint32_t instPrimID) {
  query1<OCCLUDED, ROBUST, GENERAL, false>(t, ray, hitrec, instID, instPrimID, nullptr, nullptr, nullptr, false);
}
template <bool OCCLUDED, bool ROBUST, int GENERAL>
__device__ __noinline__ void device_query1_filter(const RTCB200DeviceTraversable t, RTCRay* ray, RTCHit* hitrec, uint32_t instID, uint32_t instPrimID,
                                                  RTCFilterFunctionN filter, RTCRayQueryContext* fctx, bool enforce) {
  query1<OCCLUDED, ROBUST, GENERAL, true>(t, ray, hitrec, instID, instPrimID, t.geometries, filter, fctx, enforce);
}

// The filtered specialisations, compiled only into kernels that ask for argument filters (FILTERS): run when the arguments carry a
// filter and their feature_mask admits it (filter_sycl.h:32-43); false when the query is left to the unfiltered ones.
template <bool OCCLUDED, bool FILTERS>
struct FilterDispatch {
  template <typename Args>
  static __device__ __forceinline__ bool run(const RTCB200DeviceTraversable&, RTCRay*, RTCHit*, const Args*, uint32_t, uint32_t, int) { return false; }
};
template <bool OCCLUDED>
struct FilterDispatch<OCCLUDED, true> {
  template <typename Args>
  static __device__ __forceinline__ bool run(const RTCB200DeviceTraversable& t, RTCRay* ray, RTCHit* hit, const Args* args, uint32_t instID,
                                             uint32_t instPrimID, int variant) {
    if (!(args && args->filter && (args->feature_mask & RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS))) return false;
    const RTCFilterFunctionN f = args->filter;
    RTCRayQueryContext* fctx = args->context;
    const bool enforce = (args->flags & RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER) != 0;
    switch (variant) {
      case 0: device_query1_filter<OCCLUDED, false, 0>(t, ray, hit, instID, instPrimID, f, fctx, enforce); break;
      case 1: device_query1_filter<OCCLUDED, true, 0>(t, ray, hit, instID, instPrimID, f, fctx, enforce); break;
      case 2: device_query1_filter<OCCLUDED, false, 1>(t, ray, hit, instID, instPrimID, f, fctx, enforce); break;
      case 3: device_query1_filter<OCCLUDED, true, 1>(t, ray, hit, instID, instPrimID, f, fctx, enforce); break;
      case 4: device_query1_filter<OCCLUDED, false, 2>(t, ray, hit, instID, instPrimID, f, fctx, enforce); break;
      default: device_query1_filter<OCCLUDED, true, 2>(t, ray, hit, instID, instPrimID, f, fctx, enforce); break;
    }
    return true;
  }
};

// the specialisation the batched kernel would run for this scene (trace.cu launch_k); with FEATURES containing
// RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS, the filtered one when the arguments carry a filter
template <bool OCCLUDED, unsigned FEATURES, typename Args>
__device__ __forceinline__ void device_query1_dispatch(const RTCB200DeviceTraversable& t, RTCRay* ray, RTCHit* hit, const Args* args) {
  const RTCRayQueryContext* ctx = args ? args->context : nullptr;
  if (!t.root_valid) return;   // empty scene
  uint32_t instID = RTC_INVALID_GEOMETRY_ID, instPrimID = RTC_INVALID_GEOMETRY_ID;
  if (ctx) { instID = ctx->instID[0]; instPrimID = ctx->instPrimID[0]; }
  const int g = general_of(t.descs, t.curves);
  if (FilterDispatch<OCCLUDED, (FEATURES & RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS) != 0>::run(t, ray, hit, args, instID, instPrimID,
                                                                                                    g * 2 + (t.robust ? 1 : 0)))
    return;
  switch (g * 2 + (t.robust ? 1 : 0)) {
    case 0: device_query1<OCCLUDED, false, 0>(t, ray, hit, instID, instPrimID); break;
    case 1: device_query1<OCCLUDED, true, 0>(t, ray, hit, instID, instPrimID); break;
    case 2: device_query1<OCCLUDED, false, 1>(t, ray, hit, instID, instPrimID); break;
    case 3: device_query1<OCCLUDED, true, 1>(t, ray, hit, instID, instPrimID); break;
    case 4: device_query1<OCCLUDED, false, 2>(t, ray, hit, instID, instPrimID); break;
    default: device_query1<OCCLUDED, true, 2>(t, ray, hit, instID, instPrimID); break;
  }
}

// entry geomID of the snapshot's geomID block (the header in front of t.geometries[0] locates it), or NULL
__device__ __forceinline__ const RTCB200DeviceGeometryInfo* geometry_info(const RTCB200DeviceTraversable& t, unsigned geomID) {
  if (!t.geometries) return nullptr;
  const RTCB200DeviceGeometryHeader* h = reinterpret_cast<const RTCB200DeviceGeometryHeader*>(t.geometries) - 1;
  return geomID < h->count ? h->byGeomID + geomID : nullptr;
}

// One hit of rtcb200InterpolateHitsDevice, its value k written at index k.  A function of its own, so the caller's kernel does not
// carry the interpolation's registers through its other code.
inline __device__ __noinline__ void device_interpolate1(const RTCB200DeviceInterpolator ip, const RTCB200DeviceInterpolateArguments* a) {
  const uint32_t geomID = a->geomID;
  if (geomID == kInvalidID) return;   // a miss: nothing is written
  float* const out[6] = {a->P, a->dPdu, a->dPdv, a->ddPdudu, a->ddPdvdv, a->ddPdudv};
  interpolate_hit(static_cast<const InterpEntry*>(ip.table), ip.nentries, geomID, a->instID, a->primID, a->u, a->v, a->valueCount,
                  [&](unsigned k, const float o[6]) {
#pragma unroll
                    for (int c = 0; c < 6; ++c)
                      if (out[c]) out[c][k] = o[c];
                  });
}

}  // namespace rtk

// Closest hit of one ray: as one record of rtcb200Intersect1MDevice.  No filter code is compiled in: args->filter is not called.
__device__ __forceinline__ void rtcb200TraversableIntersect1(const RTCB200DeviceTraversable& t, RTCRayHit* rayhit,
                                                             const RTCIntersectArguments* args = nullptr) {
  rtk::device_query1_dispatch<false, RTC_FEATURE_FLAG_NONE>(t, &rayhit->ray, &rayhit->hit, args);
}
// Any hit of one ray: as one record of rtcb200Occluded1MDevice (tfar = -inf on a hit).  No filter code is compiled in.
__device__ __forceinline__ void rtcb200TraversableOccluded1(const RTCB200DeviceTraversable& t, RTCRay* ray,
                                                            const RTCOccludedArguments* args = nullptr) {
  rtk::device_query1_dispatch<true, RTC_FEATURE_FLAG_NONE>(t, ray, nullptr, args);
}
// The same with the features the kernel is compiled for (Embree 4's SYCL feature-mask specialisation):
// rtcb200TraversableIntersect1<RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS>(t, &rh, &args) compiles the filtered variants into
// the kernel and runs them when args->filter is set and args->feature_mask admits it.  Other feature bits change nothing.
template <unsigned FEATURES>
__device__ __forceinline__ void rtcb200TraversableIntersect1(const RTCB200DeviceTraversable& t, RTCRayHit* rayhit, const RTCIntersectArguments* args) {
  rtk::device_query1_dispatch<false, FEATURES>(t, &rayhit->ray, &rayhit->hit, args);
}
template <unsigned FEATURES>
__device__ __forceinline__ void rtcb200TraversableOccluded1(const RTCB200DeviceTraversable& t, RTCRay* ray, const RTCOccludedArguments* args) {
  rtk::device_query1_dispatch<true, FEATURES>(t, ray, nullptr, args);
}

// User data of geometry geomID of the traversable's scene (rtcore_sycl.cpp:114-118); NULL for an invalid id or an empty slot.
__device__ __forceinline__ void* rtcb200GetGeometryUserDataFromTraversable(const RTCB200DeviceTraversable& t, unsigned int geomID) {
  const RTCB200DeviceGeometryInfo* e = rtk::geometry_info(t, geomID);
  return e ? e->userPtr : nullptr;
}
// Local-to-world transform of instance geomID, identity for any other geometry or an invalid id (rtcore_sycl.cpp:120-133); the
// bytes of the host rtcGetGeometryTransformFromScene.  An unknown format leaves xfm untouched.
__device__ __forceinline__ void rtcb200GetGeometryTransformFromTraversable(const RTCB200DeviceTraversable& t, unsigned int geomID, float time,
                                                                           enum RTCFormat format, void* xfm) {
  (void)time;   // one time step
  const RTCB200DeviceGeometryInfo* e = rtk::geometry_info(t, geomID);
  float m[12] = {1.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f};
  if (e && e->isInstance)
    for (int k = 0; k < 12; ++k) m[k] = e->xfm[k];
  rtk::store_transform(m, (unsigned)format, static_cast<float*>(xfm));
}
// rtcInterpolate of one hit through a scene's interpolator (rtcb200GetSceneDeviceInterpolator): the values
// rtcb200InterpolateHitsDevice writes for the same hit, value k of each output at index k.
__device__ __forceinline__ void rtcb200Interpolate1(const RTCB200DeviceInterpolator& ip, const RTCB200DeviceInterpolateArguments* args) {
  rtk::device_interpolate1(ip, args);
}
