// rt_core.cuh -- data layout and per-ray / per-node core routines of the CUDA ray tracing kernels.
//
// Everything here is `RT_HD` (__host__ __device__) on purpose: the CUDA kernels in build.cu / trace.cu call
// these routines per thread, and tests/emu/ compiles the very same header with g++ so the node encoding,
// the traversal loop and the triangle test can be debugged in a container without a GPU.  The host build is
// a TEST tool only; the product library contains just the device instantiations.
//
// Reference semantics restated here (paths relative to the reference tree):
//   ray setup        kernels/bvh/node_intersector1.h:34-57, common/math/vec3fa.h:167-172 (rcp_safe)
//   slab test        kernels/bvh/node_intersector1.h:484-531  (we test 8 children of a *quantised* node)
//   traversal loop   kernels/bvh/bvh_intersector1.cpp:31-114 (closest), :116-197 (any hit)
//   triangle test    kernels/geometry/triangle_intersector_moeller.h:69-111 (+ :29-36 finalize)
//   hit commit       kernels/geometry/intersector_epilog.h:220-302 (closest), :304-369 (occluded)
#pragma once
#include <stdint.h>
#include <math.h>
#include <float.h>

#if defined(__CUDACC__)
#define RT_HD __host__ __device__ __forceinline__
#define RT_D __device__ __forceinline__
#else
#define RT_HD inline
#endif

namespace rtk {

// ------------------------------------------------------------------------------------------------
// HBM layout
// ------------------------------------------------------------------------------------------------
// BVH8 node, 96 bytes = 3 x 32 B, 32-byte aligned: one node is three whole DRAM/L2 sectors (compressed wide BVH:
// 8-bit child boxes on a per-node power-of-two grid).
//   w0..w2  : px, py, pz (float bits) -- origin of the node's grid
//   w3      : ex | ey<<8 | ez<<16 | imask<<24   (biased exponents of the grid scale per axis; imask bit s = slot s
//             holds an internal child)
//   w4, w5  : child_base, tri_base
//   w6..w11 : leaf masks, 3 bytes per slot (slot s at byte 24 + 3 s): bit k set = triangle tri_base + k belongs to the
//             leaf in slot s (<= kMaxLeafTris bits per slot, <= 24 per node, disjoint); 0 for internal / empty slots
//   w12..w23: quantised planes, one byte per slot: qlo_x[8] qlo_y[8] qlo_z[8] qhi_x[8] qhi_y[8] qhi_z[8]
// Internal children of a node are stored consecutively from child_base in slot order, the triangles of its leaf slots
// consecutively from tri_base.  Round 1 used an 80-byte node with one packed meta byte per slot: every visit then
// decoded count/offset per child and straddled three sectors with five 16-byte loads; the precomputed masks cost
// 16 bytes per node and remove the decode from the inner loop.
struct alignas(32) Node8 {
  uint32_t w[24];
};
static_assert(sizeof(Node8) == 96, "Node8 must be 96 bytes");
constexpr int kNodePlaneWord = 12;   // first word of the quantised planes
constexpr int kNodeMaskByte = 24;    // first byte of the per-slot leaf masks

// Triangle record, 48 bytes = 3 x 16 B; what the reference keeps per lane of a Triangle4 block
// (kernels/geometry/triangle.h:98-120: v0, e1 = v0 - v1, e2 = v2 - v0) plus ids and the geometry mask.
struct alignas(16) TriRec {
  float v0x, v0y, v0z; uint32_t primID;
  float e1x, e1y, e1z; uint32_t geomID;
  float e2x, e2y, e2z; uint32_t mask;
};
static_assert(sizeof(TriRec) == 48, "TriRec must be 48 bytes");

// Binary build tree (LBVH or binned SAH) that is collapsed into Node8s.  ids: [0, n-1) internal, [n-1, 2n-1) leaves.
struct alignas(16) Node2 {
  float lox, loy, loz; int32_t left;    // child id (internal); for a leaf: index into the sorted primitive list
  float hix, hiy, hiz; int32_t right;   // child id (internal); for a leaf: -1
  uint32_t first, count;                // range [first, first+count) of sorted primitives below this node
  uint32_t parent, pad;
};
static_assert(sizeof(Node2) == 48, "Node2 must be 48 bytes");

struct alignas(16) PrimRef {  // kernels/builders/primref.h:24-28 (lower, geomID | upper, primID) -> ours keeps a global prim index
  float lox, loy, loz; uint32_t prim;   // global triangle index (geometry found by prefix search)
  float hix, hiy, hiz; uint32_t valid;
};

struct Ray {  // RTCRay, include/embree4/rtcore_ray.h:11-28
  float ox, oy, oz, tnear, dx, dy, dz, time, tfar;
  uint32_t mask, id, flags;
};
struct Hit {  // what a closest-hit query commits (intersector_epilog.h:285-299)
  float t, u, v, ngx, ngy, ngz;
  uint32_t primID, geomID;
};

constexpr float kMinRcpInput = 1e-18f;   // common/math/constants.h:18
constexpr float kRcpOfMin = 5e17f;         // |1/dir| at or above this: the direction component is (nearly) the rcp_safe clamp
constexpr float kFltLarge = 1.844E18f;   // common/math/constants.h:21
constexpr uint32_t kInvalidID = 0xFFFFFFFFu;
constexpr int kMaxLeafTris = 3;
constexpr int kStackSize = 64;           // entries of 8 B; each BVH8 level pushes at most one node group

// ------------------------------------------------------------------------------------------------
// small portable helpers
// ------------------------------------------------------------------------------------------------
RT_HD uint32_t f2u(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  union { float f; uint32_t u; } c; c.f = f; return c.u;
#endif
}
RT_HD float u2f(uint32_t u) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(u);
#else
  union { float f; uint32_t u; } c; c.u = u; return c.f;
#endif
}
RT_HD int clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __clz((int)x);
#else
  return x ? __builtin_clz(x) : 32;
#endif
}
RT_HD int popc32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}
// fused multiply-add / explicitly rounded mul: the reference's AVX2/AVX-512 paths contract madd/msub
// (common/math/vec3.h:204,209), so bit-equal Ng needs the same contraction and NO other.
RT_HD float fma_rn(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
  return __fmaf_rn(a, b, c);
#else
  return fmaf(a, b, c);
#endif
}
RT_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  volatile float r = a * b; return r;  // volatile: forbid host-side contraction
#endif
}
RT_HD float sub_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  volatile float r = a - b; return r;
#endif
}
RT_HD float msub(float a, float b, float c) { return fma_rn(a, b, -c); }            // a*b - c
// a - b and a * b rounded towards -inf (_rd) or +inf (_ru).  The host versions round to nearest and step one float
// towards the required side when the exact error of that rounding (TwoSum / FMA, both exact) has the wrong sign.
RT_HD float sub_rd(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rd(a, b);
#else
  volatile float r = a - b; volatile float bb = r - a; const float e = (a - (r - bb)) + (-b - bb);
  return e < 0.0f ? nextafterf(r, -INFINITY) : r;
#endif
}
RT_HD float sub_ru(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_ru(a, b);
#else
  volatile float r = a - b; volatile float bb = r - a; const float e = (a - (r - bb)) + (-b - bb);
  return e > 0.0f ? nextafterf(r, INFINITY) : r;
#endif
}
RT_HD float mul_rd(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rd(a, b);
#else
  volatile float r = a * b; return fmaf(a, b, -r) < 0.0f ? nextafterf(r, -INFINITY) : r;
#endif
}
RT_HD float mul_ru(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_ru(a, b);
#else
  volatile float r = a * b; return fmaf(a, b, -r) > 0.0f ? nextafterf(r, INFINITY) : r;
#endif
}
RT_HD float dot3(float ax, float ay, float az, float bx, float by, float bz) {      // vec3.h:204
  return fma_rn(ax, bx, fma_rn(ay, by, mul_rn(az, bz)));
}
RT_HD float rcp_safe(float d) { return 1.0f / (fabsf(d) < kMinRcpInput ? kMinRcpInput : d); }

// ------------------------------------------------------------------------------------------------
// triangle test: MoellerTrumboreIntersector1<M>::intersect restated for one lane
// returns true when the triangle is hit inside (tnear, tfar]; outputs T,U,V scaled by absDen and Ng.
// ------------------------------------------------------------------------------------------------
struct TriHit { float T, U, V, absDen, ngx, ngy, ngz; };

RT_HD bool tri_test(const Ray& r, float tfar, float v0x, float v0y, float v0z, float e1x, float e1y, float e1z,
                    float e2x, float e2y, float e2z, TriHit& h) {
  const float cx = sub_rn(v0x, r.ox), cy = sub_rn(v0y, r.oy), cz = sub_rn(v0z, r.oz);          // C = v0 - O
  const float rx = msub(cy, r.dz, mul_rn(cz, r.dy));                                           // R = cross(C, D)
  const float ry = msub(cz, r.dx, mul_rn(cx, r.dz));
  const float rz = msub(cx, r.dy, mul_rn(cy, r.dx));
  const float ngx = msub(e2y, e1z, mul_rn(e2z, e1y));                                          // Ng = cross(e2, e1)
  const float ngy = msub(e2z, e1x, mul_rn(e2x, e1z));
  const float ngz = msub(e2x, e1y, mul_rn(e2y, e1x));
  const float den = dot3(ngx, ngy, ngz, r.dx, r.dy, r.dz);
  const float absDen = fabsf(den);
  const uint32_t sgn = f2u(den) & 0x80000000u;
  const float U = u2f(f2u(dot3(rx, ry, rz, e2x, e2y, e2z)) ^ sgn);
  const float V = u2f(f2u(dot3(rx, ry, rz, e1x, e1y, e1z)) ^ sgn);
  if (!((den != 0.0f) & (U >= 0.0f) & (V >= 0.0f) & (U + V <= absDen))) return false;
  const float T = u2f(f2u(dot3(ngx, ngy, ngz, cx, cy, cz)) ^ sgn);
  if (!((mul_rn(absDen, r.tnear) < T) & (T <= mul_rn(absDen, tfar)))) return false;
  h.T = T; h.U = U; h.V = V; h.absDen = absDen; h.ngx = ngx; h.ngy = ngy; h.ngz = ngz;
  return true;
}

// ------------------------------------------------------------------------------------------------
// robust mode (RTC_SCENE_FLAG_ROBUST): PlueckerIntersector1<M>::intersect restated for one lane
// (kernels/geometry/triangle_intersector_pluecker.h:62-118, finalize :30-37, stable_triangle_normal
// common/math/vec3.h:210-222).  Vertices are taken relative to the ray origin; the edge tests are watertight along
// shared edges; t is accepted on the closed interval [tnear, tfar].
// ------------------------------------------------------------------------------------------------
struct PlueckerHit { float t, U, V, UVW, ngx, ngy, ngz; };

RT_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  volatile float r = a + b; return r;
#endif
}
RT_HD float rcp_rn(float a) { return 1.0f / a; }

RT_HD void stable_normal(float ax, float ay, float az, float bx, float by, float bz, float cx, float cy, float cz, float& nx,
                         float& ny, float& nz) {
  const float ab_x = mul_rn(az, by), ab_y = mul_rn(ax, bz), ab_z = mul_rn(ay, bx);
  const float bc_x = mul_rn(bz, cy), bc_y = mul_rn(bx, cz), bc_z = mul_rn(by, cx);
  const float cab_x = msub(ay, bz, ab_x), cab_y = msub(az, bx, ab_y), cab_z = msub(ax, by, ab_z);
  const float cbc_x = msub(by, cz, bc_x), cbc_y = msub(bz, cx, bc_y), cbc_z = msub(bx, cy, bc_z);
  nx = fabsf(ab_x) < fabsf(bc_x) ? cab_x : cbc_x;
  ny = fabsf(ab_y) < fabsf(bc_y) ? cab_y : cbc_y;
  nz = fabsf(ab_z) < fabsf(bc_z) ? cab_z : cbc_z;
}

RT_HD bool tri_test_pluecker(const Ray& r, float tfar, float p0x, float p0y, float p0z, float p1x, float p1y, float p1z,
                             float p2x, float p2y, float p2z, PlueckerHit& h) {
  const float v0x = sub_rn(p0x, r.ox), v0y = sub_rn(p0y, r.oy), v0z = sub_rn(p0z, r.oz);
  const float v1x = sub_rn(p1x, r.ox), v1y = sub_rn(p1y, r.oy), v1z = sub_rn(p1z, r.oz);
  const float v2x = sub_rn(p2x, r.ox), v2y = sub_rn(p2y, r.oy), v2z = sub_rn(p2z, r.oz);
  const float e0x = sub_rn(v2x, v0x), e0y = sub_rn(v2y, v0y), e0z = sub_rn(v2z, v0z);
  const float e1x = sub_rn(v0x, v1x), e1y = sub_rn(v0y, v1y), e1z = sub_rn(v0z, v1z);
  const float e2x = sub_rn(v1x, v2x), e2y = sub_rn(v1y, v2y), e2z = sub_rn(v1z, v2z);
  // U = dot(cross(e0, v2+v0), D) etc.
  const float s0x = add_rn(v2x, v0x), s0y = add_rn(v2y, v0y), s0z = add_rn(v2z, v0z);
  const float s1x = add_rn(v0x, v1x), s1y = add_rn(v0y, v1y), s1z = add_rn(v0z, v1z);
  const float s2x = add_rn(v1x, v2x), s2y = add_rn(v1y, v2y), s2z = add_rn(v1z, v2z);
  const float U = dot3(msub(e0y, s0z, mul_rn(e0z, s0y)), msub(e0z, s0x, mul_rn(e0x, s0z)), msub(e0x, s0y, mul_rn(e0y, s0x)),
                       r.dx, r.dy, r.dz);
  const float V = dot3(msub(e1y, s1z, mul_rn(e1z, s1y)), msub(e1z, s1x, mul_rn(e1x, s1z)), msub(e1x, s1y, mul_rn(e1y, s1x)),
                       r.dx, r.dy, r.dz);
  const float W = dot3(msub(e2y, s2z, mul_rn(e2z, s2y)), msub(e2z, s2x, mul_rn(e2x, s2z)), msub(e2x, s2y, mul_rn(e2y, s2x)),
                       r.dx, r.dy, r.dz);
  const float UVW = add_rn(add_rn(U, V), W);
  const float eps = mul_rn(1.1920929e-07f, fabsf(UVW));
  const float mn = fminf(fminf(U, V), W), mx = fmaxf(fmaxf(U, V), W);
  if (!((mn >= -eps) | (mx <= eps))) return false;
  float ngx, ngy, ngz;
  stable_normal(e0x, e0y, e0z, e1x, e1y, e1z, e2x, e2y, e2z, ngx, ngy, ngz);
  const float d = dot3(ngx, ngy, ngz, r.dx, r.dy, r.dz);
  const float den = add_rn(d, d);
  const float T0 = dot3(v0x, v0y, v0z, ngx, ngy, ngz);
  const float T = add_rn(T0, T0);
  const float t = mul_rn(rcp_rn(den), T);
  if (!((r.tnear <= t) & (t <= tfar) & (den != 0.0f))) return false;
  h.t = t; h.U = U; h.V = V; h.UVW = UVW; h.ngx = ngx; h.ngy = ngy; h.ngz = ngz;
  return true;
}
RT_HD void pluecker_uv(const PlueckerHit& h, float& u, float& v) {   // PlueckerHitM::finalize
  const float rcpUVW = fabsf(h.UVW) < kMinRcpInput ? 0.0f : rcp_rn(h.UVW);
  u = fminf(mul_rn(h.U, rcpUVW), 1.0f);
  v = fminf(mul_rn(h.V, rcpUVW), 1.0f);
}

// ------------------------------------------------------------------------------------------------
// round linear curve segment (RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE): __roundline_internal::intersectConeSphere restated for
// one segment (kernels/geometry/roundline_intersector.h:560-650; cone :296-343, end spheres :350-395, neighbour cones
// :137-205, normals / u :432-480).  Geometry = cone touching the spheres p0/r0 and p1/r1 plus the end sphere at p1 (plus
// the one at p0 when there is no left neighbour), minus the capped cones of the neighbouring segments.  Backface culling
// of curves is off in the reference's default build, so both the entry and the exit surface are candidates; a closest-hit
// query takes the first candidate inside [tnear, tfar] exactly as the reference's epilog sequence does (:614-640).
// ------------------------------------------------------------------------------------------------
struct CurveHit { float t, u, ngx, ngy, ngz, v = 0.0f; };   // v: only the ribbons of cubic curves report one (linear curves: 0)
struct CurveVtx { float x, y, z, r; };

// Every product / sum below is an explicitly rounded fp32 operation (mul_rn / add_rn / sub_rn, dot products as the
// reference's madd chain): the compiler may not contract them, so the device evaluates exactly the expressions of the C
// oracle -- hit/miss decisions of near-tangent rays depend on the rounding of B*B - 4*A*C and of the clip tests.
struct ConeGeo {   // ConeGeometry<M> (:100-205)
  float p0x, p0y, p0z, dPx, dPy, dPz, dPdP, r0, sqr_r0, r1, dr, r0dr, g;
  bool exists;     // the reference marks a missing neighbour with p = +inf
};
RT_HD ConeGeo cone_geo(const CurveVtx& a, const CurveVtx& b, bool exists) {
  ConeGeo c;
  c.p0x = a.x; c.p0y = a.y; c.p0z = a.z;
  c.dPx = sub_rn(b.x, a.x); c.dPy = sub_rn(b.y, a.y); c.dPz = sub_rn(b.z, a.z);
  c.dPdP = dot3(c.dPx, c.dPy, c.dPz, c.dPx, c.dPy, c.dPz);
  c.r0 = a.r; c.sqr_r0 = mul_rn(a.r, a.r); c.r1 = b.r; c.dr = sub_rn(b.r, a.r);
  c.r0dr = mul_rn(c.r0, c.dr); c.g = sub_rn(c.dPdP, mul_rn(c.dr, c.dr));
  c.exists = exists;
  return c;
}
RT_HD bool cone_clipped_by_plane(const ConeGeo& c, float px, float py, float pz) {           // isClippedByPlane (:137-144)
  const float y = dot3(sub_rn(px, c.p0x), sub_rn(py, c.p0y), sub_rn(pz, c.p0z), c.dPx, c.dPy, c.dPz);
  return c.exists & (y > -c.r0dr);
}
RT_HD bool cone_inside_capped(const ConeGeo& c, float px, float py, float pz) {              // isInsideCappedCone (:190-202)
  const float qx = sub_rn(px, c.p0x), qy = sub_rn(py, c.p0y), qz = sub_rn(pz, c.p0z);
  const float y = dot3(qx, qy, qz, c.dPx, c.dPy, c.dPz);
  const float cap0 = add_rn(-c.r0dr, 1.1920929e-07f), cap1 = add_rn(mul_rn(-c.r1, c.dr), c.dPdP);
  const float qq = dot3(qx, qy, qz, qx, qy, qz);
  return c.exists & (y > cap0) & (y < cap1) &
         (sub_rn(mul_rn(qq, c.g), mul_rn(y, y)) < add_rn(mul_rn(c.dPdP, c.sqr_r0), mul_rn(mul_rn(2.0f, c.r0dr), y)));
}

RT_HD bool curve_test(float ox, float oy, float oz, float dx, float dy, float dz, float tnear, float tfar, const CurveVtx& v0,
                      const CurveVtx& v1, bool hasL, const CurveVtx& vL, bool hasR, const CurveVtx& vR, CurveHit& h) {
  const float dOdO = dot3(dx, dy, dz, dx, dy, dz);
  const float rcp_dOdO = rcp_rn(dOdO);
  // move the ray origin next to the segment (:571-574)
  const float cx = mul_rn(0.5f, add_rn(v0.x, v1.x)), cy = mul_rn(0.5f, add_rn(v0.y, v1.y)), cz = mul_rn(0.5f, add_rn(v0.z, v1.z));
  const float dt = mul_rn(dot3(sub_rn(cx, ox), sub_rn(cy, oy), sub_rn(cz, oz), dx, dy, dz), rcp_dOdO);
  const float qx = add_rn(ox, mul_rn(dt, dx)), qy = add_rn(oy, mul_rn(dt, dy)), qz = add_rn(oz, mul_rn(dt, dz));
  const ConeGeo c = cone_geo(v0, v1, true);
  const float Ox = sub_rn(qx, c.p0x), Oy = sub_rn(qy, c.p0y), Oz = sub_rn(qz, c.p0z);
  const float OdP = dot3(c.dPx, c.dPy, c.dPz, Ox, Oy, Oz);
  const float dOdP = dot3(c.dPx, c.dPy, c.dPz, dx, dy, dz);
  const float yp = add_rn(OdP, c.r0dr);
  // ---- cone (:296-343)
  float t_cone_lower = INFINITY, t_cone_upper = -INFINITY;
  float t_cone_front = 0.0f, t_cone_back = 0.0f, y_cone_front = 0.0f, y_cone_back = 0.0f;
  bool validCone;
  {
    const float OO = dot3(Ox, Oy, Oz, Ox, Oy, Oz), OdO = dot3(dx, dy, dz, Ox, Oy, Oz);
    const float A = sub_rn(mul_rn(c.g, dOdO), mul_rn(dOdP, dOdP));
    const float B = mul_rn(2.0f, sub_rn(mul_rn(c.g, OdO), mul_rn(dOdP, yp)));
    const float C = sub_rn(sub_rn(sub_rn(mul_rn(c.g, OO), mul_rn(OdP, OdP)), mul_rn(c.sqr_r0, c.dPdP)), mul_rn(mul_rn(2.0f, c.r0dr), OdP));
    const float D = sub_rn(mul_rn(B, B), mul_rn(mul_rn(4.0f, A), C));
    validCone = (D >= 0.0f) & (c.g > 0.0f) & (fabsf(A) > kMinRcpInput);
    if (validCone) {
      const float Q = sqrtf(D), rcp_2A = rcp_rn(mul_rn(2.0f, A));
      t_cone_front = mul_rn(sub_rn(-B, Q), rcp_2A); y_cone_front = add_rn(yp, mul_rn(t_cone_front, dOdP));
      t_cone_back = mul_rn(add_rn(-B, Q), rcp_2A);  y_cone_back = add_rn(yp, mul_rn(t_cone_back, dOdP));
      if ((y_cone_front > -1.1920929e-07f) & (y_cone_front <= c.g)) t_cone_lower = t_cone_front;
      if ((y_cone_back > -1.1920929e-07f) & (y_cone_back <= c.g)) t_cone_upper = t_cone_back;
    }
  }
  if (!(validCone | (c.g <= 0.0f))) return false;        // a cone entirely inside its end sphere still has the sphere (:579-581)
  // ---- cone hits inside the neighbouring capped cones are inside the curve (:583-592)
  const ConeGeo coneL = cone_geo(v0, vL, hasL), coneR = cone_geo(v1, vR, hasR);
  if (validCone) {
    const float lx = add_rn(qx, mul_rn(t_cone_lower, dx)), ly = add_rn(qy, mul_rn(t_cone_lower, dy)), lz = add_rn(qz, mul_rn(t_cone_lower, dz));
    const float ux = add_rn(qx, mul_rn(t_cone_upper, dx)), uy = add_rn(qy, mul_rn(t_cone_upper, dy)), uz = add_rn(qz, mul_rn(t_cone_upper, dz));
    if (cone_inside_capped(coneL, lx, ly, lz) | cone_inside_capped(coneR, lx, ly, lz)) t_cone_lower = INFINITY;
    if (cone_inside_capped(coneL, ux, uy, uz) | cone_inside_capped(coneR, ux, uy, uz)) t_cone_upper = -INFINITY;
  }
  // ---- end sphere at p1, clipped by the right neighbour's start plane (:350-372)
  float t_sph1_lower = INFINITY, t_sph1_upper = -INFINITY, t_sph1_front, t_sph1_back;
  {
    const float O1x = sub_rn(qx, v1.x), O1y = sub_rn(qy, v1.y), O1z = sub_rn(qz, v1.z);
    const float O1dO = dot3(O1x, O1y, O1z, dx, dy, dz);
    const float h2 = sub_rn(mul_rn(O1dO, O1dO), mul_rn(dOdO, sub_rn(dot3(O1x, O1y, O1z, O1x, O1y, O1z), mul_rn(c.r1, c.r1))));
    const float rhs1 = h2 >= 0.0f ? sqrtf(h2) : -INFINITY;
    t_sph1_front = mul_rn(sub_rn(-O1dO, rhs1), rcp_dOdO);
    t_sph1_back = mul_rn(add_rn(-O1dO, rhs1), rcp_dOdO);
    if ((h2 >= 0.0f) & (add_rn(yp, mul_rn(t_sph1_front, dOdP)) > c.g) &
        !cone_clipped_by_plane(coneR, add_rn(qx, mul_rn(t_sph1_front, dx)), add_rn(qy, mul_rn(t_sph1_front, dy)), add_rn(qz, mul_rn(t_sph1_front, dz))))
      t_sph1_lower = t_sph1_front;
    if ((h2 >= 0.0f) & (add_rn(yp, mul_rn(t_sph1_back, dOdP)) > c.g) &
        !cone_clipped_by_plane(coneR, add_rn(qx, mul_rn(t_sph1_back, dx)), add_rn(qy, mul_rn(t_sph1_back, dy)), add_rn(qz, mul_rn(t_sph1_back, dz))))
      t_sph1_upper = t_sph1_back;
  }
  // ---- begin sphere at p0 when the curve starts here (:374-395, :598-601)
  float t_sph0_lower = INFINITY, t_sph0_upper = -INFINITY, t_sph0_front = 0.0f, t_sph0_back = 0.0f;
  if (!hasL) {
    const float O1dO = dot3(Ox, Oy, Oz, dx, dy, dz);
    const float h2 = sub_rn(mul_rn(O1dO, O1dO), mul_rn(dOdO, sub_rn(dot3(Ox, Oy, Oz, Ox, Oy, Oz), mul_rn(c.r0, c.r0))));
    const float rhs1 = h2 >= 0.0f ? sqrtf(h2) : -INFINITY;
    t_sph0_front = mul_rn(sub_rn(-O1dO, rhs1), rcp_dOdO);
    t_sph0_back = mul_rn(add_rn(-O1dO, rhs1), rcp_dOdO);
    if ((h2 >= 0.0f) & (add_rn(yp, mul_rn(t_sph0_front, dOdP)) < 0.0f)) t_sph0_lower = t_sph0_front;
    if ((h2 >= 0.0f) & (add_rn(yp, mul_rn(t_sph0_back, dOdP)) < 0.0f)) t_sph0_upper = t_sph0_back;
  }
  // ---- CSG union, range test, first candidate (:603-625)
  const float t_lower = fminf(t_cone_lower, fminf(t_sph0_lower, t_sph1_lower));
  const float t_upper = fmaxf(t_cone_upper, fmaxf(t_sph0_upper, t_sph1_upper));
  const bool valid_lower = (tnear <= add_rn(dt, t_lower)) & (add_rn(dt, t_lower) <= tfar) & (t_lower != INFINITY);
  const bool valid_upper = (tnear <= add_rn(dt, t_upper)) & (add_rn(dt, t_upper) <= tfar) & (t_upper != -INFINITY);
  if (!(valid_lower | valid_upper)) return false;
  const float t_first = valid_lower ? t_lower : t_upper;
  const bool cone_hit = (t_first == t_cone_lower) | (t_first == t_cone_upper);
  const bool sph0_hit = (t_first == t_sph0_lower) | (t_first == t_sph0_upper);
  if (cone_hit) {                                          // Ng_cone / u_cone (:432-447, :470-478)
    const float y = valid_lower ? y_cone_front : y_cone_back, t = valid_lower ? t_cone_front : t_cone_back;
    h.ngx = sub_rn(mul_rn(c.g, add_rn(Ox, mul_rn(t, dx))), mul_rn(c.dPx, y));
    h.ngy = sub_rn(mul_rn(c.g, add_rn(Oy, mul_rn(t, dy))), mul_rn(c.dPy, y));
    h.ngz = sub_rn(mul_rn(c.g, add_rn(Oz, mul_rn(t, dz))), mul_rn(c.dPz, y));
    h.u = fminf(fmaxf(mul_rn(y, rcp_rn(c.g)), 0.0f), 1.0f);
  } else if (sph0_hit) {
    const float t = valid_lower ? t_sph0_front : t_sph0_back;
    h.ngx = sub_rn(add_rn(qx, mul_rn(t, dx)), v0.x); h.ngy = sub_rn(add_rn(qy, mul_rn(t, dy)), v0.y); h.ngz = sub_rn(add_rn(qz, mul_rn(t, dz)), v0.z);
    h.u = 0.0f;
  } else {
    const float t = valid_lower ? t_sph1_front : t_sph1_back;
    h.ngx = sub_rn(add_rn(qx, mul_rn(t, dx)), v1.x); h.ngy = sub_rn(add_rn(qy, mul_rn(t, dy)), v1.y); h.ngz = sub_rn(add_rn(qz, mul_rn(t, dz)), v1.z);
    h.u = 1.0f;
  }
  h.t = add_rn(dt, t_first);
  return true;
}

// flat linear curve segment (RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE): FlatLinearCurveIntersector1::intersect
// (kernels/geometry/line_intersector.h:38-89) with CurvePrecalculations1 (curve_intersector_precalculations.h:15-28) restated
// for one segment -- a ray-facing ribbon: the end points go to ray space (frame of the normalised direction, z = ray
// parameter), the closest point of the projected segment to the origin decides.  Explicitly rounded like curve_test.
RT_HD bool flat_curve_test(float ox, float oy, float oz, float dx_, float dy_, float dz_, float tnear, float tfar, const CurveVtx& v0,
                           const CurveVtx& v1, CurveHit& h) {
  const float depth_scale = rcp_rn(sqrtf(dot3(dx_, dy_, dz_, dx_, dy_, dz_)));
  const float Nx = mul_rn(depth_scale, dx_), Ny = mul_rn(depth_scale, dy_), Nz = mul_rn(depth_scale, dz_);
  // frame(N) (linearspace3.h:117-124): dx0 = (0, N.z, -N.y), dx1 = (-N.z, 0, N.x)
  const bool first = dot3(0.0f, Nz, -Ny, 0.0f, Nz, -Ny) > dot3(-Nz, 0.0f, Nx, -Nz, 0.0f, Nx);
  const float sx = first ? 0.0f : -Nz, sy = first ? Nz : 0.0f, sz = first ? -Ny : Nx;
  const float il = rcp_rn(sqrtf(dot3(sx, sy, sz, sx, sy, sz)));
  const float ax = mul_rn(sx, il), ay = mul_rn(sy, il), az = mul_rn(sz, il);                                  // dx
  float bx = msub(Ny, az, mul_rn(Nz, ay)), by = msub(Nz, ax, mul_rn(Nx, az)), bz = msub(Nx, ay, mul_rn(Ny, ax));   // cross(N, dx)
  const float jl = rcp_rn(sqrtf(dot3(bx, by, bz, bx, by, bz)));
  bx = mul_rn(bx, jl); by = mul_rn(by, jl); bz = mul_rn(bz, jl);                                              // dy
  const float zx = mul_rn(Nx, depth_scale), zy = mul_rn(Ny, depth_scale), zz = mul_rn(Nz, depth_scale);      // vz
  const float a0 = sub_rn(v0.x, ox), a1 = sub_rn(v0.y, oy), a2 = sub_rn(v0.z, oz);
  const float c0 = sub_rn(v1.x, ox), c1 = sub_rn(v1.y, oy), c2 = sub_rn(v1.z, oz);
  const float p0x = dot3(a0, a1, a2, ax, ay, az), p0y = dot3(a0, a1, a2, bx, by, bz), p0z = dot3(a0, a1, a2, zx, zy, zz);
  const float p1x = dot3(c0, c1, c2, ax, ay, az), p1y = dot3(c0, c1, c2, bx, by, bz), p1z = dot3(c0, c1, c2, zx, zy, zz);
  const float vx = sub_rn(p1x, p0x), vy = sub_rn(p1y, p0y), vz = sub_rn(p1z, p0z), vw = sub_rn(v1.r, v0.r);
  const float d0 = fma_rn(-p0x, vx, mul_rn(-p0y, vy)), d1 = fma_rn(vx, vx, mul_rn(vy, vy));
  const float u = fminf(fmaxf(mul_rn(d0, rcp_rn(d1)), 0.0f), 1.0f);
  const float px = fma_rn(u, vx, p0x), py = fma_rn(u, vy, p0y), t = fma_rn(u, vz, p0z), rr = fma_rn(u, vw, v0.r);
  const float d2 = fma_rn(px, px, mul_rn(py, py));
  if (!((d2 <= mul_rn(rr, rr)) & (tnear <= t) & (t <= tfar))) return false;
  if (!(t > mul_rn(mul_rn(2.0f, rr), depth_scale))) return false;      // EMBREE_CURVE_SELF_INTERSECTION_AVOIDANCE_FACTOR = 2.0
  const float Tx = sub_rn(v1.x, v0.x), Ty = sub_rn(v1.y, v0.y), Tz = sub_rn(v1.z, v0.z);
  if (!((Tx != 0.0f) | (Ty != 0.0f) | (Tz != 0.0f))) return false;     // denormalised segment
  h.t = t; h.u = u; h.ngx = Tx; h.ngy = Ty; h.ngz = Tz;
  return true;
}

// ------------------------------------------------------------------------------------------------
// point primitives (RTC_GEOMETRY_TYPE_SPHERE_POINT / _DISC_POINT / _ORIENTED_DISC_POINT): SphereIntersector1
// (kernels/geometry/sphere_intersector.h:76-140), DiscIntersector1 ray-facing (disc_intersector.h:85-131) and oriented
// (:133-170) restated for one point.  kind: 0 sphere, 1 ray-facing disc, 2 oriented disc (n = its normal).  u = v = 0.
// Without a filter callback the sphere's back hit is only ever offered when it does not lie behind the accepted front hit,
// so the first valid hit is the result.  Explicitly rounded like the curve tests: bit-identical to oracle point_intersect.
RT_HD bool point_test(float ox, float oy, float oz, float dx, float dy, float dz, float tnear, float tfar, float cx, float cy, float cz,
                      float radius, float nx, float ny, float nz, int kind, CurveHit& h) {
  h.u = 0.0f; h.v = 0.0f;
  const float c0x = sub_rn(cx, ox), c0y = sub_rn(cy, oy), c0z = sub_rn(cz, oz);
  if (kind == 2) {
    const float divisor = dot3(dx, dy, dz, nx, ny, nz);
    if (divisor == 0.0f) return false;
    const float t = dot3(c0x, c0y, c0z, nx, ny, nz) / divisor;
    if (!((tnear <= t) & (t <= tfar))) return false;
    const float qx = sub_rn(fma_rn(dx, t, ox), cx), qy = sub_rn(fma_rn(dy, t, oy), cy), qz = sub_rn(fma_rn(dz, t, oz), cz);
    if (!(dot3(qx, qy, qz, qx, qy, qz) < mul_rn(radius, radius))) return false;
    h.t = t; h.ngx = nx; h.ngy = ny; h.ngz = nz;
    return true;
  }
  const float rd2 = rcp_rn(dot3(dx, dy, dz, dx, dy, dz));
  const float projC0 = mul_rn(dot3(c0x, c0y, c0z, dx, dy, dz), rd2);
  if (kind == 1 && !((tnear <= projC0) & (projC0 <= tfar))) return false;
  const float px = fma_rn(-projC0, dx, c0x), py = fma_rn(-projC0, dy, c0y), pz = fma_rn(-projC0, dz, c0z);
  const float l2 = dot3(px, py, pz, px, py, pz), r2 = mul_rn(radius, radius);
  if (!(l2 <= r2)) return false;
  if (kind == 1) {
    h.t = projC0; h.ngx = -dx; h.ngy = -dy; h.ngz = -dz;
    return true;
  }
  const float td = sqrtf(mul_rn(sub_rn(r2, l2), rd2)), t_front = sub_rn(projC0, td), t_back = add_rn(projC0, td);
  const bool front = (tnear <= t_front) & (t_front <= tfar), back = (tnear <= t_back) & (t_back <= tfar);
  if (!(front | back)) return false;
  const float s = front ? -td : td;
  h.t = front ? t_front : t_back;
  h.ngx = fma_rn(s, dx, -px); h.ngy = fma_rn(s, dy, -py); h.ngz = fma_rn(s, dz, -pz);
  return true;
}

// ------------------------------------------------------------------------------------------------
// flat cubic curves (RTC_GEOMETRY_TYPE_FLAT_BEZIER_CURVE / _BSPLINE_ / _CATMULL_ROM_ / _HERMITE_): intersect_ribbon
// (kernels/geometry/curve_intersector_ribbon.h:73-190) restated for one curve.  The curve is tessellated into N =
// tessellation rate segments at u = j / N; the control points go to ray space (CurvePrecalculations1: frame of the
// normalised direction, z = ray parameter), every segment becomes a ray-facing quad p +- r * n (n = normalised 2D normal of
// the curve derivative at the segment ends) and is intersected with the z axis (intersect_quad_backface_culling,
// quad_intersector.h:14-84, with O = 0, D = (0, 0, 1)).  Segments are processed in chunks of 8 as the reference's
// 8-wide loop does: inside a chunk the smallest t wins (lowest segment on a tie, select_min), and a chunk's winner
// shortens the ray for the next chunk (the epilog writes ray.tfar).  The basis weights come from a table built by the
// host exactly as the reference builds its own at start-up (PrecomputedBezierBasis, subdiv/bezier_curve.cpp:8-27 and the
// B-spline / Catmull-Rom twins): tab[k][j], k = 0..3 position weights, 4..7 derivative weights, j = 0..N.  Hermite curves
// enter as the Bezier control points (p0, p0 + t0/3, p1 - t1/3, p1) the reference converts them to (hermite_curve.h).
// Every operation is explicitly rounded, so the device and the C oracle evaluate the same expressions.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxTess = 16;                         // PrecomputedBezierBasis::N
enum CurveBasis : uint32_t { BASIS_BEZIER = 0, BASIS_BSPLINE = 1, BASIS_CATMULL_ROM = 2 };

// basis derivative weights at parameter u (BezierBasis / BSplineBasis / CatmullRomBasis ::derivative): the hit's Ng = dP/du
RT_HD void curve_basis_derivative(uint32_t basis, float u, float b[4]) {
  const float t = u, s = sub_rn(1.0f, u);
  if (basis == BASIS_BEZIER) {
    const float st = mul_rn(s, t), ss = mul_rn(s, s), tt = mul_rn(t, t);
    b[0] = mul_rn(3.0f, -ss); b[1] = mul_rn(3.0f, fma_rn(-2.0f, st, ss)); b[2] = mul_rn(3.0f, msub(2.0f, st, tt)); b[3] = mul_rn(3.0f, tt);
  } else if (basis == BASIS_BSPLINE) {
    const float st = mul_rn(s, t), ss = mul_rn(s, s), tt = mul_rn(t, t);
    b[0] = mul_rn(0.5f, -ss); b[1] = mul_rn(0.5f, sub_rn(-tt, mul_rn(4.0f, st)));
    b[2] = mul_rn(0.5f, add_rn(ss, mul_rn(4.0f, st))); b[3] = mul_rn(0.5f, tt);
  } else {
    const float st = mul_rn(s, t), ss = mul_rn(s, s), tt = mul_rn(t, t);
    b[0] = mul_rn(0.5f, add_rn(-ss, mul_rn(2.0f, st)));
    b[1] = mul_rn(0.5f, add_rn(mul_rn(mul_rn(2.0f, t), sub_rn(mul_rn(3.0f, t), 5.0f)), mul_rn(3.0f, tt)));
    b[2] = mul_rn(0.5f, sub_rn(mul_rn(mul_rn(2.0f, s), add_rn(mul_rn(3.0f, t), 2.0f)), mul_rn(3.0f, ss)));
    b[3] = mul_rn(0.5f, add_rn(mul_rn(-2.0f, st), tt));
  }
}
// basis position / derivative weights at u as the reference's start-up tables hold them (scalar code of the base library:
// BezierBasis::eval etc. with unfused products; the derivative of the Bezier basis uses madd / msub)
RT_HD void curve_basis_table_entry(uint32_t basis, float u, float c[4], float d[4]) {
  const float t = u, s = sub_rn(1.0f, u);
  if (basis == BASIS_BEZIER) {
    c[0] = mul_rn(mul_rn(s, s), s); c[1] = mul_rn(mul_rn(3.0f, t), mul_rn(s, s));
    c[2] = mul_rn(mul_rn(3.0f, mul_rn(t, t)), s); c[3] = mul_rn(mul_rn(t, t), t);
    const float st = mul_rn(s, t), ss = mul_rn(s, s), tt = mul_rn(t, t);
    d[0] = mul_rn(3.0f, -ss); d[1] = mul_rn(3.0f, add_rn(mul_rn(-2.0f, st), ss)); d[2] = mul_rn(3.0f, sub_rn(mul_rn(2.0f, st), tt)); d[3] = mul_rn(3.0f, tt);
  } else if (basis == BASIS_BSPLINE) {
    const float sss = mul_rn(mul_rn(s, s), s), ttt = mul_rn(mul_rn(t, t), t);
    const float sts = mul_rn(mul_rn(s, t), s), tst = mul_rn(mul_rn(t, s), t);
    const float k = 1.0f / 6.0f;
    c[0] = mul_rn(k, sss);
    c[1] = mul_rn(k, add_rn(add_rn(mul_rn(4.0f, sss), ttt), add_rn(mul_rn(12.0f, sts), mul_rn(6.0f, tst))));
    c[2] = mul_rn(k, add_rn(add_rn(mul_rn(4.0f, ttt), sss), add_rn(mul_rn(12.0f, tst), mul_rn(6.0f, sts))));
    c[3] = mul_rn(k, ttt);
    curve_basis_derivative(basis, u, d);
  } else {
    c[0] = mul_rn(0.5f, mul_rn(mul_rn(-t, s), s));
    c[1] = mul_rn(0.5f, add_rn(2.0f, mul_rn(mul_rn(t, t), sub_rn(mul_rn(3.0f, t), 5.0f))));
    c[2] = mul_rn(0.5f, add_rn(2.0f, mul_rn(mul_rn(s, s), sub_rn(mul_rn(3.0f, s), 5.0f))));
    c[3] = mul_rn(0.5f, mul_rn(mul_rn(-s, t), t));
    curve_basis_derivative(basis, u, d);
  }
}
// tab[8][n + 1] for tessellation rate n (u = j / n as float(j) / float(n), bezier_curve.cpp:14)
RT_HD void curve_basis_table(uint32_t basis, int n, float* tab) {
  for (int j = 0; j <= n; ++j) {
    float c[4], d[4];
    curve_basis_table_entry(basis, (float)j / (float)n, c, d);
    for (int k = 0; k < 4; ++k) { tab[k * (n + 1) + j] = c[k]; tab[(4 + k) * (n + 1) + j] = d[k]; }
  }
}

struct RaySpace { float ax, ay, az, bx, by, bz, zx, zy, zz, depth_scale; };
// CurvePrecalculations1 (curve_intersector_precalculations.h:15-28); same operations as in flat_curve_test above
RT_HD RaySpace curve_ray_space(float dx_, float dy_, float dz_) {
  RaySpace q;
  q.depth_scale = rcp_rn(sqrtf(dot3(dx_, dy_, dz_, dx_, dy_, dz_)));
  const float Nx = mul_rn(q.depth_scale, dx_), Ny = mul_rn(q.depth_scale, dy_), Nz = mul_rn(q.depth_scale, dz_);
  const bool first = dot3(0.0f, Nz, -Ny, 0.0f, Nz, -Ny) > dot3(-Nz, 0.0f, Nx, -Nz, 0.0f, Nx);
  const float sx = first ? 0.0f : -Nz, sy = first ? Nz : 0.0f, sz = first ? -Ny : Nx;
  const float il = rcp_rn(sqrtf(dot3(sx, sy, sz, sx, sy, sz)));
  q.ax = mul_rn(sx, il); q.ay = mul_rn(sy, il); q.az = mul_rn(sz, il);
  float bx = msub(Ny, q.az, mul_rn(Nz, q.ay)), by = msub(Nz, q.ax, mul_rn(Nx, q.az)), bz = msub(Nx, q.ay, mul_rn(Ny, q.ax));
  const float jl = rcp_rn(sqrtf(dot3(bx, by, bz, bx, by, bz)));
  q.bx = mul_rn(bx, jl); q.by = mul_rn(by, jl); q.bz = mul_rn(bz, jl);
  q.zx = mul_rn(Nx, q.depth_scale); q.zy = mul_rn(Ny, q.depth_scale); q.zz = mul_rn(Nz, q.depth_scale);
  return q;
}

// weighted sum of the four control values: madd(c0, v0, madd(c1, v1, madd(c2, v2, c3 * v3))) (bezier_curve.h:512-526)
RT_HD float curve_blend(const float* w, int stride, float v0, float v1, float v2, float v3) {
  return fma_rn(w[0], v0, fma_rn(w[stride], v1, fma_rn(w[2 * stride], v2, mul_rn(w[3 * stride], v3))));
}

// `seg` >= 0 restricts the test to that one tessellation segment: the BVH holds every segment of a curve as its own
// primitive (tight boxes around thin diagonal ribbons instead of one box per curve -- the job the reference gives to its
// oriented-bounds hair BVH), and the closest hit over the segments is the closest hit of the curve.  seg < 0: all of them
// (the host instantiation the tests compare with the oracle).
RT_HD bool flat_cubic_test(float ox, float oy, float oz, float dx_, float dy_, float dz_, float tnear, float tfar, const CurveVtx cp[4],
                           uint32_t basis, int N, const float* tab, CurveHit& h, int seg = -1) {
  const RaySpace rs = curve_ray_space(dx_, dy_, dz_);
  // control points in ray space (xfm_pr, bezier_curve.h:216-223); w = radius
  float qx[4], qy[4], qz[4], qw[4];
  float amax = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float a0 = sub_rn(cp[k].x, ox), a1 = sub_rn(cp[k].y, oy), a2 = sub_rn(cp[k].z, oz);
    qx[k] = dot3(a0, a1, a2, rs.ax, rs.ay, rs.az); qy[k] = dot3(a0, a1, a2, rs.bx, rs.by, rs.bz); qz[k] = dot3(a0, a1, a2, rs.zx, rs.zy, rs.zz);
    qw[k] = cp[k].r;
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(qx[k]), fabsf(qy[k])), fabsf(qz[k])));
  }
  const float eps = mul_rn(mul_rn(4.0f, 1.1920929e-07f), amax);
  const int st = N + 1;
  bool ishit = false;
  float ray_tfar = tfar;
  for (int i0 = seg < 0 ? 0 : (seg & ~7); i0 < (seg < 0 ? N : seg + 1); i0 += 8) {
    bool any = false;
    float bt = 0.0f, bu = 0.0f, bv = 0.0f;
    int bj = 0;
    const int i1 = seg >= 0 ? seg + 1 : ((i0 + 8 < N) ? i0 + 8 : N);
    for (int j = seg >= 0 ? seg : i0; j < i1; ++j) {
      const float* c0 = tab + j;           // weights of the segment's first point, +1: of its second point
      const float p0x = curve_blend(c0, st, qx[0], qx[1], qx[2], qx[3]), p0y = curve_blend(c0, st, qy[0], qy[1], qy[2], qy[3]);
      const float p0z = curve_blend(c0, st, qz[0], qz[1], qz[2], qz[3]), p0w = curve_blend(c0, st, qw[0], qw[1], qw[2], qw[3]);
      const float p1x = curve_blend(c0 + 1, st, qx[0], qx[1], qx[2], qx[3]), p1y = curve_blend(c0 + 1, st, qy[0], qy[1], qy[2], qy[3]);
      const float p1z = curve_blend(c0 + 1, st, qz[0], qz[1], qz[2], qz[3]), p1w = curve_blend(c0 + 1, st, qw[0], qw[1], qw[2], qw[3]);
      // cylinder culling (:56-70): squared distance of the origin to the line p0 -> p1 in the projection plane
      const float ex = sub_rn(p1x, p0x), ey = sub_rn(p1y, p0y);
      const float num = msub(ex, p0y, mul_rn(ey, p0x)), den2 = fma_rn(ex, ex, mul_rn(ey, ey));
      const float rmax = fmaxf(p0w, p1w);
      if (!(mul_rn(num, num) <= mul_rn(mul_rn(rmax, rmax), den2))) continue;
      const float* d0 = tab + 4 * st + j;
      float t0x = curve_blend(d0, st, qx[0], qx[1], qx[2], qx[3]), t0y = curve_blend(d0, st, qy[0], qy[1], qy[2], qy[3]);
      const float t0z = curve_blend(d0, st, qz[0], qz[1], qz[2], qz[3]);
      float t1x = curve_blend(d0 + 1, st, qx[0], qx[1], qx[2], qx[3]), t1y = curve_blend(d0 + 1, st, qy[0], qy[1], qy[2], qy[3]);
      const float t1z = curve_blend(d0 + 1, st, qz[0], qz[1], qz[2], qz[3]);
      if (fmaxf(fmaxf(fabsf(t0x), fabsf(t0y)), fabsf(t0z)) < eps) { t0x = ex; t0y = ey; }   // vanishing derivative: the chord (:100-101)
      if (fmaxf(fmaxf(fabsf(t1x), fabsf(t1y)), fabsf(t1z)) < eps) { t1x = ex; t1y = ey; }
      // unit normals of the projected tangents, n = (dy, -dx, 0)
      const float l0 = rcp_rn(sqrtf(fma_rn(t0y, t0y, mul_rn(t0x, t0x)))), l1 = rcp_rn(sqrtf(fma_rn(t1y, t1y, mul_rn(t1x, t1x))));
      const float n0x = mul_rn(t0y, l0), n0y = mul_rn(-t0x, l0), n1x = mul_rn(t1y, l1), n1y = mul_rn(-t1x, l1);
      // quad corners: va = lp0, vb = lp1, vc = up1, vd = up0 (:106-112); z is untouched (n.z = 0)
      const float vax = fma_rn(p0w, n0x, p0x), vay = fma_rn(p0w, n0y, p0y), vaz = p0z;
      const float vbx = fma_rn(p1w, n1x, p1x), vby = fma_rn(p1w, n1y, p1y), vbz = p1z;
      const float vcx = fma_rn(-p1w, n1x, p1x), vcy = fma_rn(-p1w, n1y, p1y), vcz = p1z;
      const float vdx = fma_rn(-p0w, n0x, p0x), vdy = fma_rn(-p0w, n0y, p0y), vdz = p0z;
      // intersect_quad_backface_culling with O = 0, D = (0,0,1): dot(x, D) = x.z
      const float edbx = sub_rn(vbx, vdx), edby = sub_rn(vby, vdy);
      const float WW = msub(vdx, edby, mul_rn(vdy, edbx));
      const bool sel = WW <= 0.0f;
      const float v0x = sel ? vax : vcx, v0y = sel ? vay : vcy, v0z = sel ? vaz : vcz;
      const float v1x = sel ? vbx : vdx, v1y = sel ? vby : vdy, v1z = sel ? vbz : vdz;
      const float v2x = sel ? vdx : vbx, v2y = sel ? vdy : vby, v2z = sel ? vdz : vbz;
      const float e0x = sub_rn(v2x, v0x), e0y = sub_rn(v2y, v0y), e0z = sub_rn(v2z, v0z);
      const float e1x = sub_rn(v0x, v1x), e1y = sub_rn(v0y, v1y), e1z = sub_rn(v0z, v1z);
      const float U = msub(v0x, e0y, mul_rn(v0y, e0x)), V = msub(v1x, e1y, mul_rn(v1y, e1x));
      if (!(fmaxf(U, V) <= 0.0f)) continue;
      const float ngx = msub(e1y, e0z, mul_rn(e1z, e0y)), ngy = msub(e1z, e0x, mul_rn(e1x, e0z)), ngz = msub(e1x, e0y, mul_rn(e1y, e0x));
      const float den = ngz, rcpDen = rcp_rn(den);
      const float t = mul_rn(rcpDen, dot3(v0x, v0y, v0z, ngx, ngy, ngz));
      if (!((tnear <= t) & (t <= ray_tfar) & (den != 0.0f))) continue;
      float u = mul_rn(U, rcpDen), v = mul_rn(V, rcpDen);
      if (!sel) { u = sub_rn(1.0f, u); v = sub_rn(1.0f, v); }
      const float r = fma_rn(sub_rn(1.0f, u), p0w, mul_rn(u, p1w));            // lerp(p0.w, p1.w, u), math.h
      if (!(t > mul_rn(mul_rn(2.0f, r), rs.depth_scale))) continue;        // EMBREE_CURVE_SELF_INTERSECTION_AVOIDANCE_FACTOR = 2.0
      if (!any || t < bt) { any = true; bt = t; bu = u; bv = v; bj = j; }   // select_min: the first lane on equal t
    }
    if (any) {
      ishit = true;
      ray_tfar = bt;
      h.t = bt;
      h.u = mul_rn(add_rn(add_rn((float)(bj - i0), bu), (float)i0), 1.0f / (float)N);   // RibbonHit::finalize (:27-32)
      h.v = fma_rn(2.0f, bv, -1.0f);
    }
  }
  if (!ishit) return false;
  float b[4];
  curve_basis_derivative(basis, h.u, b);                                   // Ng = curve3D.eval_du(u): the tangent
  h.ngx = fma_rn(b[0], cp[0].x, fma_rn(b[1], cp[1].x, fma_rn(b[2], cp[2].x, mul_rn(b[3], cp[3].x))));
  h.ngy = fma_rn(b[0], cp[0].y, fma_rn(b[1], cp[1].y, fma_rn(b[2], cp[2].y, mul_rn(b[3], cp[3].y))));
  h.ngz = fma_rn(b[0], cp[0].z, fma_rn(b[1], cp[1].z, fma_rn(b[2], cp[2].z, mul_rn(b[3], cp[3].z))));
  return true;
}

// ------------------------------------------------------------------------------------------------
// round cubic curves (RTC_GEOMETRY_TYPE_ROUND_BEZIER_CURVE / _BSPLINE_ / _CATMULL_ROM_ / _HERMITE_): SweepCurve1Intersector1
// (kernels/geometry/curve_intersector_sweep.h:446-470).  The curve is the sweep of a sphere of radius r(u) along P(u).
// intersect_bezier_recursive_jacobian (:146-316, the 8-wide form of the AVX paths: 7 sub-segments per level, two levels, a third
// where the inner cylinder is grazed) bounds every sub-segment by an outer and an inner cylinder (cylinder.h:119-195) cut by the
// cap half-planes (plane.h:33-55) and starts a Newton iteration on (u, t) from the entry and the exit of the outer cylinder
// (intersect_bezier_iterative_jacobian, :59-140: at most 5 steps, converged when |f| and |g| fall below their error
// estimates).  Every accepted hit shortens the ray at once.  Explicitly rounded operations, operation for operation the C
// oracle's round_cubic_intersect.
// ------------------------------------------------------------------------------------------------
constexpr int kSweepW = 8;
RT_HD float lerp_rn(float a, float b, float t) { return fma_rn(sub_rn(1.0f, t), a, mul_rn(t, b)); }   // math/emath.h lerp
RT_HD void curve_basis_eval(uint32_t basis, float u, float b[4]) {    // BSplineBasis::eval / CatmullRomBasis::eval (live, not tabulated)
  const float t = u, s = sub_rn(1.0f, u);
  if (basis == BASIS_BSPLINE) {
    const float sss = mul_rn(mul_rn(s, s), s), ttt = mul_rn(mul_rn(t, t), t), k = 1.0f / 6.0f;
    const float sts = mul_rn(mul_rn(s, t), s), tst = mul_rn(mul_rn(t, s), t);
    b[0] = mul_rn(k, sss);
    b[1] = mul_rn(k, add_rn(add_rn(mul_rn(4.0f, sss), ttt), add_rn(mul_rn(12.0f, sts), mul_rn(6.0f, tst))));
    b[2] = mul_rn(k, add_rn(add_rn(mul_rn(4.0f, ttt), sss), add_rn(mul_rn(12.0f, tst), mul_rn(6.0f, sts))));
    b[3] = mul_rn(k, ttt);
  } else {
    b[0] = mul_rn(0.5f, mul_rn(mul_rn(-t, s), s));
    b[1] = mul_rn(0.5f, add_rn(2.0f, mul_rn(mul_rn(t, t), sub_rn(mul_rn(3.0f, t), 5.0f))));
    b[2] = mul_rn(0.5f, add_rn(2.0f, mul_rn(mul_rn(s, s), sub_rn(mul_rn(3.0f, s), 5.0f))));
    b[3] = mul_rn(0.5f, mul_rn(mul_rn(-s, t), t));
  }
}
RT_HD void curve_basis_derivative2(uint32_t basis, float u, float b[4]) {
  const float t = u, s = sub_rn(1.0f, u);
  if (basis == BASIS_BEZIER) { b[0] = mul_rn(6.0f, s); b[1] = mul_rn(6.0f, fma_rn(-2.0f, s, t)); b[2] = mul_rn(6.0f, fma_rn(-2.0f, t, s)); b[3] = mul_rn(6.0f, t); }
  else if (basis == BASIS_BSPLINE) { b[0] = s; b[1] = sub_rn(t, mul_rn(2.0f, s)); b[2] = sub_rn(s, mul_rn(2.0f, t)); b[3] = t; }
  else { b[0] = add_rn(mul_rn(-3.0f, t), 2.0f); b[1] = sub_rn(mul_rn(9.0f, t), 5.0f); b[2] = add_rn(mul_rn(-9.0f, t), 4.0f); b[3] = sub_rn(mul_rn(3.0f, t), 1.0f); }
}
// curve.eval(u, P, dPdu, ddPdu) on xyz + radius; ddP may be null
RT_HD void cubic_eval(const float cp[4][4], uint32_t basis, float u, float P[4], float dP[4], float* ddP) {
  if (basis == BASIS_BEZIER) {   // de Casteljau (bezier_curve.h:424-440)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float p10 = lerp_rn(cp[0][c], cp[1][c], u), p11 = lerp_rn(cp[1][c], cp[2][c], u), p12 = lerp_rn(cp[2][c], cp[3][c], u);
      const float p20 = lerp_rn(p10, p11, u), p21 = lerp_rn(p11, p12, u);
      P[c] = lerp_rn(p20, p21, u); dP[c] = mul_rn(3.0f, sub_rn(p21, p20));
    }
  } else {
    float b[4], d[4];
    curve_basis_eval(basis, u, b); curve_basis_derivative(basis, u, d);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      P[c] = fma_rn(b[0], cp[0][c], fma_rn(b[1], cp[1][c], fma_rn(b[2], cp[2][c], mul_rn(b[3], cp[3][c]))));
      dP[c] = fma_rn(d[0], cp[0][c], fma_rn(d[1], cp[1][c], fma_rn(d[2], cp[2][c], mul_rn(d[3], cp[3][c]))));
    }
  }
  if (ddP) {
    float dd[4];
    curve_basis_derivative2(basis, u, dd);
#pragma unroll
    for (int c = 0; c < 4; ++c) ddP[c] = fma_rn(dd[0], cp[0][c], fma_rn(dd[1], cp[1][c], fma_rn(dd[2], cp[2][c], mul_rn(dd[3], cp[3][c]))));
  }
}
RT_HD float dot3v(const float* a, const float* b) { return dot3(a[0], a[1], a[2], b[0], b[1], b[2]); }
RT_HD void cross3v(const float* a, const float* b, float* o) {
  o[0] = msub(a[1], b[2], mul_rn(a[2], b[1])); o[1] = msub(a[2], b[0], mul_rn(a[0], b[2])); o[2] = msub(a[0], b[1], mul_rn(a[1], b[0]));
}
struct SweepState { const float* dir; float tnear, tfar, dt; const float (*cp)[4]; uint32_t basis; float P_err, upper_w; bool found; CurveHit hit; };
RT_HD bool sweep_jacobian(SweepState& w, float u, float t) {
  const float* dir = w.dir;
  const float length_ray_dir = sqrtf(dot3v(dir, dir));
  const float k16 = 16.0f * 1.1920929e-07f;
  for (int it = 0; it < 5; ++it) {
    const float Q[3] = {mul_rn(t, dir[0]), mul_rn(t, dir[1]), mul_rn(t, dir[2])};
    const float Q_err = mul_rn(mul_rn(k16, length_ray_dir), t);
    float P[4], dP[4], ddP[4];
    cubic_eval(w.cp, w.basis, u, P, dP, ddP);
    const float R[3] = {sub_rn(Q[0], P[0]), sub_rn(Q[1], P[1]), sub_rn(Q[2], P[2])};
    const float RR = dot3v(R, R);
    const float len_R = sqrtf(RR);
    const float R_err = fmaxf(Q_err, w.P_err);
    const float dRdu[3] = {-dP[0], -dP[1], -dP[2]};
    const float dPdu2 = dot3v(dP, dP), rcp_len = rcp_rn(sqrtf(dPdu2));
    const float T[3] = {mul_rn(dP[0], rcp_len), mul_rn(dP[1], rcp_len), mul_rn(dP[2], rcp_len)};
    const float pdp = dot3v(dP, ddP), kk = mul_rn(rcp_rn(dPdu2), rcp_rn(sqrtf(dPdu2)));      // dnormalize (vec3fa.h:357-362)
    const float dTdu[3] = {mul_rn(sub_rn(mul_rn(dPdu2, ddP[0]), mul_rn(pdp, dP[0])), kk), mul_rn(sub_rn(mul_rn(dPdu2, ddP[1]), mul_rn(pdp, dP[1])), kk),
                           mul_rn(sub_rn(mul_rn(dPdu2, ddP[2]), mul_rn(pdp, dP[2])), kk)};
    const float cos_err = mul_rn(w.P_err, rcp_len);
    const float f = dot3v(R, T);
    const float f_err = add_rn(add_rn(mul_rn(len_R, w.P_err), R_err), mul_rn(cos_err, add_rn(1.0f, len_R)));
    const float dfdu = add_rn(dot3v(dRdu, T), dot3v(R, dTdu));
    const float dfdt = dot3v(dir, T);
    const float K = sub_rn(RR, mul_rn(f, f));
    const float dKdu = sub_rn(dot3v(R, dRdu), mul_rn(f, dfdu));
    const float dKdt = sub_rn(dot3v(R, dir), mul_rn(f, dfdt));
    const float rsqrt_K = rcp_rn(sqrtf(K));
    const float g = sub_rn(sqrtf(K), P[3]);
    const float g_err = add_rn(add_rn(R_err, f_err), mul_rn(k16, w.upper_w));
    const float dgdu = sub_rn(mul_rn(dKdu, rsqrt_K), dP[3]);
    const float dgdt = mul_rn(dKdt, rsqrt_K);
    const float rdet = rcp_rn(sub_rn(mul_rn(dfdu, dgdt), mul_rn(dfdt, dgdu)));
    const float du = mul_rn(sub_rn(mul_rn(dgdt, f), mul_rn(dfdt, g)), rdet), dtt = mul_rn(sub_rn(mul_rn(dfdu, g), mul_rn(dgdu, f)), rdet);
    u = sub_rn(u, du); t = sub_rn(t, dtt);
    if (fabsf(f) < f_err && fabsf(g) < g_err) {
      t = add_rn(t, w.dt);
      if (!(w.tnear <= t && t <= w.tfar)) return false;
      if (!(u >= 0.0f && u <= 1.0f)) return false;
      const float rl = rcp_rn(sqrtf(RR));
      const float Rn[3] = {mul_rn(R[0], rl), mul_rn(R[1], rl), mul_rn(R[2], rl)};
      const float U[3] = {fma_rn(dP[3], Rn[0], dP[0]), fma_rn(dP[3], Rn[1], dP[1]), fma_rn(dP[3], Rn[2], dP[2])};
      float V[3], Ng[3];
      cross3v(dP, Rn, V);
      cross3v(V, U, Ng);
      w.hit.t = t; w.hit.u = u; w.hit.v = 0.0f; w.hit.ngx = Ng[0]; w.hit.ngy = Ng[1]; w.hit.ngz = Ng[2];
      w.tfar = t; w.found = true;
      return true;
    }
  }
  return false;
}
// CylinderN::intersect for one lane, ray origin 0
RT_HD bool sweep_cylinder(const float* p0, const float* p1, float r, const float* dir, float& tlo, float& thi, float& u0, float* Ng0, float& u1, float* Ng1) {
  const float rr = mul_rn(r, r);
  const float e[3] = {sub_rn(p1[0], p0[0]), sub_rn(p1[1], p0[1]), sub_rn(p1[2], p0[2])};
  const float rl = rcp_rn(sqrtf(dot3v(e, e)));
  const float dP[3] = {mul_rn(e[0], rl), mul_rn(e[1], rl), mul_rn(e[2], rl)};
  const float O[3] = {-p0[0], -p0[1], -p0[2]};
  const float dOdO = dot3v(dir, dir), OdO = dot3v(dir, O), OO = dot3v(O, O), dOz = dot3v(dP, dir), Oz = dot3v(dP, O);
  const float A = sub_rn(dOdO, mul_rn(dOz, dOz)), B = mul_rn(2.0f, sub_rn(OdO, mul_rn(dOz, Oz))), C = sub_rn(sub_rn(OO, mul_rn(Oz, Oz)), rr);
  const float D = sub_rn(mul_rn(B, B), mul_rn(mul_rn(4.0f, A), C));
  bool valid = D >= 0.0f;
  const float Q = sqrtf(D), rcp_2A = rcp_rn(mul_rn(2.0f, A));
  const float t0 = mul_rn(sub_rn(-B, Q), rcp_2A), t1 = mul_rn(add_rn(-B, Q), rcp_2A);
  u0 = mul_rn(fma_rn(t0, dOz, Oz), rl);
  u1 = mul_rn(fma_rn(t1, dOz, Oz), rl);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    Ng0[k] = sub_rn(mul_rn(t0, dir[k]), fma_rn(u0, e[k], p0[k]));
    Ng1[k] = sub_rn(mul_rn(t1, dir[k]), fma_rn(u1, e[k], p0[k]));
  }
  tlo = valid ? t0 : INFINITY; thi = valid ? t1 : -INFINITY;
  const float eps = mul_rn(16.0f * 1.1920929e-07f, fmaxf(fabsf(dOdO), fabsf(mul_rn(dOz, dOz))));
  if (valid && fabsf(A) < eps) {
    const bool inside = C <= 0.0f;
    tlo = inside ? -INFINITY : INFINITY; thi = inside ? INFINITY : -INFINITY;
    valid = inside;
  }
  return valid;
}
RT_HD void sweep_halfplane(const float* P, const float* N, const float* dir, float& lo, float& hi) {
  const float O[3] = {-P[0], -P[1], -P[2]};
  const float ON = dot3v(O, N), DN = dot3v(dir, N);
  const bool eps = fabsf(DN) < 1e-18f;
  const float t = mul_rn(-ON, rcp_rn(DN));
  lo = (eps || DN < 0.0f) ? -INFINITY : t;
  hi = (eps || DN > 0.0f) ? INFINITY : t;
}
RT_HD int sweep_select_min(uint32_t valid, const float* v) {
  int best = -1;
  for (int i = 0; i < kSweepW; ++i) if ((valid >> i) & 1u) if (best < 0 || v[i] < v[best]) best = i;
  return best;
}
// first-level sub-segments of the sweep: the BVH primitives of one round cubic curve (rtk_device.h prims_per_curve)
constexpr int kRoundSubSegs = kSweepW - 1;
// `lane` >= 0 restricts the FIRST subdivision level to that one of its 7 sub-segments: the BVH holds every first-level
// sub-segment of a round curve as its own primitive (tight boxes), and the closest hit over them is the closest hit of the curve
// (the same converged roots; only the order in which candidates shorten the ray differs).  lane < 0: the whole curve.
RT_HD bool round_cubic_test(float ox, float oy, float oz, float dx, float dy, float dz, float tnear, float tfar, const CurveVtx cpv[4], uint32_t basis,
                            CurveHit& h, int lane = -1) {
  const float org[3] = {ox, oy, oz}, dir[3] = {dx, dy, dz};
  // move the ray origin next to the curve (:458-462); center(): bezier_curve.h:173, bspline_curve.h:94, catmullrom_curve.h:102
  const float cin[4][3] = {{cpv[0].x, cpv[0].y, cpv[0].z}, {cpv[1].x, cpv[1].y, cpv[1].z}, {cpv[2].x, cpv[2].y, cpv[2].z}, {cpv[3].x, cpv[3].y, cpv[3].z}};
  float co[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float c = basis == BASIS_CATMULL_ROM ? mul_rn(0.5f, add_rn(cin[0][k], cin[1][k])) : mul_rn(0.25f, add_rn(add_rn(add_rn(cin[0][k], cin[1][k]), cin[2][k]), cin[3][k]));
    co[k] = sub_rn(c, org[k]);
  }
  const float dt = mul_rn(dot3v(co, dir), rcp_rn(dot3v(dir, dir)));
  float cp[4][4];
  float amax = 0.0f, upw = -INFINITY;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int a = 0; a < 3; ++a) { cp[k][a] = sub_rn(cin[k][a], fma_rn(dt, dir[a], org[a])); amax = fmaxf(amax, fabsf(cp[k][a])); }
  }
  cp[0][3] = cpv[0].r; cp[1][3] = cpv[1].r; cp[2][3] = cpv[2].r; cp[3][3] = cpv[3].r;
  upw = fmaxf(fmaxf(cp[0][3], cp[1][3]), fmaxf(cp[2][3], cp[3][3]));
  SweepState w;
  w.dir = dir; w.tnear = tnear; w.tfar = tfar; w.dt = dt; w.cp = cp; w.basis = basis; w.found = false;
  w.P_err = mul_rn(16.0f * 1.1920929e-07f, amax); w.upper_w = upw;
  const uint32_t maxDepth = 2;
  struct Entry { uint32_t valid; float tlower[kSweepW]; float u0, u1; uint32_t depth; } stack[3];
  uint32_t sptr = 0, depth = 1;
  float u0 = 0.0f, u1 = 1.0f;
  bool first = true;
  const float k7 = 1.0f / (kSweepW - 1);
  while (first || sptr) {
    if (!first) {
      --sptr;
      uint32_t valid = stack[sptr].valid;
      for (int i = 0; i < kSweepW; ++i) if (!(add_rn(stack[sptr].tlower[i], dt) <= w.tfar)) valid &= ~(1u << i);
      if (!valid) continue;
      u0 = stack[sptr].u0; u1 = stack[sptr].u1; depth = stack[sptr].depth;
      const int i = sweep_select_min(valid, stack[sptr].tlower);
      valid &= ~(1u << i);
      stack[sptr].valid = valid;
      if (valid) ++sptr;
      const float a0 = lerp_rn(u0, u1, mul_rn((float)i, k7)), a1 = lerp_rn(u0, u1, mul_rn((float)(i + 1), k7));
      u0 = a0; u1 = a1;
    }
    first = false;
    const float dscale = mul_rn(sub_rn(u1, u0), 1.0f / (3.0f * (kSweepW - 1)));
    float P0[kSweepW][4], dP0[kSweepW][4];
    const bool one = lane >= 0 && depth == 1;                       // first level of a per-sub-segment primitive
    for (int i = one ? lane : 0; i < (one ? lane + 2 : kSweepW); ++i) {
      cubic_eval(cp, basis, lerp_rn(u0, u1, mul_rn((float)i, k7)), P0[i], dP0[i], nullptr);
      for (int a = 0; a < 4; ++a) dP0[i][a] = mul_rn(dP0[i][a], dscale);
    }
    uint32_t valid0 = 0, valid1 = 0, rec0 = 0, rec1 = 0;
    float tp0lo[kSweepW], tp1lo[kSweepW], tp1hi[kSweepW], uo0[kSweepW], uo1[kSweepW];
    for (int i = 0; i < kSweepW; ++i) { tp0lo[i] = tp1lo[i] = INFINITY; tp1hi[i] = -INFINITY; uo0[i] = uo1[i] = 0.0f; }
    for (int i = one ? lane : 0; i < (one ? lane + 1 : kSweepW - 1); ++i) {
      const float *A0 = P0[i], *A3 = P0[i + 1], *dA0 = dP0[i], *dA3 = dP0[i + 1];
      const float P1w = add_rn(A0[3], dA0[3]), P2w = sub_rn(A3[3], dA3[3]);
      const float e[3] = {sub_rn(A3[0], A0[0]), sub_rn(A3[1], A0[1]), sub_rn(A3[2], A0[2])};
      float n1[3], n2[3];
      cross3v(dA0, e, n1); cross3v(dA3, e, n2);
      const float rcp_ee = rcp_rn(dot3v(e, e));
      const float rr1 = mul_rn(dot3v(n1, n1), rcp_ee), rr2 = mul_rn(dot3v(n2, n2), rcp_ee);
      const float maxr12 = sqrtf(fmaxf(rr1, rr2));
      float r_outer = add_rn(fmaxf(fmaxf(A0[3], P1w), fmaxf(P2w, A3[3])), maxr12);
      float r_inner = sub_rn(fminf(fminf(A0[3], P1w), fminf(P2w, A3[3])), maxr12);
      r_outer = mul_rn(1.0f + 2.0f * 1.1920929e-07f, r_outer);
      r_inner = fmaxf(0.0f, mul_rn(1.0f - 2.0f * 1.1920929e-07f, r_inner));
      float tlo, thi, u_o0, u_o1, Ng_o0[3], Ng_o1[3];
      if (!sweep_cylinder(A0, A3, r_outer, dir, tlo, thi, u_o0, Ng_o0, u_o1, Ng_o1)) continue;
      float lo = fmaxf(sub_rn(w.tnear, dt), tlo), hi = fminf(sub_rn(w.tfar, dt), thi), hl, hh;
      sweep_halfplane(A0, dA0, dir, hl, hh);
      lo = fmaxf(lo, hl); hi = fminf(hi, hh);
      const float ndA3[3] = {-dA3[0], -dA3[1], -dA3[2]};
      sweep_halfplane(A3, ndA3, dir, hl, hh);
      lo = fmaxf(lo, hl); hi = fminf(hi, hh);
      if (!(lo <= hi)) continue;
      u_o0 = fminf(fmaxf(u_o0, 0.0f), 1.0f); u_o1 = fminf(fmaxf(u_o1, 0.0f), 1.0f);
      uo0[i] = lerp_rn(u0, u1, mul_rn(add_rn((float)i, u_o0), 1.0f / (float)kSweepW));
      uo1[i] = lerp_rn(u0, u1, mul_rn(add_rn((float)i, u_o1), 1.0f / (float)kSweepW));
      float ilo, ihi, ui0 = 0.0f, ui1 = 0.0f, Ng_i0[3] = {0.0f, 0.0f, 0.0f}, Ng_i1[3] = {0.0f, 0.0f, 0.0f};
      const bool valid_inner = sweep_cylinder(A0, A3, r_inner, dir, ilo, ihi, ui0, Ng_i0, ui1, Ng_i1);
      const bool unstable0 = !valid_inner || fabsf(dot3v(dir, Ng_i0)) < 0.3f;
      const bool unstable1 = !valid_inner || fabsf(dot3v(dir, Ng_i1)) < 0.3f;
      tp0lo[i] = lo; const float tp0hi = fminf(hi, ilo);
      tp1lo[i] = fmaxf(lo, ihi); tp1hi[i] = hi;
      const bool v0 = tp0lo[i] <= tp0hi, v1 = tp1lo[i] <= tp1hi[i];
      const uint32_t term0 = unstable0 ? maxDepth + 1 : maxDepth, term1 = unstable1 ? maxDepth + 1 : maxDepth;
      if (v0) { if (depth < term0) rec0 |= 1u << i; else valid0 |= 1u << i; }
      if (v1) { if (depth < term1) rec1 |= 1u << i; else valid1 |= 1u << i; }
    }
    if (!(valid0 | valid1 | rec0 | rec1)) continue;
    while (valid0) {
      const int i = sweep_select_min(valid0, tp0lo);
      valid0 &= ~(1u << i);
      sweep_jacobian(w, uo0[i], tp0lo[i]);
      for (int j = 0; j < kSweepW; ++j) if (!(add_rn(tp0lo[j], dt) <= w.tfar)) valid0 &= ~(1u << j);
    }
    for (int j = 0; j < kSweepW; ++j) if (!(add_rn(tp1lo[j], dt) <= w.tfar)) { valid1 &= ~(1u << j); rec1 &= ~(1u << j); }
    while (valid1) {
      const int i = sweep_select_min(valid1, tp1lo);
      valid1 &= ~(1u << i);
      sweep_jacobian(w, uo1[i], tp1hi[i]);
      for (int j = 0; j < kSweepW; ++j) if (!(add_rn(tp1lo[j], dt) <= w.tfar)) valid1 &= ~(1u << j);
    }
    for (int j = 0; j < kSweepW; ++j) {
      if (!(add_rn(tp0lo[j], dt) <= w.tfar)) rec0 &= ~(1u << j);
      if (!(add_rn(tp1lo[j], dt) <= w.tfar)) rec1 &= ~(1u << j);
    }
    if (rec0 | rec1) {
      stack[sptr].valid = rec0 | rec1;
      for (int j = 0; j < kSweepW; ++j) stack[sptr].tlower[j] = ((rec0 >> j) & 1u) ? tp0lo[j] : tp1lo[j];
      stack[sptr].u0 = u0; stack[sptr].u1 = u1; stack[sptr].depth = depth + 1;
      ++sptr;
    }
  }
  if (w.found) h = w.hit;
  return w.found;
}

// ------------------------------------------------------------------------------------------------
// Node8 encoding (build side)
// ------------------------------------------------------------------------------------------------
struct ChildBox { float lo[3], hi[3]; };

// per-slot leaf masks: 3 bytes at byte kNodeMaskByte + 3 s of the node
RT_HD void node_set_leafmask(Node8& nd, int s, uint32_t m24) {
  for (int k = 0; k < 3; ++k) {
    const int b = kNodeMaskByte + 3 * s + k;
    nd.w[b >> 2] |= ((m24 >> (8 * k)) & 0xFFu) << (8 * (b & 3));
  }
}
// the 24-bit mask of slot s in the low bits; bits 24..31 are NOT cleared (callers mask the union once)
RT_HD uint32_t node_leafmask_raw(const uint32_t* w, int s) {
  const int b = kNodeMaskByte + 3 * s;
  const uint32_t lo = w[b >> 2], hi = w[(b >> 2) + 1];
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(lo, hi, 8 * (b & 3));
#else
  return (uint32_t)((((uint64_t)hi << 32) | lo) >> (8 * (b & 3)));
#endif
}
// permute the 8 bits of x so that bit j moves to position j ^ k (k in 0..7)
RT_HD uint32_t xor_permute8(uint32_t x, uint32_t k) {
  if (k & 1u) x = ((x & 0x55u) << 1) | ((x >> 1) & 0x55u);
  if (k & 2u) x = ((x & 0x33u) << 2) | ((x >> 2) & 0x33u);
  if (k & 4u) x = ((x & 0x0Fu) << 4) | ((x >> 4) & 0x0Fu);
  return x;
}


// smallest biased exponent e such that (extent / 2^(e-127)) <= 255
RT_HD uint32_t grid_exponent(float extent) {
  if (!(extent > 0.0f)) return 1;                     // degenerate axis: any tiny scale works, q = 0
  // 2^k >= extent/255  ->  start from the exponent of extent/255 and bump while 255 * 2^k < extent
  float s = extent / 255.0f;
  uint32_t e = (f2u(s) >> 23) & 0xFF;
  if ((f2u(s) & 0x7FFFFF) != 0) e += 1;               // round the scale up to a power of two
  if (e < 1) e = 1;
  if (e > 254) e = 254;
  while (e < 254 && u2f(e << 23) * 255.0f < extent) e += 1;
  return e;
}

RT_HD float round_down_add(float p, float q, float s) {  // p + q*s rounded towards -inf
#if defined(__CUDA_ARCH__)
  return __fmaf_rd(q, s, p);
#else
  double d = (double)p + (double)q * (double)s; float f = (float)d; if ((double)f > d) f = nextafterf(f, -INFINITY); return f;
#endif
}
RT_HD float round_up_add(float p, float q, float s) {
#if defined(__CUDA_ARCH__)
  return __fmaf_ru(q, s, p);
#else
  double d = (double)p + (double)q * (double)s; float f = (float)d; if ((double)f < d) f = nextafterf(f, INFINITY); return f;
#endif
}

// Quantise n child boxes against the node box [plo, phi] and write the geometric part of the node.
// Conservative by construction: decoded lo <= true lo and decoded hi >= true hi (checked with directed rounding).
RT_HD void encode_node_boxes(Node8& nd, const float plo[3], const float phi[3], const ChildBox* cb, const uint8_t* slot_of,
                             int n) {
  uint32_t e[3];
  float scale[3], inv[3];
  for (int a = 0; a < 3; ++a) {
    e[a] = grid_exponent(phi[a] - plo[a]);
    // the subtraction above may round down: make sure the top grid line still covers phi
    while (e[a] < 254 && round_up_add(plo[a], 255.0f, u2f(e[a] << 23)) < phi[a]) e[a] += 1;
    scale[a] = u2f(e[a] << 23);
    inv[a] = 1.0f / scale[a];
  }
  nd.w[0] = f2u(plo[0]); nd.w[1] = f2u(plo[1]); nd.w[2] = f2u(plo[2]);
  nd.w[3] = (nd.w[3] & 0xFF000000u) | e[0] | (e[1] << 8) | (e[2] << 16);
  uint8_t q[6][8];
  for (int a = 0; a < 6; ++a) for (int s = 0; s < 8; ++s) q[a][s] = 0;
  for (int c = 0; c < n; ++c) {
    const int s = slot_of[c];
    for (int a = 0; a < 3; ++a) {
      int lo = (int)floorf((cb[c].lo[a] - plo[a]) * inv[a]);
      int hi = (int)ceilf((cb[c].hi[a] - plo[a]) * inv[a]);
      lo = lo < 0 ? 0 : (lo > 255 ? 255 : lo);
      hi = hi < 0 ? 0 : (hi > 255 ? 255 : hi);
      while (lo > 0 && round_up_add(plo[a], (float)lo, scale[a]) > cb[c].lo[a]) --lo;
      while (hi < 255 && round_down_add(plo[a], (float)hi, scale[a]) < cb[c].hi[a]) ++hi;
      q[a][s] = (uint8_t)lo;
      q[3 + a][s] = (uint8_t)hi;
    }
  }
  for (int a = 0; a < 6; ++a) {
    const uint32_t lo4 = q[a][0] | (q[a][1] << 8) | (q[a][2] << 16) | ((uint32_t)q[a][3] << 24);
    const uint32_t hi4 = q[a][4] | (q[a][5] << 8) | (q[a][6] << 16) | ((uint32_t)q[a][7] << 24);
    nd.w[kNodePlaneWord + 2 * a] = lo4;
    nd.w[kNodePlaneWord + 2 * a + 1] = hi4;
  }
}

// ------------------------------------------------------------------------------------------------
// LBVH: internal node i of the binary radix tree over n sorted 64-bit keys (duplicates are split by index), after
// Karras 2012; the reference's Morton builder splits at the highest differing bit the same way
// (kernels/builders/bvh_builder_morton.h:312-353).
// ------------------------------------------------------------------------------------------------
RT_HD int clz64(uint64_t x) {
#if defined(__CUDA_ARCH__)
  return __clzll((long long)x);
#else
  return x ? __builtin_clzll(x) : 64;
#endif
}
RT_HD int lbvh_delta(const uint64_t* keys, int n, int i, int j) {
  if (j < 0 || j >= n) return -1;
  const uint64_t x = keys[i] ^ keys[j];
  return x ? clz64(x) : 64 + clz32((uint32_t)(i ^ j));
}
RT_HD void lbvh_node(const uint64_t* keys, int n, int i, Node2* nodes) {
  const int d = (lbvh_delta(keys, n, i, i + 1) - lbvh_delta(keys, n, i, i - 1)) >= 0 ? 1 : -1;
  const int dmin = lbvh_delta(keys, n, i, i - d);
  int lmax = 2;
  while (lbvh_delta(keys, n, i, i + lmax * d) > dmin) lmax <<= 1;
  int l = 0;
  for (int t = lmax >> 1; t >= 1; t >>= 1)
    if (lbvh_delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
  const int j = i + l * d;
  const int dnode = lbvh_delta(keys, n, i, j);
  int s = 0;
  for (int t = (l + 1) >> 1;; t = (t + 1) >> 1) {
    if (lbvh_delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
    if (t == 1) break;
  }
  const int gamma = i + s * d + (d < 0 ? d : 0);
  const int first = i < j ? i : j, last = i < j ? j : i;
  const int left = (first == gamma) ? (n - 1 + gamma) : gamma;
  const int right = (last == gamma + 1) ? (n - 1 + gamma + 1) : (gamma + 1);
  Node2& nd = nodes[i];
  nd.left = left; nd.right = right;
  nd.first = (uint32_t)first; nd.count = (uint32_t)(last - first + 1); nd.pad = 0;
  nodes[left].parent = (uint32_t)i;
  nodes[right].parent = (uint32_t)i;
  if (i == 0) nd.parent = 0xFFFFFFFFu;
}

// Choose which BVH2 nodes become the (<= 8) children of one BVH8 node: start from the node's two children and
// repeatedly open the candidate with the largest surface area (the reference's heuristic for N-wide nodes,
// kernels/builders/bvh_builder_sah.h:252-279 "split the largest-area child until N children").
// A candidate with <= kMaxLeafTris primitives may stay closed and becomes a leaf slot.
RT_HD float half_area(const Node2& n) {
  const float dx = n.hix - n.lox, dy = n.hiy - n.loy, dz = n.hiz - n.loz;
  return dx * (dy + dz) + dy * dz;
}

// policy 0: open the largest-area candidate that has more than one primitive, whatever its size (leaves end up as
//           single triangles wherever slots are free);
// policy 1: first open only candidates that MUST be opened (> kMaxLeafTris primitives), largest area first, and keep
//           candidates of 2..3 primitives closed as multi-triangle leaf slots (fewer, fuller nodes at the bottom);
// policy 2: as 1, then spend the remaining slots on opening 2..3-primitive candidates by area.
RT_HD int select_children(const Node2* nodes, uint32_t root, uint32_t* cand /*[8]*/, int policy) {
  int n = 0;
  const Node2& r = nodes[root];
  if (r.right < 0) { cand[0] = root; return 1; }        // the build tree is a single leaf
  cand[n++] = (uint32_t)r.left;
  cand[n++] = (uint32_t)r.right;
  for (int phase = (policy == 0 ? 1 : 0); phase < 2; ++phase) {
    if (phase == 1 && policy == 1) break;
    while (n < 8) {
      int best = -1;
      float bestA = -1.0f;
      for (int i = 0; i < n; ++i) {
        const Node2& c = nodes[cand[i]];
        if (c.right < 0) continue;                         // a single primitive cannot be opened
        if (phase == 0 && c.count <= (uint32_t)kMaxLeafTris) continue;
        const float a = half_area(c);
        if (a > bestA) { bestA = a; best = i; }
      }
      if (best < 0) break;
      const Node2& c = nodes[cand[best]];
      cand[best] = (uint32_t)c.left;
      cand[n++] = (uint32_t)c.right;
    }
  }
  return n;
}

// ------------------------------------------------------------------------------------------------
// SAH-optimal collapse of the binary tree into 8-wide nodes (dynamic programme over the binary tree, after
// Ylitie et al. 2017, "Efficient incoherent ray traversal on GPUs through compressed wide BVHs", section 4):
//   F(n,i) = cheapest way to represent the subtree of binary node n as a forest of at most i roots, each root
//            either a leaf slot (<= kMaxLeafTris triangles, cost A*count*c_tri) or an internal BVH8 node
//            (cost A*c_node + F-forest of its <= 8 children).
// dp_node() fills F(n,1..8) and the 22-bit decision word of one binary node from its children's rows:
//   bit 0      : i == 1 -> 1 = internal BVH8 node, 0 = leaf slot
//   bits 3i-5.. : i in 2..8 -> 0 = "same as F(n,i-1)", k in 1..7 = give k roots to the left child, i-k to the right.
// The reference grows N-wide nodes greedily by area (bvh_builder_sah.h:252-279); with single-triangle leaf slots
// that leaves the bottom nodes a third full, the DP trades child count against leaf fill explicitly.
// ------------------------------------------------------------------------------------------------
RT_HD void dp_leaf(float area, float c_tri, float* F, uint32_t* dec) {
  for (int i = 0; i < 8; ++i) F[i] = area * c_tri;
  *dec = 0;
}
RT_HD void dp_node(float area, uint32_t count, const float* Fl, const float* Fr, float c_node, float c_tri, float* F,
                   uint32_t* dec) {
  float D[9];      // D[j]: best split of exactly-at-most j roots between the two children, j = 2..8
  uint32_t K[9];
  for (int j = 2; j <= 8; ++j) {
    float best = INFINITY;
    uint32_t bk = 1;
    for (int k = 1; k < j; ++k) {
      const float c = Fl[k - 1] + Fr[j - k - 1];
      if (c < best) { best = c; bk = (uint32_t)k; }
    }
    D[j] = best; K[j] = bk;
  }
  const float leaf = count <= (uint32_t)kMaxLeafTris ? area * (float)count * c_tri : INFINITY;
  const float inner = area * c_node + D[8];
  uint32_t d = 0;
  if (inner < leaf) { F[0] = inner; d |= 1u; } else F[0] = leaf;
  for (int i = 2; i <= 8; ++i) {
    if (D[i] < F[i - 2]) { F[i - 1] = D[i]; d |= K[i] << (3 * i - 5); }
    else F[i - 1] = F[i - 2];
  }
  // the children of n when n itself becomes an internal node: D[8] split, kept in bits 22..24
  d |= K[8] << 22;
  *dec = d;
}

// children of the BVH8 node rooted at binary node `root` according to the decision words
RT_HD int select_children_dp(const Node2* nodes, const uint32_t* dec, uint32_t root, uint32_t* cand /*[8]*/) {
  const Node2& r = nodes[root];
  if (r.right < 0) { cand[0] = root; return 1; }
  uint32_t st_n[8], st_i[8];
  int sp = 0, n = 0;
  const uint32_t k8 = (dec[root] >> 22) & 7u;
  st_n[sp] = (uint32_t)r.right; st_i[sp] = 8u - k8; ++sp;
  st_n[sp] = (uint32_t)r.left; st_i[sp] = k8; ++sp;
  while (sp > 0) {
    --sp;
    uint32_t c = st_n[sp], i = st_i[sp];
    for (;;) {
      const Node2& cn = nodes[c];
      if (cn.right < 0) { cand[n++] = c; break; }           // single primitive
      if (i == 1) { cand[n++] = c; break; }                   // one root: leaf slot or internal child (by count)
      const uint32_t k = (dec[c] >> (3 * i - 5)) & 7u;
      if (k == 0) { --i; continue; }                          // F(c,i) == F(c,i-1)
      st_n[sp] = (uint32_t)cn.right; st_i[sp] = i - k; ++sp;
      c = (uint32_t)cn.left; i = k;
    }
  }
  return n;
}

// Assign children to slots so that (slot ^ octant-mask) orders them front-to-back for every ray octant:
// greedy maximisation of dot(child centre - node centre, slot direction) (slot bit a set = +axis a).
RT_HD void assign_slots(const ChildBox* cb, int n, const float plo[3], const float phi[3], uint8_t* slot_of) {
  float cost[8][8];
  const float cx = 0.5f * (plo[0] + phi[0]), cy = 0.5f * (plo[1] + phi[1]), cz = 0.5f * (plo[2] + phi[2]);
  for (int c = 0; c < n; ++c) {
    const float dx = 0.5f * (cb[c].lo[0] + cb[c].hi[0]) - cx;
    const float dy = 0.5f * (cb[c].lo[1] + cb[c].hi[1]) - cy;
    const float dz = 0.5f * (cb[c].lo[2] + cb[c].hi[2]) - cz;
    for (int s = 0; s < 8; ++s)
      cost[c][s] = ((s & 1) ? dx : -dx) + ((s & 2) ? dy : -dy) + ((s & 4) ? dz : -dz);
  }
  uint32_t used_slots = 0, done = 0;
  for (int it = 0; it < n; ++it) {
    int bc = -1, bs = -1;
    float best = -INFINITY;
    for (int c = 0; c < n; ++c) {
      if (done & (1u << c)) continue;
      for (int s = 0; s < 8; ++s) {
        if (used_slots & (1u << s)) continue;
        if (cost[c][s] > best || bc < 0) { best = cost[c][s]; bc = c; bs = s; }
      }
    }
    slot_of[bc] = (uint8_t)bs;
    used_slots |= 1u << bs;
    done |= 1u << bc;
  }
}

// Emit BVH8 node q from the binary subtree src[q]: choose <= 8 children, give them octant-ordered slots, quantise
// their boxes, reserve the node ids of internal children / the triangle slots of leaf children through `alloc`
// (atomic bump counters on the device), and queue the internal children (src[child id] = binary node).
template <typename Alloc>
RT_HD void collapse_node(const Node2* n2, uint32_t* src, uint32_t q, Node8* n8, uint32_t* tri_src, const uint32_t* sortedA,
                         const uint32_t* sortedB, float inv_root_area, int policy, const uint32_t* dec, const Alloc& alloc) {
  const uint32_t root = src[q];
  uint32_t cand[8];
  const int n = dec ? select_children_dp(n2, dec, root, cand) : select_children(n2, root, cand, policy);
  const Node2 self = n2[root];
  const float plo[3] = {self.lox, self.loy, self.loz}, phi[3] = {self.hix, self.hiy, self.hiz};
  ChildBox cb[8];
  uint32_t cnt[8], first[8], half[8];  // half: which ping-pong half of the sorted ids holds the child's range
  for (int c = 0; c < n; ++c) {
    const Node2 ch = n2[cand[c]];
    cb[c].lo[0] = ch.lox; cb[c].lo[1] = ch.loy; cb[c].lo[2] = ch.loz;
    cb[c].hi[0] = ch.hix; cb[c].hi[1] = ch.hiy; cb[c].hi[2] = ch.hiz;
    cnt[c] = ch.count; first[c] = ch.first; half[c] = ch.pad;
  }
  uint8_t slot_of[8];
  assign_slots(cb, n, plo, phi, slot_of);
  // order children by slot; internal children and leaf triangles are numbered in slot order
  int child_at[8];
  for (int s = 0; s < 8; ++s) child_at[s] = -1;
  for (int c = 0; c < n; ++c) child_at[slot_of[c]] = c;
  uint32_t n_inner = 0, n_tris = 0, imask = 0;
  for (int s = 0; s < 8; ++s) {
    const int c = child_at[s];
    if (c < 0) continue;
    if (cnt[c] > (uint32_t)kMaxLeafTris) { imask |= 1u << s; ++n_inner; } else n_tris += cnt[c];
  }
  const uint32_t child_base = n_inner ? alloc.nodes(n_inner) : 0;
  const uint32_t tri_base = n_tris ? alloc.tris(n_tris) : 0;
  Node8 nd;
  for (int k = 0; k < 24; ++k) nd.w[k] = 0;
  encode_node_boxes(nd, plo, phi, cb, slot_of, n);
  nd.w[3] = (nd.w[3] & 0x00FFFFFFu) | (imask << 24);
  nd.w[4] = child_base; nd.w[5] = tri_base;
  uint32_t ir = 0, toff = 0;
  double sah = 0.0;
  for (int s = 0; s < 8; ++s) {
    const int c = child_at[s];
    if (c < 0) continue;
    if (imask & (1u << s)) {
      src[child_base + ir] = cand[c];
      ++ir;
    } else {
      const uint32_t k = cnt[c];
      node_set_leafmask(nd, s, ((1u << k) - 1u) << toff);
      const uint32_t* sorted = half[c] ? sortedB : sortedA;
      for (uint32_t t = 0; t < k; ++t) tri_src[tri_base + toff + t] = sorted[first[c] + t];
      toff += k;
      const float dx = cb[c].hi[0] - cb[c].lo[0], dy = cb[c].hi[1] - cb[c].lo[1], dz = cb[c].hi[2] - cb[c].lo[2];
      sah += (double)((dx * (dy + dz) + dy * dz) * inv_root_area) * k;
    }
  }
  n8[q] = nd;
  sah += (double)(half_area(self) * inv_root_area);
  alloc.sah(sah);
}

// ------------------------------------------------------------------------------------------------
// traversal (per ray).  `NodeLoad` / `TriLoad` abstract the 16-byte loads so the host emulation can use plain
// pointers and the device can use the read-only / cache-hinted path.
// ------------------------------------------------------------------------------------------------
struct u32x4 { uint32_t x, y, z, w; };
struct NodeW { uint32_t w[24]; };   // one node in registers (three 32-byte sectors)
struct TravStats { uint32_t nodes, tris; };

// Slab test of the 8 quantised children of one node; returns the hit mask in the layout
// [31:24] internal children ordered by traversal priority (slot s at bit 24 + (s ^ oct_inv), oct_inv = 7 - ray octant),
// [23:0] one bit per triangle of the node's leaf slots.
RT_HD uint32_t node_hitmask(const uint32_t* w, float ox, float oy, float oz, float idx, float idy, float idz, bool negx,
                            bool negy, bool negz, float tnear, float tfar, uint32_t oct_inv) {
  const uint32_t e = w[3];
  // per-axis: t = q * (2^e * idir) + (p - org) * idir
  //
  // Conservative to exact arithmetic (u = 2^-24).  Rounded to nearest, (p - org) * idir carries an absolute error of
  // up to ~2u |(p - org) idir|: with the origin inside a large node, far from p and close to a child face, that exceeds
  // any relative pad on the plane distance, and a box the ray enters is culled.  So the offset is computed twice, with
  // directed rounding: bn <= (p - org) idir <= bf exactly (the subtraction and the product are both rounded away from
  // the side each bound must lie on; which rounding of p - org gives which bound depends on the sign of idir).  Near
  // planes use bn, far planes bf.  What remains is relative: idir = (1/d)(1 + d0) and the FMA's rounding (1 + d1),
  // |di| <= u, so every computed near distance is <= max(t*, 0) (1 + u)^2 and every far distance >= t* (1 - u)^2
  // for t* >= 0 (t* the exact distance to the plane p + q 2^e).  The factor 1 + 6u on tmax covers both ends and its own
  // rounding: (1 - u)^3 (1 + 6u) >= (1 + u)^2, so tmin <= tmax whenever the exact interval is non-empty.
  // The triangle, quad, curve and point tests round too: they accept hits up to about an ulp of the coordinates outside
  // a primitive's box, which is an absolute error of the same kind.  So on every axis whose direction is not rcp_safe's
  // clamp the offsets are widened by 2^-22 of their magnitude (bn - 4u|bn|, bf + 4u|bf|); with that margin no hit the
  // reference finds is lost in the grid-aligned scenes of tests/test_traversal_bounds.py.  On a clamped axis (|1/dir| >= kRcpOfMin) the offsets stay exact: a ray lying in a face plane with a
  // zero direction component leaves or enters the box as the clamped direction says, and where p - org and the product
  // are exact the test equals the unpadded one.  The per-child work is unchanged.
  const float sx = u2f((e & 0xFFu) << 23) * idx;
  const float sy = u2f(((e >> 8) & 0xFFu) << 23) * idy;
  const float sz = u2f(((e >> 16) & 0xFFu) << 23) * idz;
  const float px = u2f(w[0]), py = u2f(w[1]), pz = u2f(w[2]);
  const float dlx = sub_rd(px, ox), dhx = sub_ru(px, ox);
  const float dly = sub_rd(py, oy), dhy = sub_ru(py, oy);
  const float dlz = sub_rd(pz, oz), dhz = sub_ru(pz, oz);
  const float kx = fabsf(idx) < kRcpOfMin ? 0x1p-22f : 0.0f, ky = fabsf(idy) < kRcpOfMin ? 0x1p-22f : 0.0f,
              kz = fabsf(idz) < kRcpOfMin ? 0x1p-22f : 0.0f;
  const float dnx = mul_rd(negx ? dhx : dlx, idx), dfx = mul_ru(negx ? dlx : dhx, idx);   // bounds of (p - org) idir
  const float dny = mul_rd(negy ? dhy : dly, idy), dfy = mul_ru(negy ? dly : dhy, idy);
  const float dnz = mul_rd(negz ? dhz : dlz, idz), dfz = mul_ru(negz ? dlz : dhz, idz);
  const float bnx = fma_rn(-kx, fabsf(dnx), dnx), bfx = fma_rn(kx, fabsf(dfx), dfx);       // near / far plane offsets
  const float bny = fma_rn(-ky, fabsf(dny), dny), bfy = fma_rn(ky, fabsf(dfy), dfy);
  const float bnz = fma_rn(-kz, fabsf(dnz), dnz), bfz = fma_rn(kz, fabsf(dfz), dfz);
  uint32_t leaf = 0, slots = 0;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    // near / far planes per axis picked by the ray's direction sign
    const uint32_t qlox = w[kNodePlaneWord + half], qloy = w[kNodePlaneWord + 2 + half], qloz = w[kNodePlaneWord + 4 + half];
    const uint32_t qhix = w[kNodePlaneWord + 6 + half], qhiy = w[kNodePlaneWord + 8 + half], qhiz = w[kNodePlaneWord + 10 + half];
    const uint32_t nx = negx ? qhix : qlox, fx = negx ? qlox : qhix;
    const uint32_t ny = negy ? qhiy : qloy, fy = negy ? qloy : qhiy;
    const uint32_t nz = negz ? qhiz : qloz, fz = negz ? qloz : qhiz;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int sh = 8 * j;
      const float tnx = fma_rn((float)((nx >> sh) & 0xFFu), sx, bnx);
      const float tny = fma_rn((float)((ny >> sh) & 0xFFu), sy, bny);
      const float tnz = fma_rn((float)((nz >> sh) & 0xFFu), sz, bnz);
      const float tfx = fma_rn((float)((fx >> sh) & 0xFFu), sx, bfx);
      const float tfy = fma_rn((float)((fy >> sh) & 0xFFu), sy, bfy);
      const float tfz = fma_rn((float)((fz >> sh) & 0xFFu), sz, bfz);
      const float tmin = fmaxf(fmaxf(tnx, tny), fmaxf(tnz, tnear));
      // 1.0000003f = 1 + 6u: the relative part of the bound above, for both ends of the interval
      const float tmax = fminf(fminf(tfx, tfy), fminf(tfz, tfar)) * 1.0000003f;
      if (tmin <= tmax) {
        leaf |= node_leafmask_raw(w, 4 * half + j);
        slots |= 1u << (4 * half + j);
      }
    }
  }
  return (xor_permute8(slots & (e >> 24), oct_inv) << 24) | (leaf & 0x00FFFFFFu);
}

// The node loop of one closest-hit (ANYHIT=false) or any-hit (ANYHIT=true) query, with the per-record test as a callable:
// `test(ti, tfar)` tests leaf record ti against the ray, `tfar` being the current hit distance, and returns true when it
// accepts the record; for a closest-hit query it has then lowered `tfar` to the hit's t and kept whatever the caller needs
// for the write-back.  idx / idy / idz are the ray's reciprocal directions (rcp_safe semantics).  Records are tested in
// the kernel's order: node children by priority, the triangles of a node highest bit first.  On a closest hit r.tfar is
// shrunk; any-hit returns true as soon as one record is accepted.
template <bool ANYHIT, bool STATS, typename NodeLoad, typename RecordTest>
RT_HD bool traverse_records(Ray& r, float idx, float idy, float idz, const NodeLoad& ldn, RecordTest& test, uint32_t root_valid,
                            TravStats* st) {
  if (!root_valid) return false;                                         // empty scene (bvh_intersector1.cpp:39)
  if (ANYHIT && r.tfar < 0.0f) return false;                             // already occluded (:128-129)
  const bool negx = idx < 0.0f, negy = idy < 0.0f, negz = idz < 0.0f;    // near/far plane selectors (node_intersector1.h:47-52)
  const uint32_t oct = (negx ? 1u : 0u) | (negy ? 2u : 0u) | (negz ? 4u : 0u);
  const float tnear_c = fmaxf(r.tnear, 0.0f);                            // TravRay clamps (bvh_intersector1.cpp:65)
  float tfar_c = fmaxf(r.tfar, 0.0f);
  float tfar_tri = r.tfar;                                               // the record test sees the raw value
  bool found = false;

  uint32_t stack_x[kStackSize], stack_y[kStackSize];
  int sp = 0;
  // node group: x = child_base, y = hits[31:24] | imask[7:0]; triangle group: x = tri_base, y = hits[23:0]
  // The root is entered as "child_base 0, imask 0, one pending internal child": slot decoding then yields node 0.
  uint32_t ngx = 0, ngy = 0x80000000u;
  uint32_t tgx = 0, tgy = 0;

  while (true) {
    if (ngy & 0xFF000000u) {
      const int bit = 31 - clz32(ngy);                                   // highest priority pending child
      ngy &= ~(1u << bit);
      if (ngy & 0xFF000000u) { stack_x[sp] = ngx; stack_y[sp] = ngy; ++sp; }
      const uint32_t slot = ((uint32_t)(bit - 24)) ^ (7u - oct);
      const uint32_t node_index = ngx + (uint32_t)popc32(ngy & 0xFFu & ((1u << slot) - 1u));
      const NodeW nw = ldn(node_index);
      if (STATS) st->nodes++;
      const uint32_t hm = node_hitmask(nw.w, r.ox, r.oy, r.oz, idx, idy, idz, negx, negy, negz, tnear_c, tfar_c, 7u - oct);
      ngx = nw.w[4];
      ngy = (hm & 0xFF000000u) | (nw.w[3] >> 24);
      tgx = nw.w[5];
      tgy = hm & 0x00FFFFFFu;
    } else {
      tgx = ngx; tgy = ngy; ngx = 0; ngy = 0;                            // popped entry was a triangle group
    }
    while (tgy) {
      const int tb = 31 - clz32(tgy);
      tgy &= ~(1u << tb);
      const uint32_t ti = tgx + (uint32_t)tb;
      if (STATS) st->tris++;
      if (test(ti, tfar_tri)) {
        if (ANYHIT) return true;
        tfar_c = fmaxf(tfar_tri, 0.0f);                                  // tray.tfar = ray.tfar (bvh_intersector1.cpp:105)
        found = true;
      }
    }
    if ((ngy & 0xFF000000u) == 0) {
      if (sp == 0) break;
      --sp;
      ngx = stack_x[sp]; ngy = stack_y[sp];
    }
  }
  if (found) r.tfar = tfar_tri;
  return found;
}

// One query over a triangle scene (the host emulation's loop): `ldt(ti, k)` loads word group k of record ti.  On a closest
// hit `hit` is filled and r.tfar shrunk; for any-hit the function returns true as soon as one triangle is accepted.
template <bool ANYHIT, bool STATS, bool ROBUST, typename NodeLoad, typename TriLoad>
RT_HD bool traverse(Ray& r, Hit& hit, const NodeLoad& ldn, const TriLoad& ldt, uint32_t root_valid, TravStats* st) {
  auto test = [&](uint32_t ti, float& tfar_tri) -> bool {
    const u32x4 a = ldt(ti, 0), b = ldt(ti, 1), c = ldt(ti, 2);
    if (ROBUST) {     // record holds v0, v1, v2 (Triangle4v); Pluecker test
      PlueckerHit ph;
      if (!tri_test_pluecker(r, tfar_tri, u2f(a.x), u2f(a.y), u2f(a.z), u2f(b.x), u2f(b.y), u2f(b.z), u2f(c.x), u2f(c.y), u2f(c.z), ph))
        return false;
      if ((c.w & r.mask) == 0) return false;
      if (ANYHIT) return true;
      hit.t = ph.t; pluecker_uv(ph, hit.u, hit.v);
      hit.ngx = ph.ngx; hit.ngy = ph.ngy; hit.ngz = ph.ngz;
      hit.primID = a.w; hit.geomID = b.w;
      tfar_tri = hit.t;
      return true;
    }
    TriHit th;
    if (!tri_test(r, tfar_tri, u2f(a.x), u2f(a.y), u2f(a.z), u2f(b.x), u2f(b.y), u2f(b.z), u2f(c.x), u2f(c.y), u2f(c.z), th))
      return false;
    if ((c.w & r.mask) == 0) return false;                               // ray mask (intersector_epilog.h:256-262)
    if (ANYHIT) return true;
    const float rcpAbsDen = 1.0f / th.absDen;                            // finalize(): t,u,v = T,U,V * rcp(absDen)
    hit.t = th.T * rcpAbsDen; hit.u = th.U * rcpAbsDen; hit.v = th.V * rcpAbsDen;
    hit.ngx = th.ngx; hit.ngy = th.ngy; hit.ngz = th.ngz;
    hit.primID = a.w; hit.geomID = b.w;
    tfar_tri = hit.t;                                                    // ray.tfar = hit.vt[i]
    return true;
  };
  return traverse_records<ANYHIT, STATS>(r, rcp_safe(r.dx), rcp_safe(r.dy), rcp_safe(r.dz), ldn, test, root_valid, st);
}

}  // namespace rtk
