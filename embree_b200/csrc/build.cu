// build.cu -- device-wide BVH construction for sm_90a.
//
// Replaces (reference paths): kernels/builders/primrefgen.cpp:14-60 + scene_triangle_mesh.h:194-215,293-305
// (PrimRef generation with the validity filter), kernels/builders/bvh_builder_morton.h:71-102,312-432
// (Morton codes, split at the highest differing bit), common/algorithms/parallel_sort.h:254-454 (8-bit LSD radix
// sort), kernels/builders/bvh_builder_sah.h:216-313 + heuristic_binning.h:17-393 (binned SAH, see build_sah.cu),
// kernels/geometry/triangle.h:98-120 (leaf fill) and kernels/bvh/bvh_node_aabb.h:33-116 (node emission).
//
// Pipeline (all on one stream, counts stay on the device except two scalar read-backs):
//   primref_gen -> morton_keys -> radix sort (8-bit digits, warp-match ranking) ->
//   { lbvh_hierarchy + refit | binned SAH top-down (build_sah.cu) } -> collapse to 96-byte BVH8 nodes
//   (ONE cooperative launch, grid-wide barrier per tree level; SAH-optimal child selection) -> leaf_pack
//   (48-byte triangle records).  A committed scene keeps the record -> primitive map and the level ranges of its
//   node array, so a later commit with unchanged topology can REFIT (refit_scene below) instead of rebuilding.
#include <cooperative_groups.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "rtk_device.h"
#include "two_level.h"

namespace rtk {

static std::atomic<unsigned long long> g_launches{0};
unsigned long long launch_count() { return g_launches.load(); }
void count_launch(unsigned n) { g_launches.fetch_add(n); }

#define CK(x)                                                                                        \
  do {                                                                                               \
    cudaError_t e_ = (x);                                                                            \
    if (e_ != cudaSuccess) {                                                                         \
      snprintf(errmsg, 256, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return (int)e_;                                                                                \
    }                                                                                                \
  } while (0)

// ---------------------------------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------------------------------
__host__ inline float ord2f_host(int i) { int j = i >= 0 ? i : i ^ 0x7FFFFFFF; float f; memcpy(&f, &j, 4); return f; }

struct BuildInfo {        // device-resident scalars of one build
  int geom_lo[3], geom_hi[3];   // ordered-int encoded bounds of all valid triangles
  int cent_lo[3], cent_hi[3];   // bounds of (lower + upper) -- "center2" as in primref.h:60-62
  uint32_t num_valid;
  uint32_t node_tail;           // BVH8 nodes allocated so far (== collapse queue tail)
  uint32_t tri_tail;            // triangle records allocated so far
  uint32_t pad;
  double sah;                   // accumulated SAH cost numerator
  int api_lo[3], api_hi[3];     // bounds of the non-instanced triangles only (rtcGetSceneBounds merges instance boxes on the host)
  uint32_t depth;               // BVH8 levels written by collapse_all
  uint32_t level_begin[kStackSize + 1];   // node id range of level l = [level_begin[l], level_begin[l+1])
};

__device__ __forceinline__ int find_geom(const uint32_t* __restrict__ offs, int ngeoms, uint32_t p) {
  int lo = 0, hi = ngeoms;  // offs has ngeoms+1 entries, offs[g] <= p < offs[g+1]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (offs[mid] <= p) lo = mid; else hi = mid;
  }
  return lo;
}

// ---------------------------------------------------------------------------------------------------
// per primitive kind: validity and box (primref_gen), leaf record (leaf_pack)
// ---------------------------------------------------------------------------------------------------
// all six box coordinates inside +-kFltLarge (isvalid(b), scene_curves.h:527)
__device__ __forceinline__ bool finite_box(const float lo[3], const float hi[3]) {
  return (lo[0] > -kFltLarge) & (hi[0] < kFltLarge) & (lo[1] > -kFltLarge) & (hi[1] < kFltLarge) & (lo[2] > -kFltLarge) & (hi[2] < kFltLarge);
}

// widen a box by `rel` of the magnitude of each coordinate
__device__ __forceinline__ void widen_rel(float lo[3], float hi[3], float rel) {
#pragma unroll
  for (int a = 0; a < 3; ++a) { lo[a] -= fabsf(lo[a]) * rel; hi[a] += fabsf(hi[a]) * rel; }
}

// point (x, y, z) through an instance's local2world (xfmPoint, common/math/affinespace.h:102) into w.  `pad` accumulates per axis a
// bound of the rounding error of this FMA chain and of the inverse map the trace kernel applies to the ray (to_object_space) -- 8 ulp
// of the summed term magnitudes, so the world-space box stays conservative for the object-space test even under cancellation
// (x*m0 ~ -p).
__device__ __forceinline__ void xfm_point(const float* xfm, float x, float y, float z, float w[3], float pad[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    w[a] = __fmaf_rn(x, xfm[a], __fmaf_rn(y, xfm[3 + a], __fmaf_rn(z, xfm[6 + a], xfm[9 + a])));
    pad[a] = fmaxf(pad[a], 9.6e-7f * (fabsf(x * xfm[a]) + fabsf(y * xfm[3 + a]) + fabsf(z * xfm[6 + a]) + fabsf(xfm[9 + a])));
  }
}

// instanced curve / point, and an instance of instance traversal: the box is in OBJECT space (where the record is tested); the BVH
// needs the world box of its eight corners through local2world `xfm` (xfmBounds, affinespace.h:106-118), widened by their pad
__device__ __forceinline__ bool xfm_box(const float* xfm, float lo[3], float hi[3]) {
  float wlo[3] = {INFINITY, INFINITY, INFINITY}, whi[3] = {-INFINITY, -INFINITY, -INFINITY}, pad[3] = {0.0f, 0.0f, 0.0f};
  for (int cnr = 0; cnr < 8; ++cnr) {
    float w[3];
    xfm_point(xfm, (cnr & 4) ? hi[0] : lo[0], (cnr & 2) ? hi[1] : lo[1], (cnr & 1) ? hi[2] : lo[2], w, pad);
#pragma unroll
    for (int a = 0; a < 3; ++a) { wlo[a] = fminf(wlo[a], w[a]); whi[a] = fmaxf(whi[a], w[a]); }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) { lo[a] = wlo[a] - pad[a]; hi[a] = whi[a] + pad[a]; }
  return finite_box(lo, hi);
}

// ---- triangles and quads (PRIM_TRIANGLE)
// object-space vertices of triangle lp; a quad's halves are (v0,v1,v3) and (v2,v1,v3), and the whole quad must be valid
// (scene_quad_mesh.h:186-203).  Valid when every index is in range and every vertex finite.
__device__ __forceinline__ bool load_tri_verts(const GeomDesc& g, uint32_t lp, float v[9]) {
  uint32_t i0, i1, i2;
  bool ok;
  if (g.is_quad) {
    const uint32_t* ip = reinterpret_cast<const uint32_t*>(g.idx + (uint64_t)(lp >> 1) * g.istride);
    const uint32_t q0 = ip[0], q1 = ip[1], q2 = ip[2], q3 = ip[3];
    ok = (q0 < g.nverts) & (q1 < g.nverts) & (q2 < g.nverts) & (q3 < g.nverts);
    if (!ok) return false;
    const uint32_t other = (lp & 1u) ? q0 : q2;   // the vertex this half does not use still has to be finite
    const float* po = reinterpret_cast<const float*>(g.verts + (uint64_t)other * g.vstride);
#pragma unroll
    for (int k = 0; k < 3; ++k) ok &= (po[k] > -kFltLarge) & (po[k] < kFltLarge);
    i0 = (lp & 1u) ? q2 : q0; i1 = q1; i2 = q3;
  } else {
    const uint32_t* ip = reinterpret_cast<const uint32_t*>(g.idx + (uint64_t)lp * g.istride);
    i0 = ip[0]; i1 = ip[1]; i2 = ip[2];
    ok = (i0 < g.nverts) & (i1 < g.nverts) & (i2 < g.nverts);          // scene_triangle_mesh.h:197-199
    if (!ok) return false;
  }
  const float* p0 = reinterpret_cast<const float*>(g.verts + (uint64_t)i0 * g.vstride);
  const float* p1 = reinterpret_cast<const float*>(g.verts + (uint64_t)i1 * g.vstride);
  const float* p2 = reinterpret_cast<const float*>(g.verts + (uint64_t)i2 * g.vstride);
  v[0] = p0[0]; v[1] = p0[1]; v[2] = p0[2];
  v[3] = p1[0]; v[4] = p1[1]; v[5] = p1[2];
  v[6] = p2[0]; v[7] = p2[1]; v[8] = p2[2];
#pragma unroll
  for (int k = 0; k < 9; ++k) ok &= (v[k] > -kFltLarge) & (v[k] < kFltLarge);  // isvalid(), vec3fa.h:304 (NaN fails)
  return ok;
}

// Box of the vertices.  An instanced triangle maps its three vertices to world space (tighter than mapping its box's corners), which
// must be finite as well, and widens their box by the pad.
__device__ __forceinline__ bool triangle_box(const GeomDesc& g, uint32_t lp, float lo[3], float hi[3]) {
  float v[9], pad[3] = {0.0f, 0.0f, 0.0f};
  bool ok = load_tri_verts(g, lp, v);
  if (!ok) return false;
  if (g.has_xfm) {
#pragma unroll
    for (int k = 0; k < 9; k += 3) xfm_point(g.xfm, v[k], v[k + 1], v[k + 2], v + k, pad);
#pragma unroll
    for (int k = 0; k < 9; ++k) ok &= (v[k] > -kFltLarge) & (v[k] < kFltLarge);
  }
  if (!ok) return false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = fminf(fminf(v[a], v[3 + a]), v[6 + a]);
    hi[a] = fmaxf(fmaxf(v[a], v[3 + a]), v[6 + a]);
  }
  if (g.has_xfm) {   // the triangle test runs in object space: widen the world box by the transform's error bound
#pragma unroll
    for (int a = 0; a < 3; ++a) { lo[a] -= pad[a]; hi[a] += pad[a]; }
  }
  return true;
}

// Record: a = (v0, primID), b = (e1 = v0 - v1, descriptor), c = (e2 = v2 - v0, mask) (triangle.h:98-120); ROBUST (Triangle4v,
// trianglev.h): b = (v1, ..), c = (v2, ..) for the Pluecker test.  OBJECT-space vertices for an instance (record_tests.cuh
// to_object_space).  A quad half's primID is the quad's, bit 31 set on the second half.  descriptor: GeomDesc index in general scenes,
// else the geomID.  `tb` (refit): the new box, empty for a triangle that became invalid, whose record then holds NaNs no ray can hit.
// Only triangles get one: the shim refits only scenes without curves, points or instances, so object space is world space.
__device__ __forceinline__ void pack_triangle(const GeomDesc& gd, uint32_t g, uint32_t lp, int robust, int general, float* tb, float4* dst) {
  float v[9];
  const bool ok = load_tri_verts(gd, lp, v);
  if (tb) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      tb[a] = ok ? fminf(fminf(v[a], v[3 + a]), v[6 + a]) : INFINITY;
      tb[3 + a] = ok ? fmaxf(fmaxf(v[a], v[3 + a]), v[6 + a]) : -INFINITY;
    }
    if (!ok) {
#pragma unroll
      for (int k = 0; k < 9; ++k) v[k] = NAN;
    }
  }
  float4 a, b, c;
  a.x = v[0]; a.y = v[1]; a.z = v[2]; a.w = __uint_as_float(gd.is_quad ? ((lp >> 1) | ((lp & 1u) << 31)) : lp);
  if (robust) {
    b.x = v[3]; b.y = v[4]; b.z = v[5];
    c.x = v[6]; c.y = v[7]; c.z = v[8];
  } else {
    b.x = __fsub_rn(v[0], v[3]); b.y = __fsub_rn(v[1], v[4]); b.z = __fsub_rn(v[2], v[5]);
    c.x = __fsub_rn(v[6], v[0]); c.y = __fsub_rn(v[7], v[1]); c.z = __fsub_rn(v[8], v[2]);
  }
  b.w = __uint_as_float(general ? g : gd.geomID);
  c.w = __uint_as_float(gd.mask);
  dst[0] = a; dst[1] = b; dst[2] = c;
}

// ---- linear curves (PRIM_ROUND_LINEAR, PRIM_FLAT_LINEAR)
// segment lp (kernels/common/scene_line_segments.h:427-441 valid(), linei.h bounds()): valid when both vertices exist, all four
// components are finite and no radius is negative
__device__ __forceinline__ bool load_curve(const GeomDesc& g, uint32_t lp, float4& p0, float4& p1, uint32_t& vid) {
  vid = *reinterpret_cast<const uint32_t*>(g.idx + (uint64_t)lp * g.istride);
  bool ok = (uint64_t)vid + 1 < g.nverts;
  if (!ok) return false;
  const float* a = reinterpret_cast<const float*>(g.verts + (uint64_t)vid * g.vstride);
  const float* b = reinterpret_cast<const float*>(g.verts + (uint64_t)(vid + 1) * g.vstride);
  p0 = make_float4(a[0], a[1], a[2], a[3]);
  p1 = make_float4(b[0], b[1], b[2], b[3]);
  const float c[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#pragma unroll
  for (int k = 0; k < 8; ++k) ok &= (c[k] > -kFltLarge) & (c[k] < kFltLarge);
  ok &= fminf(p0.w, p1.w) >= 0.0f;
  return ok;
}

// merge(p0, p1) enlarged by the larger radius; two extra ulp of the magnitudes keep it conservative
__device__ __forceinline__ bool linear_box(const GeomDesc& g, uint32_t lp, float lo[3], float hi[3]) {
  float4 c0, c1;
  uint32_t vid;
  if (!load_curve(g, lp, c0, c1, vid)) return false;
  const float r = fmaxf(c0.w, c1.w);
  const float a0[3] = {c0.x, c0.y, c0.z}, a1[3] = {c1.x, c1.y, c1.z};
#pragma unroll
  for (int a = 0; a < 3; ++a) { lo[a] = __fsub_rd(fminf(a0[a], a1[a]), r); hi[a] = __fadd_ru(fmaxf(a0[a], a1[a]), r); }
  widen_rel(lo, hi, 2.4e-7f);
  return true;
}

// Record: a = (p0.xyz, primID), b = (p1.xyz, descriptor), c = (r0, r1, first vertex | neighbour flags << 30, mask).  The round
// curve's test reads the neighbour vertices from the geometry's resident vertex buffer.
__device__ __forceinline__ void pack_linear(const GeomDesc& gd, uint32_t g, uint32_t lp, float4* dst) {
  float4 c0, c1;
  uint32_t vid;
  load_curve(gd, lp, c0, c1, vid);
  const uint32_t fl = gd.flags[lp] & 3u;
  dst[0] = make_float4(c0.x, c0.y, c0.z, __uint_as_float(lp));
  dst[1] = make_float4(c1.x, c1.y, c1.z, __uint_as_float(g));
  dst[2] = make_float4(c0.w, c1.w, __uint_as_float(vid | (fl << 30)), __uint_as_float(gd.mask));
}

// ---- cubic curves (PRIM_FLAT_CUBIC, PRIM_ROUND_CUBIC): prims_per_curve(g) BVH primitives per curve, local index = curve *
// prims_per_curve(g) + segment
// curve `curve` (scene_curves.h:498-533 valid()): all four control points (Hermite: both vertices and tangents) exist and are finite,
// radii included
__device__ __forceinline__ bool load_cubic(const GeomDesc& g, uint32_t curve, CurveVtx cp[4]) {
  const uint32_t vid = *reinterpret_cast<const uint32_t*>(g.idx + (uint64_t)curve * g.istride);
  bool ok = (uint64_t)vid + (g.hermite ? 1 : 3) < g.nverts;
  if (!ok) return false;
  if (g.hermite) {   // validity is checked on the vertices and tangents themselves (scene_curves.h:661-676)
    for (int k = 0; k < 2; ++k) {
      const float* a = reinterpret_cast<const float*>(g.verts + (uint64_t)(vid + k) * g.vstride);
      const float* t = reinterpret_cast<const float*>(g.tangents + (uint64_t)(vid + k) * g.tstride);
      for (int c = 0; c < 4; ++c) ok &= (a[c] > -kFltLarge) & (a[c] < kFltLarge) & (t[c] > -kFltLarge) & (t[c] < kFltLarge);
    }
  }
  load_cubic_cp(g, vid, cp);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    ok &= (cp[k].x > -kFltLarge) & (cp[k].x < kFltLarge) & (cp[k].y > -kFltLarge) & (cp[k].y < kFltLarge) & (cp[k].z > -kFltLarge) &
          (cp[k].z < kFltLarge) & (cp[k].r > -kFltLarge) & (cp[k].r < kFltLarge);
  return ok;
}

// Flat: one primitive per tessellation SEGMENT.  Box of the segment's two tessellation points (the last segment of a Bezier curve also
// holds the last control point, as accurateFlatBounds does, bezier_curve.h:631-664, bspline_curve.h:244-275), enlarged by the largest
// |radius| of the WHOLE curve and by 4 ulp of the largest magnitude (enlarge_bounds, scene_curves.cpp:433-437) -- so the union over a
// curve's segments is the box the reference reports for the curve.  The ribbon's quads are p +- r n with |n| = 1 evaluated in ray
// space, so the spheres around the two points hold the segment's quad; directed rounding + 2 ulp cover the world / ray-space
// difference.
__device__ __forceinline__ bool flat_cubic_box(const GeomDesc& g, uint32_t lp, float lo[3], float hi[3]) {
  CurveVtx cp[4];
  const int n = (int)g.tess, st = n + 1;
  const int seg = (int)(lp % (uint32_t)n);
  if (!load_cubic(g, lp / (uint32_t)n, cp)) return false;
  const float* tab = g.basis_tab;
  const bool bez = g.basis == BASIS_BEZIER;
  float rmax = bez ? fabsf(cp[3].r) : 0.0f;
  for (int j = 0; j <= n; ++j) rmax = fmaxf(rmax, fabsf(curve_blend(tab + j, st, cp[0].r, cp[1].r, cp[2].r, cp[3].r)));
  float plo[3] = {INFINITY, INFINITY, INFINITY}, phi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int j = seg; j <= seg + 1; ++j) {
    const float q[3] = {curve_blend(tab + j, st, cp[0].x, cp[1].x, cp[2].x, cp[3].x), curve_blend(tab + j, st, cp[0].y, cp[1].y, cp[2].y, cp[3].y),
                        curve_blend(tab + j, st, cp[0].z, cp[1].z, cp[2].z, cp[3].z)};
#pragma unroll
    for (int a = 0; a < 3; ++a) { plo[a] = fminf(plo[a], q[a]); phi[a] = fmaxf(phi[a], q[a]); }
  }
  if (bez && seg == n - 1) {
    const float q[3] = {cp[3].x, cp[3].y, cp[3].z};
#pragma unroll
    for (int a = 0; a < 3; ++a) { plo[a] = fminf(plo[a], q[a]); phi[a] = fmaxf(phi[a], q[a]); }
  }
  float size = 0.0f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = __fsub_rd(plo[a], rmax); hi[a] = __fadd_ru(phi[a], rmax);
    size = fmaxf(size, fmaxf(fabsf(lo[a]), fabsf(hi[a])));
  }
  const float e = 4.0f * 1.1920929e-07f * size;
#pragma unroll
  for (int a = 0; a < 3; ++a) { lo[a] = __fsub_rd(lo[a], e); hi[a] = __fadd_ru(hi[a], e); }
  widen_rel(lo, hi, 2.4e-7f);
  return finite_box(lo, hi);
}

// Round: one primitive per FIRST-LEVEL sub-segment of the sweep intersector, the curve between u = i/7 and (i+1)/7.  Box = hull of the
// sub-segment's Bezier control points p_i, p_i + dp_i/21, p_{i+1} - dp_{i+1}/21, p_{i+1} enlarged by the largest |radius| among them:
// the swept spheres of the sub-segment lie inside (convex hull property, radius included), and so do the bounding cylinders' hit
// points the iteration starts from only as start values.  The API box (alo, ahi) is the whole curve's accurateRoundBounds
// (bezier_curve.h:606-628: 8 points at u = i/7, each with p -+ dp/18) + enlarge_bounds, as the reference reports it.
__device__ __forceinline__ bool round_cubic_box(const GeomDesc& g, uint32_t lp, float lo[3], float hi[3], float alo[3], float ahi[3]) {
  CurveVtx cp[4];
  const int seg = (int)(lp % (uint32_t)kRoundSubSegs);
  if (!load_cubic(g, lp / (uint32_t)kRoundSubSegs, cp)) return false;
  float pl[4] = {INFINITY, INFINITY, INFINITY, INFINITY}, pu[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};     // whole curve (API bounds)
  float sl[4] = {INFINITY, INFINITY, INFINITY, INFINITY}, su[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};     // this sub-segment
  const float c4[4][4] = {{cp[0].x, cp[1].x, cp[2].x, cp[3].x}, {cp[0].y, cp[1].y, cp[2].y, cp[3].y}, {cp[0].z, cp[1].z, cp[2].z, cp[3].z}, {cp[0].r, cp[1].r, cp[2].r, cp[3].r}};
  const float scale = 1.0f / (3.0f * 6.0f), sub = 1.0f / (3.0f * kRoundSubSegs);
  for (int i = 0; i <= kRoundSubSegs; ++i) {
    float cc[4], dd[4];
    curve_basis_table_entry(g.basis, (float)i / kRoundSubSegs, cc, dd);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float pp = curve_blend(cc, 1, c4[c][0], c4[c][1], c4[c][2], c4[c][3]), dp = curve_blend(dd, 1, c4[c][0], c4[c][1], c4[c][2], c4[c][3]);
      const float pm = __fsub_rn(pp, __fmul_rn(scale, i != 0 ? dp : 0.0f)), pq = __fadd_rn(pp, __fmul_rn(scale, i != kRoundSubSegs ? dp : 0.0f));
      pl[c] = fminf(pl[c], fminf(pp, fminf(pm, pq))); pu[c] = fmaxf(pu[c], fmaxf(pp, fmaxf(pm, pq)));
      if (i == seg) { const float q = __fmaf_rn(sub, dp, pp); sl[c] = fminf(sl[c], fminf(pp, q)); su[c] = fmaxf(su[c], fmaxf(pp, q)); }
      if (i == seg + 1) { const float q = __fmaf_rn(-sub, dp, pp); sl[c] = fminf(sl[c], fminf(pp, q)); su[c] = fmaxf(su[c], fmaxf(pp, q)); }
    }
  }
  // the sub-segment's points come from the start-up-table formulas here and from de Casteljau / live basis evaluation in the
  // test: a relative 1e-6 of the coordinates covers the difference
  const float rseg = fmaxf(fabsf(sl[3]), fabsf(su[3])) * 1.000002f, rall = fmaxf(fabsf(pl[3]), fabsf(pu[3]));
  float size = 0.0f;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = __fsub_rd(sl[a], rseg); hi[a] = __fadd_ru(su[a], rseg);
    alo[a] = __fsub_rd(pl[a], rall); ahi[a] = __fadd_ru(pu[a], rall);
    size = fmaxf(size, fmaxf(fabsf(alo[a]), fabsf(ahi[a])));
  }
  widen_rel(lo, hi, 1.2e-6f);
  const float e = 4.0f * 1.1920929e-07f * size;
#pragma unroll
  for (int a = 0; a < 3; ++a) { alo[a] = __fsub_rd(alo[a], e); ahi[a] = __fadd_ru(ahi[a], e); }
  return finite_box(lo, hi);
}

// Record: a = (-, -, -, curve = primID), b = (-, -, -, descriptor), c = (segment, -, first control vertex, mask).  The test reads the
// control points from the resident vertex buffer; the segment is the ribbon's tessellation segment (flat) or the sweep's first-level
// sub-segment (round).
__device__ __forceinline__ void pack_cubic(const GeomDesc& gd, uint32_t g, uint32_t lp, float4* dst) {
  const uint32_t per = prims_per_curve(gd), curve = lp / per, seg = lp % per;
  const uint32_t vid = *reinterpret_cast<const uint32_t*>(gd.idx + (uint64_t)curve * gd.istride);
  dst[0] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(curve));
  dst[1] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(g));
  dst[2] = make_float4(__uint_as_float(seg), 0.0f, __uint_as_float(vid), __uint_as_float(gd.mask));
}

// ---- points (PRIM_SPHERE, PRIM_DISC, PRIM_ORIENTED_DISC; Points::valid + bounds, scene_points.h:146-199): centre -+ radius
__device__ __forceinline__ bool point_box(const GeomDesc& g, uint32_t lp, float lo[3], float hi[3]) {
  const float* q = reinterpret_cast<const float*>(g.verts + (uint64_t)lp * g.vstride);
  const float c[4] = {q[0], q[1], q[2], q[3]};
  bool ok = lp < g.nverts;
#pragma unroll
  for (int k = 0; k < 4; ++k) ok &= (c[k] > -kFltLarge) & (c[k] < kFltLarge);
  ok &= c[3] >= 0.0f;
  if (!ok) return false;
  const float rp = __fmul_ru(c[3], 1.000001f);   // the test's own rounding can accept a point a few ulp of the radius outside the exact sphere
#pragma unroll
  for (int a = 0; a < 3; ++a) { lo[a] = __fsub_rd(c[a], rp); hi[a] = __fadd_ru(c[a], rp); }
  widen_rel(lo, hi, 2.4e-7f);
  return true;
}

// Record: a = (centre, primID), b = (normal of an oriented disc, else 0; descriptor), c = (radius, -, -, mask); the test needs
// nothing else.
__device__ __forceinline__ void pack_point(const GeomDesc& gd, uint32_t g, uint32_t lp, float4* dst) {
  const float* q = reinterpret_cast<const float*>(gd.verts + (uint64_t)lp * gd.vstride);
  float nx = 0.0f, ny = 0.0f, nz = 0.0f;
  if (gd.kind == PRIM_ORIENTED_DISC) {
    const float* n = reinterpret_cast<const float*>(gd.tangents + (uint64_t)lp * gd.tstride);
    nx = n[0]; ny = n[1]; nz = n[2];
  }
  dst[0] = make_float4(q[0], q[1], q[2], __uint_as_float(lp));
  dst[1] = make_float4(nx, ny, nz, __uint_as_float(g));
  dst[2] = make_float4(q[3], 0.0f, 0.0f, __uint_as_float(gd.mask));
}

// ---- instances of instance traversal (PRIM_INSTANCE): g.verts is the InstRec table, one primitive per instance.  Valid when the
// instanced scene is not empty and local2world is finite; the box is the instanced scene's BVH bounds through local2world.
__device__ __forceinline__ bool instance_box(const GeomDesc& g, uint32_t lp, float lo[3], float hi[3]) {
  const InstRec& ir = reinterpret_cast<const InstRec*>(g.verts)[lp];
  bool ok = ir.lo[0] <= ir.hi[0];
#pragma unroll
  for (int k = 0; k < 12; ++k) ok &= (ir.xfm[k] > -kFltLarge) & (ir.xfm[k] < kFltLarge);
  if (!ok) return false;
#pragma unroll
  for (int a = 0; a < 3; ++a) { lo[a] = ir.lo[a]; hi[a] = ir.hi[a]; }
  return xfm_box(ir.xfm, lo, hi);
}

// Record: a = (0, 0, 0, instance index), b = (0, 0, 0, kInstRecord), c = (0, 0, 0, instance mask): the trace kernel's instance step
// finds everything else in the InstRec.
__device__ __forceinline__ void pack_instance(const GeomDesc& gd, uint32_t lp, float4* dst) {
  const InstRec& ir = reinterpret_cast<const InstRec*>(gd.verts)[lp];
  dst[0] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(lp));
  dst[1] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(kInstRecord));
  dst[2] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(ir.mask));
}

// Validity and world-space box of local primitive lp of g; a round cubic also returns the box the API reports for it (own_api).
__device__ __forceinline__ bool prim_box(const GeomDesc& g, uint32_t lp, float lo[3], float hi[3], float alo[3], float ahi[3], bool& own_api) {
  if (g.kind == PRIM_TRIANGLE) return triangle_box(g, lp, lo, hi);   // maps its vertices to world space itself
  if (g.kind == PRIM_INSTANCE) return instance_box(g, lp, lo, hi);
  bool ok;
  if (g.kind == PRIM_ROUND_CUBIC) {
    own_api = true;
    ok = round_cubic_box(g, lp, lo, hi, alo, ahi);
  } else if (g.kind == PRIM_FLAT_CUBIC) ok = flat_cubic_box(g, lp, lo, hi);
  else if (g.kind >= PRIM_SPHERE) ok = point_box(g, lp, lo, hi);
  else ok = linear_box(g, lp, lo, hi);
  if (ok && g.has_xfm) ok = xfm_box(g.xfm, lo, hi);
  return ok;
}

// ---------------------------------------------------------------------------------------------------
// 1. PrimRef generation + scene / centroid bounds
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) primref_gen(const GeomDesc* __restrict__ geoms, const uint32_t* __restrict__ offs,
                                                   int ngeoms, uint32_t ntot, PrimRef* __restrict__ out,
                                                   BuildInfo* __restrict__ info) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  float alo[3] = {INFINITY, INFINITY, INFINITY}, ahi[3] = {-INFINITY, -INFINITY, -INFINITY};   // API-visible box when it is not the primitive's own (own_api)
  bool ok = false, skipb = false, own_api = false;
  if (p < ntot) {
    const int g = find_geom(offs, ngeoms, p);
    ok = prim_box(geoms[g], p - offs[g], lo, hi, alo, ahi, own_api);
    skipb = geoms[g].skip_bounds != 0;
    PrimRef pr;
    pr.lox = lo[0]; pr.loy = lo[1]; pr.loz = lo[2]; pr.prim = p;
    pr.hix = hi[0]; pr.hiy = hi[1]; pr.hiz = hi[2]; pr.valid = ok ? 1u : 0u;
    out[p] = pr;
  }
  // an invalid primitive has no box: the curve kinds compute one and only then reject it when it crosses +-kFltLarge, and that box
  // must not reach the scene bounds (the SAH root's box) or the API bounds
  if (!ok) {
#pragma unroll
    for (int a = 0; a < 3; ++a) { lo[a] = INFINITY; hi[a] = -INFINITY; }
  }
  // warp reduce, then one set of atomics per warp
  float c_lo[3], c_hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) { c_lo[a] = ok ? lo[a] + hi[a] : INFINITY; c_hi[a] = ok ? lo[a] + hi[a] : -INFINITY; }
  float a_lo[3], a_hi[3];   // API-visible bounds: instanced triangles are represented by their instance box (host side)
#pragma unroll
  for (int a = 0; a < 3; ++a) { a_lo[a] = (skipb || !ok) ? INFINITY : (own_api ? alo[a] : lo[a]); a_hi[a] = (skipb || !ok) ? -INFINITY : (own_api ? ahi[a] : hi[a]); }
  unsigned cnt = ok ? 1u : 0u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xFFFFFFFFu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xFFFFFFFFu, hi[a], o));
      c_lo[a] = fminf(c_lo[a], __shfl_xor_sync(0xFFFFFFFFu, c_lo[a], o));
      c_hi[a] = fmaxf(c_hi[a], __shfl_xor_sync(0xFFFFFFFFu, c_hi[a], o));
      a_lo[a] = fminf(a_lo[a], __shfl_xor_sync(0xFFFFFFFFu, a_lo[a], o));
      a_hi[a] = fmaxf(a_hi[a], __shfl_xor_sync(0xFFFFFFFFu, a_hi[a], o));
    }
    cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      atomicMin(&info->geom_lo[a], f2ord(lo[a]));
      atomicMax(&info->geom_hi[a], f2ord(hi[a]));
      atomicMin(&info->cent_lo[a], f2ord(c_lo[a]));
      atomicMax(&info->cent_hi[a], f2ord(c_hi[a]));
      atomicMin(&info->api_lo[a], f2ord(a_lo[a]));
      atomicMax(&info->api_hi[a], f2ord(a_hi[a]));
    }
    atomicAdd(&info->num_valid, cnt);
  }
}

__global__ void init_info(BuildInfo* info) {
  for (int a = 0; a < 3; ++a) {
    info->geom_lo[a] = info->cent_lo[a] = f2ord(INFINITY);
    info->geom_hi[a] = info->cent_hi[a] = f2ord(-INFINITY);
    info->api_lo[a] = f2ord(INFINITY); info->api_hi[a] = f2ord(-INFINITY);
  }
  info->num_valid = 0; info->node_tail = 1; info->tri_tail = 0; info->pad = 0; info->sah = 0.0; info->depth = 0;
}

// ---------------------------------------------------------------------------------------------------
// 2. Morton keys: 21 bits per axis of the box centre, invalid primitives get the maximum key
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t expand21(uint32_t v) {
  uint64_t x = v & 0x1FFFFFull;
  x = (x | x << 32) & 0x1F00000000FFFFull;
  x = (x | x << 16) & 0x1F0000FF0000FFull;
  x = (x | x << 8) & 0x100F00F00F00F00Full;
  x = (x | x << 4) & 0x10C30C30C30C30C3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}

__global__ void __launch_bounds__(256) morton_keys(const PrimRef* __restrict__ prims, uint32_t ntot,
                                                   const BuildInfo* __restrict__ info, uint64_t* __restrict__ keys,
                                                   uint32_t* __restrict__ vals) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= ntot) return;
  const PrimRef pr = prims[p];
  uint64_t key = ~0ull;
  if (pr.valid) {
    const float c[3] = {pr.lox + pr.hix, pr.loy + pr.hiy, pr.loz + pr.hiz};
    uint32_t q[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float lo = ord2f(info->cent_lo[a]), hi = ord2f(info->cent_hi[a]);
      const float ext = hi - lo;
      float f = ext > 0.0f ? (c[a] - lo) / ext : 0.0f;
      f = fminf(fmaxf(f * 2097152.0f, 0.0f), 2097151.0f);
      q[a] = (uint32_t)f;
    }
    key = (expand21(q[2]) << 2) | (expand21(q[1]) << 1) | expand21(q[0]);  // < 2^63, so never collides with ~0
  }
  keys[p] = key;
  vals[p] = p;
}

// ---------------------------------------------------------------------------------------------------
// 3. LSD radix sort of (u64 key, u32 value), 8-bit digits.  Per pass: tile histograms -> scan -> stable scatter
//    with warp-level multi-split ranking (__match_any_sync).
// ---------------------------------------------------------------------------------------------------
constexpr int RS_THREADS = 256;
constexpr int RS_ITEMS = 16;
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;  // 4096 keys per block

__global__ void __launch_bounds__(RS_THREADS) radix_hist(const uint64_t* __restrict__ keys, uint32_t n, int shift,
                                                         uint32_t* __restrict__ block_hist, uint32_t nblocks) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t base = blockIdx.x * RS_TILE;
#pragma unroll
  for (int i = 0; i < RS_ITEMS; ++i) {
    const uint32_t idx = base + i * RS_THREADS + threadIdx.x;
    if (idx < n) atomicAdd(&h[(uint32_t)(keys[idx] >> shift) & 0xFFu], 1u);
  }
  __syncthreads();
  block_hist[threadIdx.x * nblocks + blockIdx.x] = h[threadIdx.x];  // digit-major
}

// one block per digit: exclusive scan of that digit's row (over tiles); row total -> digit_total[d]
__global__ void __launch_bounds__(256) radix_scan_rows(uint32_t* __restrict__ block_hist, uint32_t nblocks,
                                                       uint32_t* __restrict__ digit_total) {
  __shared__ uint32_t wsum[8];
  __shared__ uint32_t carry;
  uint32_t* row = block_hist + (size_t)blockIdx.x * nblocks;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < nblocks; base += 256) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < nblocks ? row[i] : 0;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = x;
    __syncthreads();
    uint32_t woff = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) woff += wsum[w];
    const uint32_t incl = x + woff + carry;
    if (i < nblocks) row[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == 255) carry = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) digit_total[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(256) radix_scan_digits(const uint32_t* __restrict__ digit_total,
                                                         uint32_t* __restrict__ digit_base) {
  __shared__ uint32_t s[256];
  s[threadIdx.x] = digit_total[threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int d = 0; d < 256; ++d) { const uint32_t c = s[d]; s[d] = run; run += c; }
  }
  __syncthreads();
  digit_base[threadIdx.x] = s[threadIdx.x];
}

__global__ void __launch_bounds__(RS_THREADS) radix_scatter(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                                                            uint64_t* __restrict__ kout, uint32_t* __restrict__ vout,
                                                            uint32_t n, int shift, const uint32_t* __restrict__ row_prefix,
                                                            const uint32_t* __restrict__ digit_base, uint32_t nblocks) {
  __shared__ uint32_t wcnt[RS_THREADS / 32][256];
  __shared__ uint32_t gbase[256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < (RS_THREADS / 32) * 256; i += RS_THREADS) (&wcnt[0][0])[i] = 0;
  __syncthreads();
  // warp w owns the contiguous slice [w*32*ITEMS, (w+1)*32*ITEMS) of the tile: stable order = (warp, item, lane)
  const uint32_t wbase = blockIdx.x * RS_TILE + warp * (32 * RS_ITEMS);
  uint64_t k[RS_ITEMS];
#pragma unroll
  for (int i = 0; i < RS_ITEMS; ++i) {
    const uint32_t idx = wbase + i * 32 + lane;
    k[i] = idx < n ? kin[idx] : ~0ull;  // out-of-range slots sit at the very end of the last tile: harmless
  }
#pragma unroll
  for (int i = 0; i < RS_ITEMS; ++i) {
    const uint32_t d = (uint32_t)(k[i] >> shift) & 0xFFu;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
    if (lane == __ffs(peers) - 1) wcnt[warp][d] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  {
    const int d = threadIdx.x;  // RS_THREADS == 256 digits
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < RS_THREADS / 32; ++w) { const uint32_t c = wcnt[w][d]; wcnt[w][d] = run; run += c; }
    gbase[d] = digit_base[d] + row_prefix[(size_t)d * nblocks + blockIdx.x];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < RS_ITEMS; ++i) {
    const uint32_t idx = wbase + i * 32 + lane;
    const uint32_t d = (uint32_t)(k[i] >> shift) & 0xFFu;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
    const int leader = __ffs(peers) - 1;
    uint32_t old = 0;
    if (lane == leader) { old = wcnt[warp][d]; wcnt[warp][d] = old + __popc(peers); }
    old = __shfl_sync(0xFFFFFFFFu, old, leader);
    __syncwarp();
    if (idx < n) {
      const uint32_t pos = gbase[d] + old + __popc(peers & ((1u << lane) - 1u));
      kout[pos] = k[i];
      vout[pos] = vin[idx];
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// 4. LBVH hierarchy (parallel radix tree over the sorted keys, duplicates split by index) + bottom-up refit
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) lbvh_hierarchy(const uint64_t* __restrict__ keys, int n, Node2* __restrict__ nodes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n - 1) return;
  lbvh_node(keys, n, i, nodes);
}

__global__ void __launch_bounds__(256) lbvh_leaves_refit(const PrimRef* __restrict__ prims, const uint32_t* __restrict__ sorted,
                                                         int n, Node2* nodes, uint32_t* __restrict__ flags) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const PrimRef pr = prims[sorted[j]];
  Node2& lf = nodes[n - 1 + j];
  lf.lox = pr.lox; lf.loy = pr.loy; lf.loz = pr.loz; lf.left = j;
  lf.hix = pr.hix; lf.hiy = pr.hiy; lf.hiz = pr.hiz; lf.right = -1;
  lf.first = (uint32_t)j; lf.count = 1; lf.pad = 0;
  if (n == 1) { lf.parent = 0xFFFFFFFFu; return; }
  uint32_t cur = lf.parent;
  __threadfence();
  while (cur != 0xFFFFFFFFu) {
    if (atomicAdd(&flags[cur], 1u) == 0) return;  // first arrival: the sibling subtree is not finished yet
    __threadfence();
    Node2& nd = nodes[cur];
    const float4* L = reinterpret_cast<const float4*>(&nodes[nd.left]);
    const float4* R = reinterpret_cast<const float4*>(&nodes[nd.right]);
    const float4 l0 = __ldcg(L), l1 = __ldcg(L + 1), r0 = __ldcg(R), r1 = __ldcg(R + 1);
    nd.lox = fminf(l0.x, r0.x); nd.loy = fminf(l0.y, r0.y); nd.loz = fminf(l0.z, r0.z);
    nd.hix = fmaxf(l1.x, r1.x); nd.hiy = fmaxf(l1.y, r1.y); nd.hiz = fmaxf(l1.z, r1.z);
    __threadfence();
    cur = nd.parent;
  }
}

// ---------------------------------------------------------------------------------------------------
// 5. Collapse the binary tree into BVH8 nodes, one tree level per launch.  Queue slot q == BVH8 node id q.
// ---------------------------------------------------------------------------------------------------
struct DeviceAlloc {  // allocation callbacks of collapse_node() on the device: global atomic bump counters
  BuildInfo* info;
  __device__ __forceinline__ uint32_t nodes(uint32_t k) const { return atomicAdd(&info->node_tail, k); }
  __device__ __forceinline__ uint32_t tris(uint32_t k) const { return atomicAdd(&info->tri_tail, k); }
  __device__ __forceinline__ void sah(double x) const { atomicAdd(&info->sah, x); }
};

// All levels in ONE cooperative launch: the grid walks the queue level by level with a grid-wide barrier between
// levels (round 1 launched one kernel per level and read the queue tail back to the host each time: 2 + depth host
// round trips per commit).  The level boundaries are kept for refit_scene().
__global__ void __launch_bounds__(128) collapse_all(const Node2* __restrict__ n2, uint32_t* __restrict__ src, Node8* __restrict__ n8,
                                                    uint32_t* __restrict__ tri_src, const uint32_t* __restrict__ sortedA,
                                                    const uint32_t* __restrict__ sortedB, BuildInfo* info, float inv_root_area, int policy,
                                                    const uint32_t* __restrict__ dec) {
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
  uint32_t begin = 0, end = 1, depth = 0;
  while (begin < end && depth < (uint32_t)kStackSize) {
    for (uint32_t q = begin + tid; q < end; q += nthreads)
      collapse_node(n2, src, q, n8, tri_src, sortedA, sortedB, inv_root_area, policy, dec, DeviceAlloc{info});
    grid.sync();
    const uint32_t tail = *reinterpret_cast<volatile uint32_t*>(&info->node_tail);
    if (tid == 0) info->level_begin[depth] = begin;
    grid.sync();                      // everyone has read the tail before the next level bumps it
    begin = end; end = tail; ++depth;
  }
  if (tid == 0) { info->level_begin[depth] = begin; info->depth = (begin < end) ? 0xFFFFFFFFu : depth; }   // too deep -> error on the host
}

// bottom-up dynamic programme for the SAH-optimal collapse (rt_core.cuh dp_node): one thread per primitive climbs
// towards the root; the second arrival at a node (atomic flag) owns it, exactly like the refit.
__global__ void __launch_bounds__(256) collapse_dp(const Node2* __restrict__ nodes, int n, uint32_t* __restrict__ flags,
                                                   float* F /*[2n][8]*/, uint32_t* dec, float c_node, float c_tri) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t leaf = (uint32_t)(n - 1 + j);
  {
    float f[8];
    uint32_t d;
    dp_leaf(half_area(nodes[leaf]), c_tri, f, &d);
    float4* dst = reinterpret_cast<float4*>(F + (size_t)leaf * 8);
    dst[0] = make_float4(f[0], f[1], f[2], f[3]); dst[1] = make_float4(f[4], f[5], f[6], f[7]);
    dec[leaf] = d;
  }
  if (n == 1) return;
  uint32_t cur = nodes[leaf].parent;
  __threadfence();
  while (cur != 0xFFFFFFFFu) {
    if (atomicAdd(&flags[cur], 1u) == 0) return;
    __threadfence();
    const Node2 nd = nodes[cur];
    float fl[8], fr[8], f[8];
    const float4* L = reinterpret_cast<const float4*>(F + (size_t)nd.left * 8);
    const float4* R = reinterpret_cast<const float4*>(F + (size_t)nd.right * 8);
    const float4 l0 = __ldcg(L), l1 = __ldcg(L + 1), r0 = __ldcg(R), r1 = __ldcg(R + 1);
    fl[0] = l0.x; fl[1] = l0.y; fl[2] = l0.z; fl[3] = l0.w; fl[4] = l1.x; fl[5] = l1.y; fl[6] = l1.z; fl[7] = l1.w;
    fr[0] = r0.x; fr[1] = r0.y; fr[2] = r0.z; fr[3] = r0.w; fr[4] = r1.x; fr[5] = r1.y; fr[6] = r1.z; fr[7] = r1.w;
    uint32_t d;
    dp_node(half_area(nd), nd.count, fl, fr, c_node, c_tri, f, &d);
    float4* dst = reinterpret_cast<float4*>(F + (size_t)cur * 8);
    dst[0] = make_float4(f[0], f[1], f[2], f[3]); dst[1] = make_float4(f[4], f[5], f[6], f[7]);
    dec[cur] = d;
    __threadfence();
    cur = nd.parent;
  }
}

// ---------------------------------------------------------------------------------------------------
// 6. leaf_pack: the 48-byte record of every BVH primitive, laid out by its kind's packer above
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) leaf_pack(const GeomDesc* __restrict__ geoms, const uint32_t* __restrict__ offs, int ngeoms,
                                                 const uint32_t* __restrict__ tri_src, uint32_t ntris, TriRec* __restrict__ out, int robust,
                                                 int general, float* __restrict__ tribox = nullptr) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntris) return;
  const uint32_t p = tri_src[t];
  const int g = find_geom(offs, ngeoms, p);
  const GeomDesc gd = geoms[g];
  const uint32_t lp = p - offs[g];
  float4* dst = reinterpret_cast<float4*>(&out[t]);
  if (gd.kind == PRIM_INSTANCE) pack_instance(gd, lp, dst);
  else if (gd.kind == PRIM_FLAT_CUBIC || gd.kind == PRIM_ROUND_CUBIC) pack_cubic(gd, (uint32_t)g, lp, dst);
  else if (gd.kind >= PRIM_SPHERE) pack_point(gd, (uint32_t)g, lp, dst);
  else if (gd.kind != PRIM_TRIANGLE) pack_linear(gd, (uint32_t)g, lp, dst);
  else pack_triangle(gd, (uint32_t)g, lp, robust, general, tribox ? tribox + (size_t)t * 6 : nullptr, dst);
}

// binned-SAH top-down build of the binary tree (build_sah.cu)
int build_sah_tree(const PrimRef* prims, uint32_t* idsA, uint32_t* idsB, uint32_t n, Node2* nodes, const float* scene_bounds,
                   const float* cent_bounds, cudaStream_t stream, char* errmsg);

// ---------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------
// Build temporaries come from the device's stream-ordered memory pool (cudaMallocAsync): after the first commit the
// pool serves every later build without touching the driver allocator, which is what keeps per-frame rebuilds of
// dynamic scenes at kernel time (a plain cudaMalloc/cudaFree pair per buffer is slow at 10 M triangles).
// The pool is the device's default one, which other users of cudaMallocAsync in the process share: the amount it may keep
// cached after a commit is bounded (device config key "pool_keep_mb", default 8192 MB -- enough for the temporaries of a
// 10 M-triangle build; memory above that goes back to the driver at the next synchronisation).
static unsigned long long g_pool_keep_bytes = 8192ull << 20;
void set_pool_keep_bytes(unsigned long long bytes) { g_pool_keep_bytes = bytes; }
static void ensure_pool(int device) {
  static bool done[64] = {};
  if (device < 0 || device >= 64 || done[device]) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    unsigned long long keep = 0;
    cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    if (keep < g_pool_keep_bytes) { keep = g_pool_keep_bytes; cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep); }
  }
  cudaGetLastError();
  done[device] = true;
}

template <typename T>
struct DevBuf {
  T* p = nullptr;
  cudaStream_t st = nullptr;
  ~DevBuf() { if (p) cudaFreeAsync(p, st); }
  cudaError_t alloc(size_t n, cudaStream_t stream) {
    st = stream;
    return cudaMallocAsync(reinterpret_cast<void**>(&p), std::max<size_t>(n, 1) * sizeof(T), stream);
  }
};

struct EventTimer {   // stream time between start() and stop(); the events are released on every exit path
  cudaEvent_t a = nullptr, b = nullptr;
  ~EventTimer() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
  cudaError_t start(cudaStream_t st) {
    cudaError_t e = cudaEventCreate(&a);
    if (e == cudaSuccess) e = cudaEventCreate(&b);
    return e == cudaSuccess ? cudaEventRecord(a, st) : e;
  }
  cudaError_t stop(cudaStream_t st) { return cudaEventRecord(b, st); }
  float ms() const { float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms; }   // after a synchronisation past stop()
};

// first global primitive index of every geometry, offs[ngeoms] = the total, which is returned
static uint64_t prim_offsets(const GeomDesc* geoms, int ngeoms, std::vector<uint32_t>& offs) {
  offs.assign(ngeoms + 1, 0);
  uint64_t tot64 = 0;
  for (int g = 0; g < ngeoms; ++g) { offs[g] = (uint32_t)tot64; tot64 += geoms[g].ntris; }
  offs[ngeoms] = (uint32_t)tot64;
  return tot64;
}

// the stat counters of a traced scene: [3] rays, nodes, tris, allocated and zeroed once
static cudaError_t alloc_stat(SceneGPU& s, cudaStream_t st) {
  if (s.d_stat) return cudaSuccess;
  const cudaError_t e = cudaMalloc(&s.d_stat, 3 * sizeof(unsigned long long));
  return e == cudaSuccess ? cudaMemsetAsync(s.d_stat, 0, 3 * sizeof(unsigned long long), st) : e;
}

// the arrays of `s` are about to change (SceneGPU::content)
static void renew_content(SceneGPU& s) {
  static std::atomic<uint64_t> last{0};
  s.content = ++last;
}

// the BVH arrays, what refit_scene keeps and the layout of an assembly (pool memory: goes back to the pool for the next commit)
static void release_arrays(SceneGPU& s, cudaStream_t st) {
  renew_content(s);
  if (s.nodes) cudaFreeAsync(s.nodes, st);
  if (s.tris) cudaFreeAsync(s.tris, st);
  if (s.d_descs) cudaFreeAsync(s.d_descs, st);
  if (s.tri_src) cudaFreeAsync(s.tri_src, st);
  if (s.d_insts) cudaFreeAsync(s.d_insts, st);
  s.nodes = nullptr; s.tris = nullptr; s.d_descs = nullptr; s.tri_src = nullptr; s.d_insts = nullptr; s.levels.clear();
  s.num_insts = 0;
  s.num_nodes = s.num_tris = 0; s.root_valid = 0;
  s.subs.clear(); s.top_cap = s.top_tri_cap = 0;
}

void free_scene(SceneGPU& s, cudaStream_t st) {
  release_arrays(s, st);
  if (s.d_stat) cudaFree(s.d_stat);
  s.d_stat = nullptr;
}

int build_scene(SceneGPU& s, const GeomDesc* geoms, int ngeoms, BuilderKind kind, cudaStream_t st, char* errmsg) {
  errmsg[0] = 0;
  release_arrays(s, st);   // renews s.content
  s.max_depth = 0; s.sah_cost = 0; s.builder = kind;
  for (int a = 0; a < 3; ++a) { s.bounds[a] = s.api_bounds[a] = INFINITY; s.bounds[3 + a] = s.api_bounds[3 + a] = -INFINITY; }
  if (!s.is_sub) CK(alloc_stat(s, st));

  std::vector<uint32_t> offs;
  const uint64_t tot64 = prim_offsets(geoms, ngeoms, offs);
  if (tot64 >= 0x7FFFFFFFull) { snprintf(errmsg, 256, "too many triangles (%llu)", (unsigned long long)tot64); return -1; }
  const uint32_t ntot = (uint32_t)tot64;
  if (ntot == 0) return 0;  // empty scene: queries return immediately (bvh_intersector1.cpp:39)
  ensure_pool(s.device);

  EventTimer timer;
  CK(timer.start(st));

  DevBuf<GeomDesc> d_geoms; DevBuf<uint32_t> d_offs; DevBuf<BuildInfo> d_info; DevBuf<PrimRef> d_prims;
  DevBuf<uint64_t> d_k0, d_k1; DevBuf<uint32_t> d_v0, d_v1, d_hist, d_dtot, d_dbase;
  CK(d_geoms.alloc(ngeoms, st)); CK(d_offs.alloc(ngeoms + 1, st)); CK(d_info.alloc(1, st)); CK(d_prims.alloc(ntot, st));
  CK(d_k0.alloc(ntot, st)); CK(d_k1.alloc(ntot, st)); CK(d_v0.alloc(ntot, st)); CK(d_v1.alloc(ntot, st));
  const uint32_t nb = (ntot + RS_TILE - 1) / RS_TILE;
  CK(d_hist.alloc((size_t)256 * nb, st)); CK(d_dtot.alloc(256, st)); CK(d_dbase.alloc(256, st));
  CK(cudaMemcpyAsync(d_geoms.p, geoms, sizeof(GeomDesc) * ngeoms, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_offs.p, offs.data(), 4 * (ngeoms + 1), cudaMemcpyHostToDevice, st));

  const uint32_t g256 = (ntot + 255) / 256;
  init_info<<<1, 1, 0, st>>>(d_info.p);
  primref_gen<<<g256, 256, 0, st>>>(d_geoms.p, d_offs.p, ngeoms, ntot, d_prims.p, d_info.p);
  morton_keys<<<g256, 256, 0, st>>>(d_prims.p, ntot, d_info.p, d_k0.p, d_v0.p);
  count_launch(3);
  uint64_t *kin = d_k0.p, *kout = d_k1.p;
  uint32_t *vin = d_v0.p, *vout = d_v1.p;
  for (int pass = 0; pass < 8; ++pass) {
    const int shift = 8 * pass;
    radix_hist<<<nb, RS_THREADS, 0, st>>>(kin, ntot, shift, d_hist.p, nb);
    radix_scan_rows<<<256, 256, 0, st>>>(d_hist.p, nb, d_dtot.p);
    radix_scan_digits<<<1, 256, 0, st>>>(d_dtot.p, d_dbase.p);
    radix_scatter<<<nb, RS_THREADS, 0, st>>>(kin, vin, kout, vout, ntot, shift, d_hist.p, d_dbase.p, nb);
    count_launch(4);
    std::swap(kin, kout); std::swap(vin, vout);
  }
  CK(cudaGetLastError());
  BuildInfo hinfo;
  CK(cudaMemcpyAsync(&hinfo, d_info.p, sizeof(BuildInfo), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint32_t n = hinfo.num_valid;  // valid primitives are sorted[0..n); invalid ones carry key ~0 at the end
  if (n == 0) return 0;
  for (int a = 0; a < 3; ++a) {
    s.bounds[a] = ord2f_host(hinfo.geom_lo[a]); s.bounds[3 + a] = ord2f_host(hinfo.geom_hi[a]);
    s.api_bounds[a] = ord2f_host(hinfo.api_lo[a]); s.api_bounds[3 + a] = ord2f_host(hinfo.api_hi[a]);
  }

  // ---- binary tree
  DevBuf<Node2> d_n2; DevBuf<uint32_t> d_flags;
  CK(d_n2.alloc((size_t)2 * n, st)); CK(d_flags.alloc(n, st));
  uint32_t root2 = 0;
  if (kind == BUILDER_SAH && n > 1) {
    float cb[6];
    for (int a = 0; a < 3; ++a) { cb[a] = ord2f_host(hinfo.cent_lo[a]); cb[3 + a] = ord2f_host(hinfo.cent_hi[a]); }
    int r = build_sah_tree(d_prims.p, vin, vout, n, d_n2.p, s.bounds, cb, st, errmsg);
    if (r) return r;
    root2 = 0;
  } else {
    CK(cudaMemsetAsync(d_flags.p, 0, 4 * (size_t)n, st));
    const uint32_t gn = (n + 255) / 256;
    if (n > 1) { lbvh_hierarchy<<<gn, 256, 0, st>>>(kin, (int)n, d_n2.p); count_launch(); }
    lbvh_leaves_refit<<<gn, 256, 0, st>>>(d_prims.p, vin, (int)n, d_n2.p, d_flags.p);
    count_launch();
    root2 = (n == 1) ? 0u : 0u;  // n == 1: the only node is leaf id n-1+0 == 0
  }

  // ---- collapse into BVH8, level by level (children chosen by the SAH-optimal DP unless policy says greedy)
  DevBuf<uint32_t> d_src, d_trisrc, d_dec;
  DevBuf<float> d_F;
  const bool use_dp = tuning().collapse_policy >= 3 && n > 1;
  if (use_dp) {
    CK(d_F.alloc((size_t)2 * n * 8, st)); CK(d_dec.alloc((size_t)2 * n, st));
    CK(cudaMemsetAsync(d_flags.p, 0, 4 * (size_t)n, st));
    collapse_dp<<<(n + 255) / 256, 256, 0, st>>>(d_n2.p, (int)n, d_flags.p, d_F.p, d_dec.p, tuning().c_node * 0.01f, tuning().c_tri * 0.01f);
    count_launch();
  }
  s.node_capacity = (size_t)n + 1; s.tri_capacity = n;
  CK(d_src.alloc(s.node_capacity, st)); CK(d_trisrc.alloc(n, st));
  DevBuf<Node8> d_n8;      // worst-case sized scratch; the final array is an exact-size copy
  CK(d_n8.alloc(s.node_capacity, st));
  Node8* n8 = d_n8.p;
  CK(cudaMemcpyAsync(d_src.p, &root2, 4, cudaMemcpyHostToDevice, st));
  const float ex = s.bounds[3] - s.bounds[0], ey = s.bounds[4] - s.bounds[1], ez = s.bounds[5] - s.bounds[2];
  const float ra = ex * (ey + ez) + ey * ez;
  const float inv_ra = ra > 0.0f ? 1.0f / ra : 0.0f;
  {
    static int coop_blocks = 0;       // co-resident blocks of collapse_all on this device (one grid-wide barrier per level)
    if (!coop_blocks) {
      int per_sm = 0, sms = 0;
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, collapse_all, 128, 0));
      CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s.device));
      coop_blocks = std::max(1, per_sm * sms);
    }
    const Node2* a_n2 = d_n2.p; uint32_t* a_src = d_src.p; uint32_t* a_trisrc = d_trisrc.p; const uint32_t *a_vin = vin, *a_vout = vout;
    BuildInfo* a_info = d_info.p; float a_inv = inv_ra; int a_pol = tuning().collapse_policy; const uint32_t* a_dec = use_dp ? d_dec.p : nullptr;
    void* kargs[] = {&a_n2, &a_src, &n8, &a_trisrc, &a_vin, &a_vout, &a_info, &a_inv, &a_pol, &a_dec};
    const int blocks = (int)std::min<size_t>((size_t)coop_blocks, std::max<size_t>(1, ((size_t)n + 127) / 128));
    CK(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(collapse_all), dim3(blocks), dim3(128), kargs, 0, st));
    count_launch();
  }
  CK(cudaMemcpyAsync(&hinfo, d_info.p, sizeof(BuildInfo), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const uint32_t depth = hinfo.depth, end = hinfo.node_tail;
  if (depth == 0xFFFFFFFFu || depth >= (uint32_t)kStackSize) { snprintf(errmsg, 256, "BVH too deep for the traversal stack (%u levels)", (unsigned)kStackSize); return -1; }
  if (hinfo.tri_tail != n) { snprintf(errmsg, 256, "internal: packed %u of %u triangles", hinfo.tri_tail, n); return -1; }

  // ---- triangle records, then shrink the node array to its final size
  DevBuf<TriRec> d_tris;
  DevBuf<Node8> d_final;
  CK(d_tris.alloc(n, st));
  leaf_pack<<<(n + 255) / 256, 256, 0, st>>>(d_geoms.p, d_offs.p, ngeoms, d_trisrc.p, n, d_tris.p, s.robust, s.general);
  count_launch();
  CK(d_final.alloc(end, st));
  CK(cudaMemcpyAsync(d_final.p, n8, (size_t)end * sizeof(Node8), cudaMemcpyDeviceToDevice, st));
  CK(timer.stop(st));
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  s.nodes = d_final.p; s.tris = d_tris.p; d_final.p = nullptr; d_tris.p = nullptr;   // ownership moves to the scene
  if (s.general) { s.d_descs = d_geoms.p; d_geoms.p = nullptr; s.num_descs = (uint32_t)ngeoms; }
  s.num_nodes = end; s.num_tris = n; s.root_valid = 1;
  s.build_ms = timer.ms(); s.sah_cost = hinfo.sah; s.max_depth = depth;
  // kept for refit_scene(): which primitive every triangle record came from, and the level ranges of the node array
  s.tri_src = d_trisrc.p; d_trisrc.p = nullptr;
  s.total_prims = ntot;
  s.levels.assign(hinfo.level_begin, hinfo.level_begin + depth + 1);
  s.levels.back() = end;
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// REFIT (RTC_BUILD_QUALITY_REFIT, kernels/bvh/bvh_refit.cpp): the vertices moved, the topology did not.  Triangle
// records are re-packed from the new vertex data, then the BVH8 levels are revisited bottom-up: every node takes the
// new boxes of its children (triangle bounds for leaf slots, the child's node box for internal slots), re-derives its
// own box and re-quantises -- same slots, same child / triangle ranges, no sort, no hierarchy construction.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) refit_level(Node8* __restrict__ n8, uint32_t begin, uint32_t end, const float* __restrict__ tribox,
                                                   float* __restrict__ nodebox) {
  const uint32_t q = begin + blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= end) return;
  Node8 nd = n8[q];
  const uint32_t imask = nd.w[3] >> 24, child_base = nd.w[4], tri_base = nd.w[5];
  ChildBox cb[8];
  uint8_t slot_of[8];
  bool empty[8];
  int n = 0;
  float plo[3] = {INFINITY, INFINITY, INFINITY}, phi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int sl = 0; sl < 8; ++sl) {
    const uint32_t lm = node_leafmask_raw(nd.w, sl) & 0x00FFFFFFu;
    const bool inner = (imask >> sl) & 1u;
    if (!inner && lm == 0) continue;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    if (inner) {
      const float* b = nodebox + (size_t)(child_base + __popc(imask & ((1u << sl) - 1u))) * 6;
      for (int a = 0; a < 3; ++a) { lo[a] = b[a]; hi[a] = b[3 + a]; }
    } else {
      for (uint32_t m = lm; m; m &= m - 1) {
        const float* b = tribox + (size_t)(tri_base + (uint32_t)(__ffs((int)m) - 1)) * 6;
        for (int a = 0; a < 3; ++a) { lo[a] = fminf(lo[a], b[a]); hi[a] = fmaxf(hi[a], b[3 + a]); }
      }
    }
    empty[n] = !(lo[0] <= hi[0]);
    for (int a = 0; a < 3; ++a) { cb[n].lo[a] = lo[a]; cb[n].hi[a] = hi[a]; plo[a] = fminf(plo[a], lo[a]); phi[a] = fmaxf(phi[a], hi[a]); }
    slot_of[n] = (uint8_t)sl;
    ++n;
  }
  if (!(plo[0] <= phi[0])) { for (int a = 0; a < 3; ++a) plo[a] = phi[a] = 0.0f; }
  for (int c = 0; c < n; ++c)
    if (empty[c]) for (int a = 0; a < 3; ++a) cb[c].lo[a] = cb[c].hi[a] = plo[a];   // nothing in it can be hit (NaN records / empty subtree)
  float* out = nodebox + (size_t)q * 6;
  const bool any = n > 0;
  for (int a = 0; a < 3; ++a) { out[a] = any ? plo[a] : INFINITY; out[3 + a] = any ? phi[a] : -INFINITY; }
  encode_node_boxes(nd, plo, phi, cb, slot_of, n);
  n8[q] = nd;
}

// RefitStaging::host: the root box (32 bytes), the descriptors, then the primitive offsets
constexpr size_t kStagingGeomsAt = 32;
static size_t staging_offs_at(int ngeoms) { return kStagingGeomsAt + ((sizeof(GeomDesc) * ngeoms + 15) & ~size_t(15)); }
size_t refit_staging_bytes(int ngeoms) { return staging_offs_at(ngeoms) + 4 * ((size_t)ngeoms + 1); }

int refit_scene(SceneGPU& s, const GeomDesc* geoms, int ngeoms, cudaStream_t st, char* errmsg, RefitStaging* staging) {
  errmsg[0] = 0;
  if (!s.root_valid || !s.tri_src || s.levels.size() < 2) { snprintf(errmsg, 256, "refit: scene has no kept topology"); return -1; }
  std::vector<uint32_t> offs;
  if (prim_offsets(geoms, ngeoms, offs) != s.total_prims) { snprintf(errmsg, 256, "refit: primitive count changed"); return -1; }
  if (staging && staging->cap < refit_staging_bytes(ngeoms)) { snprintf(errmsg, 256, "internal: refit staging block too small"); return -1; }
  renew_content(s);
  ensure_pool(s.device);
  EventTimer timer;
  float rb_local[6];
  float* rb = rb_local;
  const GeomDesc* src_geoms = geoms;
  const uint32_t* src_offs = offs.data();
  if (staging) {   // the uploads read pinned memory, so neither they nor the root box's copy back wait for the stream
    char* h = static_cast<char*>(staging->host);
    memcpy(h + kStagingGeomsAt, geoms, sizeof(GeomDesc) * ngeoms);
    memcpy(h + staging_offs_at(ngeoms), offs.data(), 4 * ((size_t)ngeoms + 1));
    src_geoms = reinterpret_cast<const GeomDesc*>(h + kStagingGeomsAt);
    src_offs = reinterpret_cast<const uint32_t*>(h + staging_offs_at(ngeoms));
    rb = reinterpret_cast<float*>(h);
    CK(cudaEventRecord(staging->t0, st));
  } else {
    CK(timer.start(st));
  }
  const uint32_t n = s.num_tris;
  DevBuf<GeomDesc> d_geoms; DevBuf<uint32_t> d_offs; DevBuf<float> d_tribox, d_nodebox;
  CK(d_geoms.alloc(ngeoms, st)); CK(d_offs.alloc(ngeoms + 1, st)); CK(d_tribox.alloc((size_t)n * 6, st)); CK(d_nodebox.alloc((size_t)s.num_nodes * 6, st));
  CK(cudaMemcpyAsync(d_geoms.p, src_geoms, sizeof(GeomDesc) * ngeoms, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_offs.p, src_offs, 4 * (ngeoms + 1), cudaMemcpyHostToDevice, st));
  leaf_pack<<<(n + 255) / 256, 256, 0, st>>>(d_geoms.p, d_offs.p, ngeoms, s.tri_src, n, s.tris, s.robust, s.general, d_tribox.p);
  count_launch();
  for (size_t l = s.levels.size() - 1; l-- > 0;) {
    const uint32_t begin = s.levels[l], end = s.levels[l + 1];
    if (end <= begin) continue;
    refit_level<<<(end - begin + 127) / 128, 128, 0, st>>>(s.nodes, begin, end, d_tribox.p, d_nodebox.p);
    count_launch();
  }
  CK(cudaMemcpyAsync(rb, d_nodebox.p, 6 * sizeof(float), cudaMemcpyDeviceToHost, st));
  s.builder = BUILDER_REFIT;
  if (staging) {
    CK(cudaEventRecord(staging->t1, st));
    CK(cudaGetLastError());
    return 0;
  }
  CK(timer.stop(st));
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  for (int a = 0; a < 6; ++a) s.bounds[a] = s.api_bounds[a] = rb[a];
  s.build_ms = timer.ms();
  return 0;
}

void resolve_refit(SceneGPU& s, const RefitStaging& staging) {
  const float* rb = static_cast<const float*>(staging.host);
  for (int a = 0; a < 6; ++a) s.bounds[a] = s.api_bounds[a] = rb[a];
  float ms = 0;
  cudaEventElapsedTime(&ms, staging.t0, staging.t1);
  s.build_ms = ms;
}


// ---------------------------------------------------------------------------------------------------
// linear curves: one neighbour-flag byte per segment (LineSegments::commit, scene_line_segments.cpp:209-232)
// ---------------------------------------------------------------------------------------------------
// The application's flags & 3 when it set a flags buffer, otherwise derived from the index buffer: a segment has a right neighbour
// when the next segment starts at its end vertex, and a left one when the previous segment ends at its start vertex.
__global__ void __launch_bounds__(256) curve_flags(const uint8_t* __restrict__ idx, uint64_t istride, const uint8_t* __restrict__ app,
                                                   uint64_t fstride, uint32_t n, uint8_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (app) { out[i] = app[(uint64_t)i * fstride] & 3u; return; }
  const uint32_t cur = __ldg(reinterpret_cast<const uint32_t*>(idx + (uint64_t)i * istride));
  const bool left = i > 0 && __ldg(reinterpret_cast<const uint32_t*>(idx + (uint64_t)(i - 1) * istride)) + 1u == cur;
  const bool right = i + 1 < n && __ldg(reinterpret_cast<const uint32_t*>(idx + (uint64_t)(i + 1) * istride)) == cur + 1u;
  out[i] = (uint8_t)((left ? 1u : 0u) | (right ? 2u : 0u));   // RTC_CURVE_FLAG_NEIGHBOR_LEFT | _RIGHT
}

int linear_curve_flags(const uint8_t* idx, uint64_t istride, const uint8_t* app, uint64_t fstride, uint32_t n, uint8_t* out, cudaStream_t st) {
  if (n == 0) return 0;
  curve_flags<<<(n + 255) / 256, 256, 0, st>>>(idx, istride, app, fstride, n, out);
  count_launch();
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// two-level scenes: relocation of a sub-BVH into the scene's arrays + host-built top level (see rtk_device.h)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) relocate_nodes(const Node8* __restrict__ src, uint32_t n, Node8* __restrict__ dst, uint32_t node_off, uint32_t tri_off) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Node8 nd = src[i];
  nd.w[4] += node_off;     // child_base (unused when the node has no internal child)
  nd.w[5] += tri_off;      // tri_base   (unused when it has no leaf slot)
  dst[i] = nd;
}


int assemble_scene(SceneGPU& s, SceneGPU* const* subs, int nsubs, cudaStream_t st, char* errmsg) {
  errmsg[0] = 0;
  renew_content(s);
  ensure_pool(s.device);
  CK(alloc_stat(s, st));
  EventTimer timer;
  CK(timer.start(st));
  const uint32_t top_cap = (uint32_t)(2 * nsubs + 8);
  uint64_t nn, nt;
  const std::vector<SubSlot> L = sub_layout(subs, nsubs, top_cap, nn, nt);
  // same layout as last time?  (every sub in its place, with unchanged node / record counts)
  bool same = s.nodes && s.tris && s.subs.size() == L.size();
  for (int i = 0; same && i < nsubs; ++i)
    same = s.subs[i].node_off == L[i].node_off && s.subs[i].nodes == L[i].nodes && s.subs[i].tris == L[i].tris;
  if (!same) {
    if (s.nodes) { cudaFreeAsync(s.nodes, st); s.nodes = nullptr; }
    if (s.tris) { cudaFreeAsync(s.tris, st); s.tris = nullptr; }
    s.subs = L; s.top_cap = top_cap;
    if (nn >= 0x7FFFFFFFull || nt >= 0x7FFFFFFFull) { snprintf(errmsg, 256, "two-level scene too large"); return -1; }
    CK(cudaMallocAsync(reinterpret_cast<void**>(&s.nodes), std::max<uint64_t>(nn, 1) * sizeof(Node8), st));
    CK(cudaMallocAsync(reinterpret_cast<void**>(&s.tris), std::max<uint64_t>(nt, 1) * sizeof(TriRec), st));
    s.num_nodes = (uint32_t)nn; s.num_tris = (uint32_t)nt;
  }
  for (int i = 0; i < nsubs; ++i) {   // a slot is copied when it holds no copy of its sub-BVH as it is now
    const SceneGPU& b = *subs[i];
    SubSlot& sl = s.subs[i];
    if (sl.content == b.content) continue;
    sl.content = b.content;
    if (!b.root_valid) continue;
    relocate_nodes<<<(b.num_nodes + 255) / 256, 256, 0, st>>>(b.nodes, b.num_nodes, s.nodes + sl.node_off, sl.node_off, sl.tri_off);
    count_launch();
    CK(cudaMemcpyAsync(s.tris + sl.tri_off, b.tris, (size_t)b.num_tris * sizeof(TriRec), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(&sl.root, s.nodes + sl.node_off, sizeof(Node8), cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));   // the relocated root nodes are on the host now
  CK(cudaGetLastError());
  // top level on the host: a few hundred meshes at most cost microseconds here
  std::vector<TopItem> items;
  std::vector<Node8> roots;
  for (int a = 0; a < 3; ++a) { s.bounds[a] = s.api_bounds[a] = INFINITY; s.bounds[3 + a] = s.api_bounds[3 + a] = -INFINITY; }
  for (int i = 0; i < nsubs; ++i) {
    roots.push_back(s.subs[i].root);
    if (!subs[i]->root_valid) continue;
    TopItem it;
    for (int a = 0; a < 3; ++a) {
      it.lo[a] = subs[i]->bounds[a]; it.hi[a] = subs[i]->bounds[3 + a];
      s.bounds[a] = s.api_bounds[a] = fminf(s.bounds[a], it.lo[a]); s.bounds[3 + a] = s.api_bounds[3 + a] = fmaxf(s.bounds[3 + a], it.hi[a]);
    }
    it.sub = i;
    items.push_back(it);
  }
  s.root_valid = items.empty() ? 0u : 1u;
  s.levels.clear();
  if (!items.empty()) {
    const std::vector<Node8> top = build_top_level(items, roots);
    if (top.size() > s.top_cap) { snprintf(errmsg, 256, "internal: top level needs %zu of %u nodes", top.size(), s.top_cap); return -1; }
    CK(cudaMemcpyAsync(s.nodes, top.data(), top.size() * sizeof(Node8), cudaMemcpyHostToDevice, st));
    s.levels = {0u, s.num_nodes};
  }
  CK(timer.stop(st));
  CK(cudaStreamSynchronize(st));
  s.build_ms = timer.ms(); s.builder = BUILDER_TWO_LEVEL; s.max_depth = 0; s.sah_cost = 0;
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// instance traversal: the instanced scenes' BVHs and the top level in one node / record array (see rtk_device.h)
// ---------------------------------------------------------------------------------------------------
// records of a sub-BVH moved into the scene's array: descriptor indices shift by `desc_off` (instance records keep their marker)
__global__ void __launch_bounds__(256) relocate_records(const TriRec* __restrict__ src, uint32_t n, TriRec* __restrict__ dst, uint32_t desc_off) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  TriRec t = src[i];
  if (t.geomID != kInstRecord) t.geomID += desc_off;   // b.w: the descriptor
  dst[i] = t;
}

int assemble_instanced(SceneGPU& s, const SceneGPU& top, SceneGPU* const* kids, const uint32_t* kid_desc_off, int nkids, uint32_t top_desc_off,
                       cudaStream_t st, char* errmsg) {
  errmsg[0] = 0;
  renew_content(s);
  CK(alloc_stat(s, st));
  EventTimer timer;
  CK(timer.start(st));
  uint64_t kn, kt;
  std::vector<SubSlot> L = sub_layout(kids, nkids, 1, kn, kt);
  const uint32_t kid_nodes = (uint32_t)kn, kid_tris = (uint32_t)kt;
  const uint32_t tn = top.root_valid ? top.num_nodes : 0u, tt = top.root_valid ? top.num_tris : 0u;
  // the instanced scenes stay where they are while every slot holds the same BVH and the top level fits the room left for it
  bool keep = s.nodes && s.tris && s.subs.size() == L.size() && tn <= s.top_cap && tt <= s.top_tri_cap;
  for (int i = 0; keep && i < nkids; ++i) keep = s.subs[i].content == kids[i]->content;
  if (!keep) {
    if (s.nodes) { cudaFreeAsync(s.nodes, st); s.nodes = nullptr; }
    if (s.tris) { cudaFreeAsync(s.tris, st); s.tris = nullptr; }
    s.top_cap = tn + tn / 2 + 16; s.top_tri_cap = tt + tt / 2 + 16;   // room for a top level that grows a little between commits
    const uint64_t nn = kn + s.top_cap, nt = kt + s.top_tri_cap;
    if (nn >= 0x7FFFFFFFull || nt >= 0x7FFFFFFFull) { snprintf(errmsg, 256, "instanced scene too large"); return -1; }
    CK(cudaMallocAsync(reinterpret_cast<void**>(&s.nodes), nn * sizeof(Node8), st));
    CK(cudaMallocAsync(reinterpret_cast<void**>(&s.tris), nt * sizeof(TriRec), st));
    for (int i = 0; i < nkids; ++i) {
      const SceneGPU& b = *kids[i];
      L[i].content = b.content;
      if (!b.root_valid) continue;
      relocate_nodes<<<(b.num_nodes + 255) / 256, 256, 0, st>>>(b.nodes, b.num_nodes, s.nodes + L[i].node_off, L[i].node_off, L[i].tri_off);
      relocate_records<<<(b.num_tris + 255) / 256, 256, 0, st>>>(b.tris, b.num_tris, s.tris + L[i].tri_off, kid_desc_off[i]);
      count_launch(2);
    }
    s.subs = L;
  }
  s.root_valid = 0;
  s.num_nodes = kid_nodes + tn; s.num_tris = kid_tris + tt;
  if (tn) {   // the top level after the instanced scenes, its root copied to node 0 where traversal starts
    relocate_nodes<<<(tn + 255) / 256, 256, 0, st>>>(top.nodes, tn, s.nodes + kid_nodes, kid_nodes, kid_tris);
    relocate_records<<<(tt + 255) / 256, 256, 0, st>>>(top.tris, tt, s.tris + kid_tris, top_desc_off);
    count_launch(2);
    CK(cudaMemcpyAsync(s.nodes, s.nodes + kid_nodes, sizeof(Node8), cudaMemcpyDeviceToDevice, st));
    s.root_valid = 1;
  }
  CK(timer.stop(st));
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  uint32_t kid_depth = 0;
  for (int i = 0; i < nkids; ++i) kid_depth = std::max(kid_depth, kids[i]->max_depth);
  s.max_depth = top.max_depth + kid_depth;
  for (int a = 0; a < 6; ++a) { s.bounds[a] = top.bounds[a]; s.api_bounds[a] = top.api_bounds[a]; }
  s.levels = {0u, s.num_nodes};
  s.build_ms = timer.ms(); s.builder = top.builder; s.sah_cost = top.sah_cost;
  return 0;
}

}  // namespace rtk
