// emu.cpp -- TEST TOOL ONLY: runs the host instantiation of embree_b200/csrc/rt_core.cuh serially on the CPU so the
// shared core routines (LBVH node construction, BVH8 collapse + slot assignment + box quantisation, the traversal
// loop and the triangle test) can be debugged in a container without a GPU.  It is compiled by tests/emu/build.sh
// into tests/emu/_build/libemu.so, loaded only by the tests (the `emu` fixture), never by the product and never by bench.py.
// The GPU-only parts (radix sort, atomics-based refit, level scheduling) are replaced by trivial serial code here.
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../embree_b200/csrc/rt_core.cuh"

using namespace rtk;

namespace {
struct EmuScene {
  std::vector<Node8> nodes;
  std::vector<TriRec> tris;
  uint32_t root_valid = 0;
  int robust = 0;
  uint32_t depth = 0;
  double sah = 0;
};

struct HostAlloc {
  uint32_t* node_tail;
  uint32_t* tri_tail;
  double* sah_acc;
  uint32_t nodes(uint32_t k) const { uint32_t o = *node_tail; *node_tail += k; return o; }
  uint32_t tris(uint32_t k) const { uint32_t o = *tri_tail; *tri_tail += k; return o; }
  void sah(double x) const { *sah_acc += x; }
};

uint64_t expand21(uint32_t v) {
  uint64_t x = v & 0x1FFFFFull;
  x = (x | x << 32) & 0x1F00000000FFFFull;
  x = (x | x << 16) & 0x1F0000FF0000FFull;
  x = (x | x << 8) & 0x100F00F00F00F00Full;
  x = (x | x << 4) & 0x10C30C30C30C30C3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}
}  // namespace

extern "C" {

// vertices: float[nverts][3] (stride 12), indices: uint32[ntris][3]; mode = collapse policy (0, 1, 2 greedy variants; 3 = SAH-optimal DP)
void* emu_build(const float* verts, uint32_t nverts, const uint32_t* idx, uint32_t ntris, uint32_t geomID, uint32_t mask, int mode) {
  EmuScene* sc = new EmuScene();
  sc->robust = (mode & 0x100) ? 1 : 0;   // bit 8 of `mode`: RTC_SCENE_FLAG_ROBUST (records keep v0,v1,v2)
  mode &= 0xFF;
  std::vector<PrimRef> prims;
  float clo[3] = {INFINITY, INFINITY, INFINITY}, chi[3] = {-INFINITY, -INFINITY, -INFINITY};
  float glo[3] = {INFINITY, INFINITY, INFINITY}, ghi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (uint32_t p = 0; p < ntris; ++p) {
    const uint32_t i0 = idx[3 * p], i1 = idx[3 * p + 1], i2 = idx[3 * p + 2];
    if (i0 >= nverts || i1 >= nverts || i2 >= nverts) continue;
    bool ok = true;
    float lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
      const float x = verts[3 * i0 + a], y = verts[3 * i1 + a], z = verts[3 * i2 + a];
      ok &= (x > -kFltLarge) & (x < kFltLarge) & (y > -kFltLarge) & (y < kFltLarge) & (z > -kFltLarge) & (z < kFltLarge);
      lo[a] = fminf(fminf(x, y), z); hi[a] = fmaxf(fmaxf(x, y), z);
    }
    if (!ok) continue;
    PrimRef pr;
    pr.lox = lo[0]; pr.loy = lo[1]; pr.loz = lo[2]; pr.prim = p;
    pr.hix = hi[0]; pr.hiy = hi[1]; pr.hiz = hi[2]; pr.valid = 1;
    prims.push_back(pr);
    for (int a = 0; a < 3; ++a) {
      clo[a] = fminf(clo[a], lo[a] + hi[a]); chi[a] = fmaxf(chi[a], lo[a] + hi[a]);
      glo[a] = fminf(glo[a], lo[a]); ghi[a] = fmaxf(ghi[a], hi[a]);
    }
  }
  const uint32_t n = (uint32_t)prims.size();
  if (n == 0) return sc;
  std::vector<uint64_t> keys(n);
  for (uint32_t k = 0; k < n; ++k) {
    uint32_t q[3];
    const float c[3] = {prims[k].lox + prims[k].hix, prims[k].loy + prims[k].hiy, prims[k].loz + prims[k].hiz};
    for (int a = 0; a < 3; ++a) {
      const float ext = chi[a] - clo[a];
      float f = ext > 0.0f ? (c[a] - clo[a]) / ext : 0.0f;
      f = fminf(fmaxf(f * 2097152.0f, 0.0f), 2097151.0f);
      q[a] = (uint32_t)f;
    }
    keys[k] = (expand21(q[2]) << 2) | (expand21(q[1]) << 1) | expand21(q[0]);
  }
  std::vector<uint32_t> order(n);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
  std::vector<uint64_t> skeys(n);
  std::vector<uint32_t> sorted(n);  // sorted[j] = index into prims
  for (uint32_t j = 0; j < n; ++j) { skeys[j] = keys[order[j]]; sorted[j] = order[j]; }

  std::vector<Node2> n2(2 * (size_t)n);
  memset(n2.data(), 0, n2.size() * sizeof(Node2));
  for (int i = 0; i + 1 < (int)n; ++i) lbvh_node(skeys.data(), (int)n, i, n2.data());
  for (uint32_t j = 0; j < n; ++j) {
    Node2& lf = n2[n - 1 + j];
    const PrimRef& pr = prims[sorted[j]];
    lf.lox = pr.lox; lf.loy = pr.loy; lf.loz = pr.loz; lf.left = (int)j;
    lf.hix = pr.hix; lf.hiy = pr.hiy; lf.hiz = pr.hiz; lf.right = -1;
    lf.first = j; lf.count = 1;
    if (n == 1) lf.parent = 0xFFFFFFFFu;
  }
  // serial refit: process internal nodes by decreasing range size is not needed -- recurse
  if (n > 1) {
    std::vector<int> stack{0};
    std::vector<int> post;
    while (!stack.empty()) {
      int i = stack.back(); stack.pop_back();
      post.push_back(i);
      if (n2[i].left < (int)n - 1) stack.push_back(n2[i].left);
      if (n2[i].right < (int)n - 1) stack.push_back(n2[i].right);
    }
    for (auto it = post.rbegin(); it != post.rend(); ++it) {
      Node2& nd = n2[*it];
      const Node2 &l = n2[nd.left], &r = n2[nd.right];
      nd.lox = fminf(l.lox, r.lox); nd.loy = fminf(l.loy, r.loy); nd.loz = fminf(l.loz, r.loz);
      nd.hix = fmaxf(l.hix, r.hix); nd.hiy = fmaxf(l.hiy, r.hiy); nd.hiz = fmaxf(l.hiz, r.hiz);
    }
  }
  // SAH-optimal collapse decisions (mode 3): children before parents
  std::vector<float> F((size_t)2 * n * 8);
  std::vector<uint32_t> dec((size_t)2 * n, 0u);
  if (mode >= 3 && n > 1) {
    for (uint32_t j = 0; j < n; ++j) dp_leaf(half_area(n2[n - 1 + j]), 0.3f, &F[(size_t)(n - 1 + j) * 8], &dec[n - 1 + j]);
    std::vector<int> stack{0}, post;
    while (!stack.empty()) {
      int i = stack.back(); stack.pop_back();
      post.push_back(i);
      if (n2[i].left < (int)n - 1) stack.push_back(n2[i].left);
      if (n2[i].right < (int)n - 1) stack.push_back(n2[i].right);
    }
    for (auto it = post.rbegin(); it != post.rend(); ++it) {
      const Node2& nd = n2[*it];
      dp_node(half_area(nd), nd.count, &F[(size_t)nd.left * 8], &F[(size_t)nd.right * 8], 1.0f, 0.3f, &F[(size_t)*it * 8], &dec[*it]);
    }
  }
  // collapse
  std::vector<uint32_t> src(n + 1), tri_src(n);
  sc->nodes.resize(n + 1);
  uint32_t node_tail = 1, tri_tail = 0;
  src[0] = 0;  // root: internal node 0, or leaf 0 when n == 1 (id n-1+0 == 0)
  const float ex = ghi[0] - glo[0], ey = ghi[1] - glo[1], ez = ghi[2] - glo[2];
  const float ra = ex * (ey + ez) + ey * ez;
  const float inv_ra = ra > 0 ? 1.0f / ra : 0.0f;
  HostAlloc alloc{&node_tail, &tri_tail, &sc->sah};
  uint32_t begin = 0, end = 1, depth = 0;
  std::vector<uint32_t> sorted_prim(n);
  for (uint32_t j = 0; j < n; ++j) sorted_prim[j] = prims[sorted[j]].prim;
  while (begin < end) {
    for (uint32_t q = begin; q < end; ++q)
      collapse_node(n2.data(), src.data(), q, sc->nodes.data(), tri_src.data(), sorted_prim.data(), sorted_prim.data(), inv_ra, mode,
                    (mode >= 3 && n > 1) ? dec.data() : nullptr, alloc);
    begin = end; end = node_tail; ++depth;
  }
  sc->nodes.resize(node_tail);
  sc->depth = depth;
  sc->tris.resize(n);
  for (uint32_t t = 0; t < n; ++t) {
    const uint32_t p = tri_src[t];
    const float* a = verts + 3 * (size_t)idx[3 * p];
    const float* b = verts + 3 * (size_t)idx[3 * p + 1];
    const float* c = verts + 3 * (size_t)idx[3 * p + 2];
    TriRec& r = sc->tris[t];
    r.v0x = a[0]; r.v0y = a[1]; r.v0z = a[2]; r.primID = p;
    if (sc->robust) { r.e1x = b[0]; r.e1y = b[1]; r.e1z = b[2]; r.e2x = c[0]; r.e2y = c[1]; r.e2z = c[2]; }
    else {
      r.e1x = sub_rn(a[0], b[0]); r.e1y = sub_rn(a[1], b[1]); r.e1z = sub_rn(a[2], b[2]);
      r.e2x = sub_rn(c[0], a[0]); r.e2y = sub_rn(c[1], a[1]); r.e2z = sub_rn(c[2], a[2]);
    }
    r.geomID = geomID; r.mask = mask;
  }
  sc->root_valid = (tri_tail == n) ? 1 : 0;
  return sc;
}

void emu_free(void* h) { delete static_cast<EmuScene*>(h); }
// copies the scene's nodes (emu_num_nodes x 96 B) and leaf records (48 B each) into `nodes` / `records` when they are not NULL;
// returns the number of records
uint32_t emu_export(void* h, void* nodes, void* records) {
  const EmuScene* sc = static_cast<EmuScene*>(h);
  if (nodes && !sc->nodes.empty()) memcpy(nodes, sc->nodes.data(), sc->nodes.size() * sizeof(Node8));
  if (records && !sc->tris.empty()) memcpy(records, sc->tris.data(), sc->tris.size() * sizeof(TriRec));
  return (uint32_t)sc->tris.size();
}
uint32_t emu_num_nodes(void* h) { return (uint32_t)static_cast<EmuScene*>(h)->nodes.size(); }
uint32_t emu_depth(void* h) { return static_cast<EmuScene*>(h)->depth; }
double emu_sah(void* h) { return static_cast<EmuScene*>(h)->sah; }

// rayhits: RTCRayHit[n] (96 B) when occluded == 0, RTCRay[n] (48 B) when occluded == 1; stats: u64[2] nodes, tris (or NULL)
void emu_trace(void* h, void* rays, uint64_t n, int occluded, uint64_t* stats) {
  EmuScene* sc = static_cast<EmuScene*>(h);
  const Node8* nodes = sc->nodes.data();
  const TriRec* tris = sc->tris.data();
  auto ldn = [nodes](uint32_t node) { NodeW nw; memcpy(nw.w, nodes[node].w, sizeof nw.w); return nw; };
  auto ldt = [tris](uint32_t t, int k) { const uint32_t* w = reinterpret_cast<const uint32_t*>(&tris[t]) + 4 * k; return u32x4{w[0], w[1], w[2], w[3]}; };
  const size_t stride = occluded ? 48 : 96;
  for (uint64_t i = 0; i < n; ++i) {
    char* rec = static_cast<char*>(rays) + i * stride;
    Ray r;
    memcpy(&r, rec, 48);
    Hit hit;
    TravStats st{0, 0};
    bool found;
    if (sc->robust) found = occluded ? traverse<true, true, true>(r, hit, ldn, ldt, sc->root_valid, &st)
                                     : traverse<false, true, true>(r, hit, ldn, ldt, sc->root_valid, &st);
    else found = occluded ? traverse<true, true, false>(r, hit, ldn, ldt, sc->root_valid, &st)
                          : traverse<false, true, false>(r, hit, ldn, ldt, sc->root_valid, &st);
    if (stats) { stats[0] += st.nodes; stats[1] += st.tris; }
    if (!found) continue;
    if (occluded) { float ninf = -INFINITY; memcpy(rec + 32, &ninf, 4); continue; }
    memcpy(rec + 32, &hit.t, 4);
    float h4[5] = {hit.ngx, hit.ngy, hit.ngz, hit.u, hit.v};
    memcpy(rec + 48, h4, 20);
    uint32_t ids[4] = {hit.primID, hit.geomID, 0xFFFFFFFFu, 0xFFFFFFFFu};
    memcpy(rec + 68, ids, 16);
  }
}

// One BVH8 node over n <= 8 child boxes (float[n][6]: lo xyz, hi xyz), built as collapse_node builds it: the node box is
// the union of the children, assign_slots orders them, encode_node_boxes quantises them.  Each ray (float[8]: org xyz,
// tnear, dir xyz, tfar) is set up as traverse() sets it up and tested with node_hitmask; out[i] bit c = child c passed.
void emu_node_hitmask(const float* boxes, int n, const float* rays, uint64_t m, uint32_t* out) {
  ChildBox cb[8];
  float plo[3] = {INFINITY, INFINITY, INFINITY}, phi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int c = 0; c < n; ++c)
    for (int a = 0; a < 3; ++a) {
      cb[c].lo[a] = boxes[6 * c + a]; cb[c].hi[a] = boxes[6 * c + 3 + a];
      plo[a] = fminf(plo[a], cb[c].lo[a]); phi[a] = fmaxf(phi[a], cb[c].hi[a]);
    }
  uint8_t slot_of[8];
  assign_slots(cb, n, plo, phi, slot_of);
  Node8 nd;
  for (int k = 0; k < 24; ++k) nd.w[k] = 0;
  encode_node_boxes(nd, plo, phi, cb, slot_of, n);
  uint32_t imask = 0;
  for (int c = 0; c < n; ++c) imask |= 1u << slot_of[c];
  nd.w[3] = (nd.w[3] & 0x00FFFFFFu) | (imask << 24);   // every child internal: the hit slots come back in bits 31:24
  for (uint64_t i = 0; i < m; ++i) {
    const float* r = rays + 8 * i;
    const float idx = rcp_safe(r[4]), idy = rcp_safe(r[5]), idz = rcp_safe(r[6]);
    const bool negx = idx < 0.0f, negy = idy < 0.0f, negz = idz < 0.0f;
    const uint32_t oct = (negx ? 1u : 0u) | (negy ? 2u : 0u) | (negz ? 4u : 0u);
    const uint32_t hm = node_hitmask(nd.w, r[0], r[1], r[2], idx, idy, idz, negx, negy, negz, fmaxf(r[3], 0.0f),
                                     fmaxf(r[7], 0.0f), 7u - oct);
    const uint32_t slots = xor_permute8(hm >> 24, 7u - oct);
    uint32_t mask = 0;
    for (int c = 0; c < n; ++c) mask |= ((slots >> slot_of[c]) & 1u) << c;
    out[i] = mask;
  }
}

}  // extern "C"

// ---- experiment (test tool): the same BVH8 traversed with exact front-to-back child ordering (per-child stack
// entries sorted by entry distance, far entries culled against the current hit) to measure how many node visits the
// octant-order approximation of the production traversal costs.
extern "C" void emu_trace_sorted(void* h, void* rays, uint64_t n, uint64_t* stats) {
  EmuScene* sc = static_cast<EmuScene*>(h);
  const Node8* nodes = sc->nodes.data();
  const TriRec* tris = sc->tris.data();
  for (uint64_t ri = 0; ri < n; ++ri) {
    char* rec = static_cast<char*>(rays) + ri * 96;
    Ray r; memcpy(&r, rec, 48);
    if (!sc->root_valid) continue;
    const float idx = rcp_safe(r.dx), idy = rcp_safe(r.dy), idz = rcp_safe(r.dz);
    float tfar = r.tfar; bool found = false; Hit hit{};
    struct E { uint32_t node; float t; };
    std::vector<E> st; st.push_back({0u, 0.0f});
    while (!st.empty()) {
      E e = st.back(); st.pop_back();
      if (e.t > tfar) continue;
      const Node8& nd = nodes[e.node];
      stats[0]++;
      const uint32_t ex = nd.w[3];
      const float sx = u2f((ex & 0xFF) << 23) * idx, sy = u2f(((ex >> 8) & 0xFF) << 23) * idy, sz = u2f(((ex >> 16) & 0xFF) << 23) * idz;
      const float bx = (u2f(nd.w[0]) - r.ox) * idx, by = (u2f(nd.w[1]) - r.oy) * idy, bz = (u2f(nd.w[2]) - r.oz) * idz;
      const uint8_t* q = reinterpret_cast<const uint8_t*>(&nd.w[kNodePlaneWord]);   // qlox[8] qloy[8] qloz[8] qhix[8] qhiy[8] qhiz[8]
      const uint32_t imask = ex >> 24;
      E kids[8]; int nk = 0;
      for (int s = 0; s < 8; ++s) {
        const uint32_t lm = node_leafmask_raw(nd.w, s) & 0xFFFFFFu;
        if (lm == 0 && !(imask & (1u << s))) continue;
        const float lx = q[s], ly = q[8 + s], lz = q[16 + s], hx = q[24 + s], hy = q[32 + s], hz = q[40 + s];
        const float tnx = (idx < 0 ? hx : lx) * sx + bx, tfx = (idx < 0 ? lx : hx) * sx + bx;
        const float tny = (idy < 0 ? hy : ly) * sy + by, tfy = (idy < 0 ? ly : hy) * sy + by;
        const float tnz = (idz < 0 ? hz : lz) * sz + bz, tfz = (idz < 0 ? lz : hz) * sz + bz;
        const float tmin = fmaxf(fmaxf(tnx, tny), fmaxf(tnz, fmaxf(r.tnear, 0.0f)));
        const float tmax = fminf(fminf(tfx, tfy), fminf(tfz, fmaxf(tfar, 0.0f))) * 1.0000003f;
        if (!(tmin <= tmax)) continue;
        if (imask & (1u << s)) {
          const uint32_t child = nd.w[4] + (uint32_t)popc32(imask & ((1u << s) - 1u));
          kids[nk++] = {child, tmin};
        } else {
          for (uint32_t m = lm; m;) {       // highest bit first, as the production loop
            const int tb = 31 - clz32(m);
            m &= ~(1u << tb);
            const TriRec& t = tris[nd.w[5] + (uint32_t)tb];
            stats[1]++;
            TriHit th;
            if (tri_test(r, tfar, t.v0x, t.v0y, t.v0z, t.e1x, t.e1y, t.e1z, t.e2x, t.e2y, t.e2z, th) && (t.mask & r.mask)) {
              const float rcp = 1.0f / th.absDen;
              hit.t = th.T * rcp; hit.u = th.U * rcp; hit.v = th.V * rcp; hit.ngx = th.ngx; hit.ngy = th.ngy; hit.ngz = th.ngz;
              hit.primID = t.primID; hit.geomID = t.geomID; tfar = hit.t; found = true;
            }
          }
        }
      }
      std::sort(kids, kids + nk, [](const E& a, const E& b) { return a.t > b.t; });  // far first -> near popped first
      for (int k = 0; k < nk; ++k) st.push_back(kids[k]);
    }
    if (!found) continue;
    memcpy(rec + 32, &hit.t, 4);
    float h4[5] = {hit.ngx, hit.ngy, hit.ngz, hit.u, hit.v};
    memcpy(rec + 48, h4, 20);
    uint32_t ids[4] = {hit.primID, hit.geomID, 0xFFFFFFFFu, 0xFFFFFFFFu};
    memcpy(rec + 68, ids, 16);
  }
}

// ---- experiment (test tool): the production traversal order, logging the per-ray operation sequence -- 'N' = one node
// step (fetch + 8-child slab test), 'T' = one triangle test, each ray terminated by 0 -- for the offline warp-scheduling
// model in scripts/warp_model.py.  Same loop as rtk::traverse<false,...> (closest hit, Moeller-Trumbore).
extern "C" uint64_t emu_trace_ops(void* h, void* rays, uint64_t n, uint8_t* ops, uint64_t cap) {
  EmuScene* sc = static_cast<EmuScene*>(h);
  const Node8* nodes = sc->nodes.data();
  const TriRec* tris = sc->tris.data();
  uint64_t len = 0;
  auto put = [&](uint8_t c) { if (len < cap) ops[len] = c; ++len; };
  for (uint64_t ri = 0; ri < n; ++ri) {
    char* rec = static_cast<char*>(rays) + ri * 96;
    Ray r; memcpy(&r, rec, 48);
    if (sc->root_valid) {
      const float idx = rcp_safe(r.dx), idy = rcp_safe(r.dy), idz = rcp_safe(r.dz);
      const bool negx = idx < 0.0f, negy = idy < 0.0f, negz = idz < 0.0f;
      const uint32_t oct = (negx ? 1u : 0u) | (negy ? 2u : 0u) | (negz ? 4u : 0u);
      const float tnear_c = fmaxf(r.tnear, 0.0f);
      float tfar_c = fmaxf(r.tfar, 0.0f), tfar_tri = r.tfar;
      uint32_t stack_x[kStackSize], stack_y[kStackSize];
      int sp = 0;
      uint32_t ngx = 0, ngy = 0x80000000u, tgx = 0, tgy = 0;
      while (true) {
        if (ngy & 0xFF000000u) {
          const int bit = 31 - clz32(ngy);
          ngy &= ~(1u << bit);
          if (ngy & 0xFF000000u) { stack_x[sp] = ngx; stack_y[sp] = ngy; ++sp; }
          const uint32_t slot = ((uint32_t)(bit - 24)) ^ (7u - oct);
          const uint32_t ni = ngx + (uint32_t)popc32(ngy & 0xFFu & ((1u << slot) - 1u));
          const uint32_t* w = nodes[ni].w;
          put('N');
          const uint32_t hm = node_hitmask(w, r.ox, r.oy, r.oz, idx, idy, idz, negx, negy, negz, tnear_c, tfar_c, 7u - oct);
          ngx = w[4]; ngy = (hm & 0xFF000000u) | (w[3] >> 24);
          tgx = w[5]; tgy = hm & 0x00FFFFFFu;
        } else { tgx = ngx; tgy = ngy; ngx = 0; ngy = 0; }
        while (tgy) {
          const int tb = 31 - clz32(tgy);
          tgy &= ~(1u << tb);
          const uint32_t* t = reinterpret_cast<const uint32_t*>(&tris[tgx + (uint32_t)tb]);
          put('T');
          TriHit th;
          if (tri_test(r, tfar_tri, u2f(t[0]), u2f(t[1]), u2f(t[2]), u2f(t[4]), u2f(t[5]), u2f(t[6]), u2f(t[8]), u2f(t[9]), u2f(t[10]), th) &&
              (t[11] & r.mask) != 0) {
            tfar_tri = th.T * (1.0f / th.absDen);
            tfar_c = fmaxf(tfar_tri, 0.0f);
          }
        }
        if ((ngy & 0xFF000000u) == 0) {
          if (sp == 0) break;
          --sp; ngx = stack_x[sp]; ngy = stack_y[sp];
        }
      }
    }
    put(0);
  }
  return len;
}

// ---- round linear curve segment test (rt_core.cuh curve_test), host instantiation of the routine the GENERAL = 2 trace kernels
// call per curve record.  ray8 = ox oy oz tnear dx dy dz tfar; v* = float4 vertices; out5 = t, u, Ng.xyz.
extern "C" int emu_curve_test(const float* ray8, const float* v0, const float* v1, int hasL, const float* vL, int hasR, const float* vR, float* out5) {
  CurveHit h;
  const CurveVtx a{v0[0], v0[1], v0[2], v0[3]}, b{v1[0], v1[1], v1[2], v1[3]}, l{vL[0], vL[1], vL[2], vL[3]}, r{vR[0], vR[1], vR[2], vR[3]};
  if (!curve_test(ray8[0], ray8[1], ray8[2], ray8[4], ray8[5], ray8[6], ray8[3], ray8[7], a, b, hasL != 0, l, hasR != 0, r, h)) return 0;
  out5[0] = h.t; out5[1] = h.u; out5[2] = h.ngx; out5[3] = h.ngy; out5[4] = h.ngz;
  return 1;
}

extern "C" int emu_flat_curve_test(const float* ray8, const float* v0, const float* v1, float* out5) {
  CurveHit h;
  const CurveVtx a{v0[0], v0[1], v0[2], v0[3]}, b{v1[0], v1[1], v1[2], v1[3]};
  if (!flat_curve_test(ray8[0], ray8[1], ray8[2], ray8[4], ray8[5], ray8[6], ray8[3], ray8[7], a, b, h)) return 0;
  out5[0] = h.t; out5[1] = h.u; out5[2] = h.ngx; out5[3] = h.ngy; out5[4] = h.ngz;
  return 1;
}

// ---- linear curves (rt_core.cuh curve_test / flat_curve_test), host instantiation: the segments idx[0..n) of a FLOAT4 vertex buffer in
// order against the ray as shortened by the hits so far; flags[i] bit 0 / bit 1: the segment has a left / right neighbour (vertex
// idx - 1 / idx + 2).  Returns the winning position in idx or -1; out6 = t, u, v, Ng.xyz.
extern "C" int emu_linear_curve_closest(const float* ray8, const float* verts, const unsigned* idx, const unsigned char* flags, int n, int flat, float* out6) {
  int best = -1;
  float tfar = ray8[7];
  for (int i = 0; i < n; ++i) {
    const float* a = verts + 4 * (size_t)idx[i];
    const CurveVtx v0{a[0], a[1], a[2], a[3]}, v1{a[4], a[5], a[6], a[7]};
    const bool hasL = flags[i] & 1, hasR = flags[i] & 2;
    const CurveVtx vL = hasL ? CurveVtx{a[-4], a[-3], a[-2], a[-1]} : v0, vR = hasR ? CurveVtx{a[8], a[9], a[10], a[11]} : v1;
    CurveHit h;
    const bool hit = flat ? flat_curve_test(ray8[0], ray8[1], ray8[2], ray8[4], ray8[5], ray8[6], ray8[3], tfar, v0, v1, h)
                          : curve_test(ray8[0], ray8[1], ray8[2], ray8[4], ray8[5], ray8[6], ray8[3], tfar, v0, v1, hasL, vL, hasR, vR, h);
    if (!hit) continue;
    best = i; tfar = h.t;
    out6[0] = h.t; out6[1] = h.u; out6[2] = h.v; out6[3] = h.ngx; out6[4] = h.ngy; out6[5] = h.ngz;
  }
  return best;
}

// ---- point primitives (rt_core.cuh point_test), host instantiation.  verts = n x (centre, radius), normals = n x float3 (oriented
// discs) or NULL; kind 0 sphere, 1 ray-facing disc, 2 oriented disc.  Every point is tested in order against the ray as shortened
// by the hits so far (the sequential leaf loop); returns the winning point or -1.  out6 = t, u, v, Ng.xyz.
extern "C" int emu_point_closest(const float* ray8, const float* verts, const float* normals, int n, int kind, float* out6) {
  int best = -1;
  float tfar = ray8[7];
  for (int i = 0; i < n; ++i) {
    CurveHit h;
    const float* v = verts + 4 * (size_t)i;
    const float zero[3] = {0.0f, 0.0f, 0.0f};
    const float* nn = normals ? normals + 3 * (size_t)i : zero;
    if (!point_test(ray8[0], ray8[1], ray8[2], ray8[4], ray8[5], ray8[6], ray8[3], tfar, v[0], v[1], v[2], v[3], nn[0], nn[1], nn[2], kind, h)) continue;
    best = i; tfar = h.t;
    out6[0] = h.t; out6[1] = h.u; out6[2] = h.v; out6[3] = h.ngx; out6[4] = h.ngy; out6[5] = h.ngz;
  }
  return best;
}

// ---- flat cubic curves (rt_core.cuh flat_cubic_test + curve_basis_table), host instantiation.  cps = n curves x 4 control points
// x float4 (Hermite input already converted); every curve is tested in order against the ray as shortened by the hits so far
// (the sequential leaf loop); returns the winning curve or -1.  out6 = t, u, v, Ng.xyz.
extern "C" int emu_flat_cubic_closest(const float* ray8, const float* cps, int n, unsigned basis, int N, float* out6) {
  float tab[8 * (kMaxTess + 1)];
  curve_basis_table(basis, N, tab);
  float tfar = ray8[7];
  int win = -1;
  for (int i = 0; i < n; ++i) {
    CurveVtx cp[4];
    for (int k = 0; k < 4; ++k) cp[k] = CurveVtx{cps[i * 16 + k * 4], cps[i * 16 + k * 4 + 1], cps[i * 16 + k * 4 + 2], cps[i * 16 + k * 4 + 3]};
    CurveHit h;
    if (!flat_cubic_test(ray8[0], ray8[1], ray8[2], ray8[4], ray8[5], ray8[6], ray8[3], tfar, cp, basis, N, tab, h)) continue;
    tfar = h.t; win = i;
    out6[0] = h.t; out6[1] = h.u; out6[2] = h.v; out6[3] = h.ngx; out6[4] = h.ngy; out6[5] = h.ngz;
  }
  return win;
}

// ---- experiment (test tool): the production traversal order (leaf slots inside the node step, children in octant order)
// with the entry distance of the pending children remembered.  mode 0: production (every pending child is visited);
// mode 1: a pending child whose entry distance lies behind the current hit is skipped (per-child culling at pop time, what
// the reference's stack does with its per-entry distance); mode 2: a pending GROUP is dropped when the smallest entry
// distance of all children hit in that node lies behind the current hit (16 spare bits of the 8-byte stack entry would do).
// stats[0] += node visits, stats[1] += triangle tests.
namespace {
struct CullCtx { const Node8* nodes; const TriRec* tris; Ray r; float idx, idy, idz, tfar; uint32_t oct; int mode; uint64_t* stats; };
void cull_visit(CullCtx& c, uint32_t node) {
  const Node8& nd = c.nodes[node];
  c.stats[0]++;
  const uint32_t ex = nd.w[3];
  const float sx = u2f((ex & 0xFF) << 23) * c.idx, sy = u2f(((ex >> 8) & 0xFF) << 23) * c.idy, sz = u2f(((ex >> 16) & 0xFF) << 23) * c.idz;
  const float bx = (u2f(nd.w[0]) - c.r.ox) * c.idx, by = (u2f(nd.w[1]) - c.r.oy) * c.idy, bz = (u2f(nd.w[2]) - c.r.oz) * c.idz;
  const uint8_t* q = reinterpret_cast<const uint8_t*>(&nd.w[kNodePlaneWord]);
  const uint32_t imask = ex >> 24;
  float tmin_s[8]; bool hit_s[8]; uint32_t leaf = 0;
  float gmin = INFINITY;
  for (int s = 0; s < 8; ++s) {
    hit_s[s] = false;
    const uint32_t lm = node_leafmask_raw(nd.w, s) & 0xFFFFFFu;
    if (lm == 0 && !(imask & (1u << s))) continue;
    const float lx = q[s], ly = q[8 + s], lz = q[16 + s], hx = q[24 + s], hy = q[32 + s], hz = q[40 + s];
    const float tnx = (c.idx < 0 ? hx : lx) * sx + bx, tfx = (c.idx < 0 ? lx : hx) * sx + bx;
    const float tny = (c.idy < 0 ? hy : ly) * sy + by, tfy = (c.idy < 0 ? ly : hy) * sy + by;
    const float tnz = (c.idz < 0 ? hz : lz) * sz + bz, tfz = (c.idz < 0 ? lz : hz) * sz + bz;
    const float tmin = fmaxf(fmaxf(tnx, tny), fmaxf(tnz, fmaxf(c.r.tnear, 0.0f)));
    const float tmax = fminf(fminf(tfx, tfy), fminf(tfz, fmaxf(c.tfar, 0.0f))) * 1.0000003f;
    if (!(tmin <= tmax)) continue;
    if (imask & (1u << s)) { hit_s[s] = true; tmin_s[s] = tmin; gmin = fminf(gmin, tmin); }
    else leaf |= lm;
  }
  for (uint32_t m = leaf; m;) {
    const int tb = 31 - clz32(m);
    m &= ~(1u << tb);
    const TriRec& t = c.tris[nd.w[5] + (uint32_t)tb];
    c.stats[1]++;
    TriHit th;
    if (tri_test(c.r, c.tfar, t.v0x, t.v0y, t.v0z, t.e1x, t.e1y, t.e1z, t.e2x, t.e2y, t.e2z, th) && (t.mask & c.r.mask)) c.tfar = th.T * (1.0f / th.absDen);
  }
  for (int b = 7; b >= 0; --b) {
    const int s = b ^ (int)(7u - c.oct);
    if (!hit_s[s]) continue;
    if (c.mode == 1 && tmin_s[s] > c.tfar) continue;
    if (c.mode == 2 && gmin > c.tfar) break;
    cull_visit(c, nd.w[4] + (uint32_t)popc32(imask & ((1u << s) - 1u)));
  }
}
}  // namespace
extern "C" void emu_trace_cull(void* h, void* rays, uint64_t n, int mode, uint64_t* stats) {
  EmuScene* sc = static_cast<EmuScene*>(h);
  if (!sc->root_valid) return;
  for (uint64_t ri = 0; ri < n; ++ri) {
    CullCtx c;
    c.nodes = sc->nodes.data(); c.tris = sc->tris.data(); c.mode = mode; c.stats = stats;
    memcpy(&c.r, static_cast<char*>(rays) + ri * 96, 48);
    c.idx = rcp_safe(c.r.dx); c.idy = rcp_safe(c.r.dy); c.idz = rcp_safe(c.r.dz);
    c.oct = (c.idx < 0 ? 1u : 0u) | (c.idy < 0 ? 2u : 0u) | (c.idz < 0 ? 4u : 0u);
    c.tfar = c.r.tfar;
    cull_visit(c, 0);
  }
}

// ---- round cubic curves (rt_core.cuh round_cubic_test), host instantiation; same calling convention as emu_flat_cubic_closest
extern "C" int emu_round_cubic_closest(const float* ray8, const float* cps, int n, unsigned basis, float* out6) {
  float tfar = ray8[7];
  int win = -1;
  for (int i = 0; i < n; ++i) {
    CurveVtx cp[4];
    for (int k = 0; k < 4; ++k) cp[k] = CurveVtx{cps[i * 16 + k * 4], cps[i * 16 + k * 4 + 1], cps[i * 16 + k * 4 + 2], cps[i * 16 + k * 4 + 3]};
    CurveHit h;
    if (!round_cubic_test(ray8[0], ray8[1], ray8[2], ray8[4], ray8[5], ray8[6], ray8[3], tfar, cp, basis, h)) continue;
    tfar = h.t; win = i;
    out6[0] = h.t; out6[1] = h.u; out6[2] = h.v; out6[3] = h.ngx; out6[4] = h.ngy; out6[5] = h.ngz;
  }
  return win;
}

// ---- two-level assembly on the host (embree_b200/csrc/two_level.h + the relocation of build.cu relocate_nodes): `n` emulated scenes
// become ONE scene -- [top level | scene 0 nodes | scene 1 nodes ...], node / record indices relocated, root-node copies under a
// top-level BVH8 -- exactly what assemble_scene does on the device.  Returns a new handle (free with emu_free).
#include "../../embree_b200/csrc/two_level.h"
extern "C" void* emu_assemble(void** handles, int n) {
  EmuScene* out = new EmuScene();
  std::vector<TopItem> items;
  std::vector<Node8> roots(n);
  const uint32_t top_cap = (uint32_t)(2 * n + 8);
  uint32_t nn = top_cap, nt = 0;
  std::vector<uint32_t> noff(n), toff(n);
  for (int i = 0; i < n; ++i) {
    EmuScene* s = static_cast<EmuScene*>(handles[i]);
    noff[i] = nn; toff[i] = nt;
    if (!s->root_valid) continue;
    nn += (uint32_t)s->nodes.size(); nt += (uint32_t)s->tris.size();
  }
  out->nodes.resize(nn); out->tris.resize(nt);
  for (int i = 0; i < n; ++i) {
    EmuScene* s = static_cast<EmuScene*>(handles[i]);
    if (!s->root_valid) continue;
    out->robust = s->robust;
    for (size_t k = 0; k < s->nodes.size(); ++k) { Node8 nd = s->nodes[k]; nd.w[4] += noff[i]; nd.w[5] += toff[i]; out->nodes[noff[i] + k] = nd; }
    for (size_t k = 0; k < s->tris.size(); ++k) out->tris[toff[i] + k] = s->tris[k];
    roots[i] = out->nodes[noff[i]];
    TopItem it;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    // the mesh box: decoded from its root node's grid (conservative) -- p + [0, 255] * 2^e per axis covers all children
    const Node8& r = s->nodes[0];
    for (int a = 0; a < 3; ++a) { lo[a] = u2f(r.w[a]); hi[a] = lo[a] + 255.0f * u2f(((r.w[3] >> (8 * a)) & 0xFFu) << 23); }
    for (int a = 0; a < 3; ++a) { it.lo[a] = lo[a]; it.hi[a] = hi[a]; }
    it.sub = i;
    items.push_back(it);
  }
  if (!items.empty()) {
    const std::vector<Node8> top = build_top_level(items, roots);
    if (top.size() > top_cap) { delete out; return nullptr; }
    for (size_t k = 0; k < top.size(); ++k) out->nodes[k] = top[k];
    out->root_valid = 1;
  }
  return out;
}
