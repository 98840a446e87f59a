// trace.cu -- closest-hit / any-hit traversal kernels for sm_90a.
//
// Replaces kernels/bvh/bvh_intersector1.cpp:31-197 (single ray) and, through the packet I/O adapters below,
// kernels/bvh/bvh_intersector_hybrid.cpp:106-370,600-783 (rtcIntersect4/8/16, rtcOccluded4/8/16): on this
// device a "packet" is only an I/O layout -- every lane is traced as an independent ray of a 32-wide warp, which is
// what the reference's hybrid traverser degenerates to below its switch threshold (bvh_intersector_hybrid.h:33-37).
#include <stdio.h>

#include "record_tests.cuh"
#include "rtk_device.h"

namespace rtk {

// ---- loads of the BVH through the read-only path -----------------------------------------------------------------
// A node is 96 bytes, 32-byte aligned: three sectors.  sm_90 has no 256-bit load, so each sector is two 128-bit
// read-only loads (ld.global.nc.v4.b32 -> LDG.E.128.CONSTANT) issued back to back; both halves hit the same sector.
__device__ __forceinline__ void ldg256(const void* p, uint32_t* d) {
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3]), "=r"(d[4]), "=r"(d[5]), "=r"(d[6]), "=r"(d[7])
               : "l"(p));
}
__device__ __forceinline__ void load_node(const Node8* __restrict__ nodes, uint32_t node_index, NodeW& nw) {
  const char* np = reinterpret_cast<const char*>(nodes) + (size_t)node_index * sizeof(Node8);
  ldg256(np, nw.w); ldg256(np + 32, nw.w + 8); ldg256(np + 64, nw.w + 16);
}

// ---- ray / hit I/O adapters ------------------------------------------------------------------------------------
// K == 1 : AoS RTCRayHit (96 B, hit at +48) or RTCRay (48 B).  K in {4,8,16}: SoA inside each packet
// (include/embree4/rtcore_ray.h:55-184): field f of lane l of packet m lives at m*PACKET + (f*K + l)*4.
template <int K, bool OCCLUDED>
struct RayIO;

template <bool OCCLUDED>
struct RayIO<1, OCCLUDED> {
  static constexpr int kStride = OCCLUDED ? 48 : 96;
  static constexpr int kRayBytes = kStride;   // bytes per ray of a contiguous 32-ray block
  // `base` is either p.rays (i = global ray index) or a shared-memory copy of one 32-ray block (i = index in block)
  static __device__ __forceinline__ void load(const char* base, unsigned long long i, Ray& r) {
    const float4* src = reinterpret_cast<const float4*>(base + i * kStride);
    const float4 a = src[0], b = src[1], c = src[2];
    r.ox = a.x; r.oy = a.y; r.oz = a.z; r.tnear = a.w;
    r.dx = b.x; r.dy = b.y; r.dz = b.z; r.time = b.w;
    r.tfar = c.x; r.mask = __float_as_uint(c.y); r.id = __float_as_uint(c.z); r.flags = __float_as_uint(c.w);
  }
  static __device__ __forceinline__ void store_tfar(const TraceParams& p, unsigned long long i, float tfar) {
    *reinterpret_cast<float*>(static_cast<char*>(p.rays) + i * kStride + 32) = tfar;
  }
  static __device__ __forceinline__ void store_hit(const TraceParams& p, unsigned long long i, const Hit& h, uint32_t instID, uint32_t instPrimID) {
    char* rec = static_cast<char*>(p.rays) + i * kStride;
    *reinterpret_cast<float*>(rec + 32) = h.t;
    float4 a, b;
    a.x = h.ngx; a.y = h.ngy; a.z = h.ngz; a.w = h.u;
    b.x = h.v; b.y = __uint_as_float(h.primID); b.z = __uint_as_float(h.geomID); b.w = __uint_as_float(instID);
    *reinterpret_cast<float4*>(rec + 48) = a;
    *reinterpret_cast<float4*>(rec + 64) = b;
    *reinterpret_cast<uint32_t*>(rec + 80) = instPrimID;
  }
};

template <int K, bool OCCLUDED>
struct RayIO {
  static constexpr int kPacket = (OCCLUDED ? 12 : 21) * 4 * K;
  static constexpr int kRayBytes = (OCCLUDED ? 12 : 21) * 4;   // 32 consecutive rays = 32/K consecutive packets
  static __device__ __forceinline__ char* field(const TraceParams& p, unsigned long long i, int f) {
    return static_cast<char*>(p.rays) + (i / K) * kPacket + ((size_t)f * K + (i % K)) * 4;
  }
  static __device__ __forceinline__ const char* cfield(const char* base, unsigned long long i, int f) {
    return base + (i / K) * kPacket + ((size_t)f * K + (i % K)) * 4;
  }
  static __device__ __forceinline__ void load(const char* base, unsigned long long i, Ray& r) {
    r.ox = *reinterpret_cast<const float*>(cfield(base, i, 0)); r.oy = *reinterpret_cast<const float*>(cfield(base, i, 1));
    r.oz = *reinterpret_cast<const float*>(cfield(base, i, 2)); r.tnear = *reinterpret_cast<const float*>(cfield(base, i, 3));
    r.dx = *reinterpret_cast<const float*>(cfield(base, i, 4)); r.dy = *reinterpret_cast<const float*>(cfield(base, i, 5));
    r.dz = *reinterpret_cast<const float*>(cfield(base, i, 6)); r.time = *reinterpret_cast<const float*>(cfield(base, i, 7));
    r.tfar = *reinterpret_cast<const float*>(cfield(base, i, 8)); r.mask = *reinterpret_cast<const uint32_t*>(cfield(base, i, 9));
    r.id = 0; r.flags = 0;
  }
  static __device__ __forceinline__ void store_tfar(const TraceParams& p, unsigned long long i, float tfar) {
    *reinterpret_cast<float*>(field(p, i, 8)) = tfar;
  }
  static __device__ __forceinline__ void store_hit(const TraceParams& p, unsigned long long i, const Hit& h, uint32_t instID, uint32_t instPrimID) {
    *reinterpret_cast<float*>(field(p, i, 8)) = h.t;
    *reinterpret_cast<float*>(field(p, i, 12)) = h.ngx; *reinterpret_cast<float*>(field(p, i, 13)) = h.ngy;
    *reinterpret_cast<float*>(field(p, i, 14)) = h.ngz; *reinterpret_cast<float*>(field(p, i, 15)) = h.u;
    *reinterpret_cast<float*>(field(p, i, 16)) = h.v; *reinterpret_cast<uint32_t*>(field(p, i, 17)) = h.primID;
    *reinterpret_cast<uint32_t*>(field(p, i, 18)) = h.geomID; *reinterpret_cast<uint32_t*>(field(p, i, 19)) = instID;
    *reinterpret_cast<uint32_t*>(field(p, i, 20)) = instPrimID;
  }
};

// one 32-byte aligned sector written as two 128-bit global stores (sm_90 has no 256-bit store)
__device__ __forceinline__ void store_256(void* dst, float a0, float a1, float a2, float a3, float a4, float a5, float a6, float a7) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};\n\t"
               "st.global.v4.f32 [%0+16], {%5, %6, %7, %8};" ::"l"(dst), "f"(a0), "f"(a1), "f"(a2), "f"(a3), "f"(a4),
               "f"(a5), "f"(a6), "f"(a7)
               : "memory");
}

constexpr int TRACE_THREADS = 128;
constexpr int TRACE_WARPS = TRACE_THREADS / 32;

// ---- TMA bulk prefetch of one 32-ray block (1.5 .. 3 KB contiguous) into L2 ------------------------------------------
// Staging the blocks in shared memory (cp.async.bulk.shared + mbarrier) instead would take 24 KB of shared memory per
// CTA x 8 CTAs/SM out of the 256 KB an SM shares between L1 and shared memory, and the BVH lives on L1 hits.  The bulk
// prefetch keeps the TMA unit pulling the ray stream ahead of the warps without costing L1 capacity.
__device__ __forceinline__ void tma_prefetch_l2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}

// compile-time experiment switch (A/B builds only; the shipped value is the default below)
#ifndef RTK_MIN_BLOCKS
#define RTK_MIN_BLOCKS 8   // resident CTAs per SM the register allocation is bounded for (8 x 128 threads -> 64 registers)
#endif
#ifndef RTK_SMEM_STACK
#define RTK_SMEM_STACK 8   // traversal-stack entries per lane kept in shared memory (deeper ones spill to local memory)
#endif
#ifndef RTK_TRI2
#define RTK_TRI2 1   // a lane with two or more pending triangles tests two per triangle step (both records fetched together)
#endif

// Persistent warps.  Every warp owns the 32-ray blocks w, w+W, w+2W, ... of the stream (W = warps in the grid).  When
// a warp starts consuming a block, lane 0 issues a TMA bulk prefetch (cp.async.bulk.prefetch.L2) of the block two ahead,
// so the ray records are L2-resident by the time lanes load them.  A lane is EMPTY (no ray), TRACING, or DONE (its ray
// has terminated, the result is still in registers).  One loop iteration =
//   1. when enough lanes are not TRACING: DONE lanes write their hit records back together (the winning triangle's
//      record is re-read for Ng and the ids: batching overlaps those loads across lanes instead of paying the latency
//      once per ray), then EMPTY lanes take the next unassigned rays of the block (ballot + popc ranking, no atomics);
//   2. at most one node step (pop a child of the current node group, fetch the 96-byte node, slab-test 8 children);
//   3. at most one triangle step, batched across the warp;
//   4. pop.  The top stack entry lives in registers as a write-back cache of the local-memory stack: a pop that
//      follows a push costs no memory access, and a local-memory load is only waited for when two pops follow each
//      other (reloading the register copy on every pop stalls on the local-memory load).
// The phases are warp-synchronous so lanes in the same phase execute together instead of serialising through a
// per-thread while-while loop.
//
// GATHER (K == 1 closest hit only) adds the fused multi-GPU hit gather: every ray also produces one compact 32-byte
// record {tfar, Ng, u, v, primID, geomID} in `compact_out`, which may be a PEER GPU's memory (NVLink).
//   GATHER 1: the lane stores its record when the ray is written back -- one sector (two 128-bit stores).
//   GATHER 2: records are first stored to a LOCAL staging buffer (p.stage, same indexing); the warp tracks which records of
//             its two newest 32-ray blocks have arrived and, when a block is complete, re-reads its 1 KB (L2 hits) and sends
//             it as ONE warp-wide store of eight full 128-byte lines.  With several peers storing into rank 0, single-sector
//             stores make rank 0's ingest request-rate bound.  A block that stops being tracked before all its rays have
//             finished is sent partially (masked lanes) and its stragglers fall back to the direct store.  (The staging
//             buffer is in global memory: two 1 KB slots per warp in shared memory would take 8 KB of L1 per CTA.)
//
// FILTER (K == 1 closest hit, host-pointer entry points only): the host side of filter callbacks (rtcore_shim.cpp
// trace_filtered).  Every ray carries a list of record indices that a callback has already rejected
// (p.excl_idx[p.excl_off[i] .. p.excl_off[i+1])); those records are skipped, and the winning record's index goes to p.win[i]
// so that the host can extend the list when the callback rejects this hit as well.
//
// INST (instance traversal, GENERAL >= 1): the top level's instance records (b.w == kInstRecord) are entered instead of tested.  The
// lane checks the instance mask, pushes what is left of its node group and of its leaf group, then an exit marker (y == 0), takes
// the ray into object space with the instance's w2l (to_object_space: the records see the ray flattening gives them), recomputes
// 1/dir and the octant, and continues at the instanced scene's root.  Popping the marker reloads the world ray from the ray buffer;
// t is shared by both spaces, so the hit distance carries over.  The entries under the marker were pushed in world space and are
// decoded with the world octant again.  A leaf group on the stack has no pending-child bits (y & 0xFF000000 == 0, y != 0).
template <int K, bool OCCLUDED, bool STATS, bool ROBUST, int GENERAL, int GATHER = 0, bool SPREAD = false, bool FILTER = false, bool INST = false>
__global__ void __launch_bounds__(TRACE_THREADS, RTK_MIN_BLOCKS) trace_kernel(const TraceParams p) {
  const bool USE_TMA = p.use_prefetch != 0;
  using IO = RayIO<K, OCCLUDED>;
  const unsigned FULL = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31;
  const unsigned lt_mask = (1u << lane) - 1u;
  const uint32_t warp_id = blockIdx.x * TRACE_WARPS + (threadIdx.x >> 5);
  const uint32_t num_warps = gridDim.x * TRACE_WARPS;
  const uint32_t n = (uint32_t)p.n;
  const Node8* __restrict__ nodes = p.nodes;
  const uint4* __restrict__ tris = reinterpret_cast<const uint4*>(p.tris);
  const int tri_batch_min = p.tri_batch_min, tri_wait_max = p.tri_wait_max, refill_min = p.refill_min;

  // per-lane ray state
  enum : uint32_t { EMPTY = 0, TRACING = 1, DONE = 2 };
  uint32_t state = EMPTY;
  Ray r;
  float idx = 0, idy = 0, idz = 0, tfar_tri = 0;
  uint32_t oct = 0;
  // closest hit so far: t = tfar_tri (register), barycentrics and the winning record's index; the ray's index in the stream.
  // These four are written on a hit / at refill and read at write-back only: with 64 registers per thread they are
  // better placed in shared memory ([field][thread], conflict-free) than left to the register allocator, which spills
  // other values inside the node step otherwise.
  // GENERAL == 2 (curve scenes): 9-11 the normal of a curve hit -- the round cubic test is an iteration whose result depends on
  // the tfar it was started with, so the normal is kept from the winning test instead of re-running the test at write-back
  // INST: two more, the instance the lane is in (kInvalidID: none) and that of the winning record
  __shared__ uint32_t s_lane[(GENERAL == 2 ? 12 : 9) + (INST ? 2 : 0)][TRACE_THREADS];   // 0 u, 1 v, 2 winning record, 3 ray index, 4-6 ray direction, 7 ray mask, 8 the ray's own tfar
#define hit_u (reinterpret_cast<float*>(s_lane[0])[threadIdx.x])
#define hit_v (reinterpret_cast<float*>(s_lane[1])[threadIdx.x])
#define hit_tri (s_lane[2][threadIdx.x])
#define ray_index (s_lane[3][threadIdx.x])
#define CURVE_NG(k) (s_lane[GENERAL == 2 ? 9 + (k) : 0][threadIdx.x])
#define CUR_INST (s_lane[INST ? (GENERAL == 2 ? 12 : 9) : 0][threadIdx.x])
#define HIT_INST (s_lane[INST ? (GENERAL == 2 ? 13 : 10) : 0][threadIdx.x])
  // The ray's direction, mask and original tfar are only needed by triangle / curve tests: the node step works with
  // org, 1/dir, tnear and the current hit distance.  They are parked in shared memory too (read by the SPREAD workers by
  // owner index -- instead of five shuffles -- and by the non-SPREAD test of the lane itself).
#define RAY_DX(t) (reinterpret_cast<float*>(s_lane[4])[t])
#define RAY_DY(t) (reinterpret_cast<float*>(s_lane[5])[t])
#define RAY_DZ(t) (reinterpret_cast<float*>(s_lane[6])[t])
#define RAY_MASK(t) (s_lane[7][t])
#define RAY_TFAR(t) (reinterpret_cast<float*>(s_lane[8])[t])
  // this lane's ray with the parked fields filled in (non-SPREAD triangle / curve tests, ROBUST write-back)
  auto full_ray = [&]() -> Ray {
    Ray q = r;
    q.dx = RAY_DX(threadIdx.x); q.dy = RAY_DY(threadIdx.x); q.dz = RAY_DZ(threadIdx.x);
    q.mask = RAY_MASK(threadIdx.x); q.tfar = RAY_TFAR(threadIdx.x);
    return q;
  };
  auto curve_normal = [&]() -> float3 { return make_float3(__uint_as_float(CURVE_NG(0)), __uint_as_float(CURVE_NG(1)), __uint_as_float(CURVE_NG(2))); };
  bool found = false;
  uint32_t ngx = 0, ngy = 0, tgx = 0, tgy = 0;
  uint32_t top_x = 0, top_y = 0;          // register copy of the newest stack entry (top_y == 0: none)
  // older entries: the first RTK_SMEM_STACK per lane in shared memory ([entry][thread]: conflict-free 8-byte accesses),
  // deeper ones in local memory.  A stack wholly in local memory competes with the streaming node / triangle data for L1,
  // a pop that misses costs an L2 round trip, and every push is written through to L2.
  __shared__ uint2 s_stack[RTK_SMEM_STACK > 0 ? RTK_SMEM_STACK * TRACE_THREADS : 1];
  uint2 stack[kStackSize];
  int sp = 0;
  auto push_entry = [&](uint32_t x, uint32_t y) {
    if (sp < RTK_SMEM_STACK) s_stack[sp * TRACE_THREADS + threadIdx.x] = make_uint2(x, y);
    else stack[sp - RTK_SMEM_STACK] = make_uint2(x, y);
    ++sp;
  };
  auto pop_entry = [&]() -> uint2 {
    --sp;
    return sp < RTK_SMEM_STACK ? s_stack[sp * TRACE_THREADS + threadIdx.x] : stack[sp - RTK_SMEM_STACK];
  };
  // warp-uniform block cursor
  int blk = -1;                           // index into this warp's block sequence
  uint32_t blk_first = 0, blk_count = 0, consumed = 0;
  bool warp_done = false;
  int tri_wait = 0;
  unsigned long long st_rays = 0, st_nodes = 0, st_tris = 0;
  // GATHER 2: the two newest blocks of this warp are tracked; slot_blk = index (in this warp's block sequence), slot_have =
  // which of its 32 records have been written to the local staging buffer (warp-uniform values)
  // The state lives in shared memory (16 B per warp: first ray index and arrival mask of the two tracked blocks), not in
  // registers: it is only touched in the write-back phase, and four more live registers in the traversal loop spill in the
  // node step.
  __shared__ uint32_t s_slot[GATHER == 2 ? TRACE_WARPS : 1][4];   // first0, have0, first1, have1; first == ~0u: free
  constexpr uint32_t kNoBlock = 0xFFFFFFFFu;
  if (GATHER == 2) {
    if (lane < 4) s_slot[threadIdx.x >> 5][lane] = (lane & 1) ? 0u : kNoBlock;
    __syncwarp();
  }

  auto block_first = [&](int b) -> unsigned long long { return ((unsigned long long)b * num_warps + warp_id) * 32ull; };
  auto prefetch = [&](int b) {   // lane 0 only
    const unsigned long long first = block_first(b);
    if (first >= n) return;
    const uint32_t cnt = (n - first) < 32u ? (uint32_t)(n - first) : 32u;
    tma_prefetch_l2(static_cast<const char*>(p.rays) + first * IO::kRayBytes, cnt * IO::kRayBytes);
  };
  if (USE_TMA && lane == 0) { prefetch(0); prefetch(1); }

  // hit epilogue of one terminated ray (intersector_epilog.h:285-299; occluded: bvh_intersector1.cpp:186-188)
  // `rec_dst`: where the compact 32-byte record goes (GATHER), chosen by the caller
  auto write_back = [&](void* rec_dst) {
    float cngx = 0.0f, cngy = 0.0f, cngz = 0.0f;
    uint32_t cprim = kInvalidID, cgeom = kInvalidID;
    if (found) {
      if (OCCLUDED) IO::store_tfar(p, ray_index, -INFINITY);
      else {   // Ng and the ids come from the winning record, re-read here
        Hit hit;
        uint32_t instID = p.instID, instPrimID = p.instPrimID;
        if constexpr (INST) {
          // a record hit inside an instance reports the instance's ids, and ROBUST's Ng takes the object-space origin
          const uint32_t hi = HIT_INST;
          auto hit_ray = [&]() -> Ray { Ray q = full_ray(); if (hi != kInvalidID) to_object_space(p.insts[hi], q); return q; };
          record_write_back<ROBUST, GENERAL>(tris, p.descs, hit_tri, hit_ray, curve_normal, hit_u, hit_v, hit, instID, instPrimID);
          if (hi != kInvalidID) { instID = p.insts[hi].instID; instPrimID = 0u; }   // instance_id_stack::push(context, instID, 0)
        } else {
          record_write_back<ROBUST, GENERAL>(tris, p.descs, hit_tri, full_ray, curve_normal, hit_u, hit_v, hit, instID, instPrimID);
        }
        hit.t = tfar_tri;
        IO::store_hit(p, ray_index, hit, instID, instPrimID);
        cngx = hit.ngx; cngy = hit.ngy; cngz = hit.ngz; cprim = hit.primID; cgeom = hit.geomID;
      }
    }
    if (FILTER) p.win[ray_index] = found ? hit_tri : kInvalidID;
    if (GATHER)   // a full 32-byte sector; a miss (also: empty scene) yields {tfar, 0.., -1, -1}
      store_256(rec_dst, tfar_tri, cngx, cngy, cngz, found ? hit_u : 0.0f, found ? hit_v : 0.0f, __uint_as_float(cprim), __uint_as_float(cgeom));
  };
  // GATHER 2: send the arrived records of a tracked block from the staging buffer to the gather buffer, lane i = record i
  auto flush_block = [&](uint32_t first, unsigned have) {
    __syncwarp();                    // the records were stored by other lanes of this warp: order them before the re-read
    __threadfence_block();
    if (have & (1u << lane)) {
      const size_t off = (size_t)(first + lane) * 32;
      const float4* src = reinterpret_cast<const float4*>(static_cast<const char*>(p.stage) + off);
      const float4 x = __ldcg(src), y = __ldcg(src + 1);       // L2 (the stores went through L1 write-through)
      store_256(static_cast<char*>(p.compact_out) + off, x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w);
    }
  };

  // one triangle record against this lane's ray (closest hit: shrinks tfar_tri; any hit: terminates the ray)
  auto test_tri = [&](uint32_t ti, const uint4& a, const uint4& b, const uint4& c) {
    if (FILTER) {   // a record the filter callback has rejected for this ray is no candidate any more
      const uint32_t e0 = p.excl_off[ray_index], e1 = p.excl_off[ray_index + 1];
      for (uint32_t e = e0; e < e1; ++e)
        if (p.excl_idx[e] == ti) return;
    }
    record_test<ROBUST, GENERAL, !OCCLUDED, false>(p.descs, a, b, c, full_ray(), tfar_tri, hit_u, hit_v, [&](const RecordHit& h) {
      found = true;
      if (OCCLUDED) { ngy = 0; tgy = 0; sp = 0; top_y = 0; }     // any hit terminates the ray
      else {
        tfar_tri = h.t; hit_tri = ti;
        if constexpr (INST) HIT_INST = CUR_INST;
        if (GENERAL == 2 && h.curve) { CURVE_NG(0) = __float_as_uint(h.ngx); CURVE_NG(1) = __float_as_uint(h.ngy); CURVE_NG(2) = __float_as_uint(h.ngz); }
      }
    });
  };

  for (;;) {
    // ---- 1. write back finished rays and refill, in batches: this code runs for the whole warp, so wait until a few
    // lanes have nothing to trace (or none has)
    const unsigned idle = __ballot_sync(FULL, state != TRACING);
    if (idle && (__popc(idle) >= refill_min || idle == FULL)) {
      // (Issuing the record fetches of the write-back together with the ray fetches of the refill -- one latency instead
      // of two -- is not done: the extra live registers spill in the node step.)
      const bool has_rec = state == DONE;
      int slot = -1;
      uint32_t first0 = 0, first1 = 0;
      uint32_t* ss = s_slot[GATHER == 2 ? (threadIdx.x >> 5) : 0];
      if (GATHER == 2) {
        first0 = ss[0]; first1 = ss[2];
        const uint32_t my_first = ray_index & ~31u;
        slot = !has_rec ? -1 : (my_first == first0 ? 0 : (my_first == first1 ? 1 : -1));
      }
      if (has_rec) {
        // GATHER 1: straight to the gather buffer.  GATHER 2: records of a tracked block go to the local staging buffer,
        // stragglers of a block that is no longer tracked straight to the gather buffer.
        char* dst = GATHER ? static_cast<char*>((GATHER == 2 && slot >= 0) ? p.stage : p.compact_out) + (size_t)ray_index * 32 : nullptr;
        write_back(dst);
        state = EMPTY;
      }
      if (GATHER == 2) {
        const unsigned have0 = ss[1] | __reduce_or_sync(FULL, slot == 0 ? 1u << (ray_index & 31u) : 0u);
        const unsigned have1 = ss[3] | __reduce_or_sync(FULL, slot == 1 ? 1u << (ray_index & 31u) : 0u);
        auto full_mask = [&](uint32_t first) -> unsigned { return (n - first) >= 32u ? 0xFFFFFFFFu : ((1u << (n - first)) - 1u); };
        const bool done0 = first0 != kNoBlock && have0 == full_mask(first0), done1 = first1 != kNoBlock && have1 == full_mask(first1);
        if (done0) flush_block(first0, have0);
        if (done1) flush_block(first1, have1);
        __syncwarp();
        if (lane == 0) { ss[0] = done0 ? kNoBlock : first0; ss[1] = done0 ? 0u : have0; ss[2] = done1 ? kNoBlock : first1; ss[3] = done1 ? 0u : have1; }
        __syncwarp();
      }
      if (!warp_done) {
        if (consumed == blk_count) {       // resident block used up (or nothing loaded yet): move to the next one
          if (USE_TMA && lane == 0) prefetch(blk + 3);   // keep the stream two blocks ahead in L2
          ++blk;
          const unsigned long long first = block_first(blk);
          if (first >= n) { warp_done = true; blk_count = 0; consumed = 0; }
          else {
            blk_first = (uint32_t)first;
            blk_count = (n - blk_first) < 32u ? (n - blk_first) : 32u;
            consumed = 0;
            if (GATHER == 2) {   // the new block becomes tracked: in a free slot, else the older block is sent as far as it got
              uint32_t* ss = s_slot[threadIdx.x >> 5];
              const uint32_t f0 = ss[0], h0 = ss[1], f1 = ss[2], h1 = ss[3];
              int use = f0 == kNoBlock ? 0 : (f1 == kNoBlock ? 1 : (f0 < f1 ? 0 : 1));
              if (f0 != kNoBlock && f1 != kNoBlock) flush_block(use == 0 ? f0 : f1, use == 0 ? h0 : h1);
              __syncwarp();
              if (lane == 0) { ss[2 * use] = blk_first; ss[2 * use + 1] = 0u; }
              __syncwarp();
            }
          }
        }
        if (!warp_done) {
          const uint32_t avail = blk_count - consumed;
          const uint32_t rank = __popc(idle & lt_mask);
          if (state == EMPTY && rank < avail) {
            ray_index = blk_first + consumed + rank;
            bool valid = true;
            if (K > 1) valid = (p.valid == nullptr) || (p.valid[ray_index] == -1);   // inactive lanes stay untouched
            if (valid) {
              IO::load(static_cast<const char*>(p.rays), ray_index, r);
              if (STATS) ++st_rays;
              found = false;
              sp = 0; top_y = 0; tgx = 0; tgy = 0;
              if constexpr (INST) { CUR_INST = kInvalidID; HIT_INST = kInvalidID; }
              // empty scene / already occluded rays terminate at once (bvh_intersector1.cpp:39,128-129); they still
              // pass through DONE so that a gather buffer receives their miss record
              const bool go = p.root_valid && !(OCCLUDED && r.tfar < 0.0f);
              RAY_DX(threadIdx.x) = r.dx; RAY_DY(threadIdx.x) = r.dy; RAY_DZ(threadIdx.x) = r.dz;
              RAY_MASK(threadIdx.x) = r.mask; RAY_TFAR(threadIdx.x) = r.tfar;
              idx = rcp_safe_fast(r.dx); idy = rcp_safe_fast(r.dy); idz = rcp_safe_fast(r.dz);
              oct = (idx < 0.0f ? 1u : 0u) | (idy < 0.0f ? 2u : 0u) | (idz < 0.0f ? 4u : 0u);
              tfar_tri = r.tfar;
              ngx = 0; ngy = go ? 0x80000000u : 0u;   // root entered as "one pending internal child, imask 0"
              state = go ? TRACING : DONE;
            }
          }
          const uint32_t want = __popc(idle);
          consumed += want < avail ? want : avail;
        }
      }
      if (!__any_sync(FULL, state == TRACING)) {
        if (warp_done && !__any_sync(FULL, state == DONE)) break;
        continue;
      }
    }
    const bool tracing = state == TRACING;
    // ---- 2. node step for lanes that have no triangle pending and a node child pending
    if (tracing && tgy == 0 && (ngy & 0xFF000000u)) {
      const int bit = 31 - __clz((int)ngy);
      ngy &= ~(1u << bit);
      if (ngy & 0xFF000000u) {           // push the rest of the group
        if (top_y) push_entry(top_x, top_y);
        top_x = ngx; top_y = ngy;
      }
      const uint32_t slot = ((uint32_t)(bit - 24)) ^ (7u - oct);
      const uint32_t node_index = ngx + (uint32_t)__popc(ngy & 0xFFu & ((1u << slot) - 1u));
      NodeW nw;
      load_node(nodes, node_index, nw);
      if (STATS) ++st_nodes;
      // TravRay clamps tnear/tfar at 0 for the slab test only (bvh_intersector1.cpp:65); after a hit tray.tfar = ray.tfar (:105)
      const uint32_t hm = node_hitmask(nw.w, r.ox, r.oy, r.oz, idx, idy, idz, (oct & 1u) != 0, (oct & 2u) != 0, (oct & 4u) != 0,
                                       fmaxf(r.tnear, 0.0f), fmaxf(tfar_tri, 0.0f), 7u - oct);
      ngx = nw.w[4];
      ngy = (hm & 0xFF000000u) | (nw.w[3] >> 24);
      tgx = nw.w[5];
      tgy = hm & 0x00FFFFFFu;
    }
    // ---- 3. triangle step, batched across the warp
    const unsigned tri_lanes = __ballot_sync(FULL, tracing && tgy != 0);
    const unsigned node_lanes = __ballot_sync(FULL, tracing && tgy == 0 && (ngy & 0xFF000000u));
    if (tri_lanes && (__popc(tri_lanes) >= tri_batch_min || node_lanes == 0 || ++tri_wait >= tri_wait_max)) {
      tri_wait = 0;
      if (SPREAD) {
        // Closest-hit Moeller-Trumbore triangle scenes (rtcb200SetTuning "tri_spread" 0 turns it off): the pending
        // triangles of ALL lanes become work items that the whole warp tests in one step, instead of each lane testing
        // one of its own while the others idle: on the headline stream about half as many triangle steps, each with about
        // twice as many busy lanes.  Owners queue (record index, owner lane) in shared memory; worker lane w takes item w, fetches the
        // owner's ray by shuffles and tests the record; hits meet in a 64-bit atomicMin per owner keyed by (t, item) --
        // among equal t (-0 and +0 included) the later item wins, as in the sequential order -- and the owner reads t, u, v
        // back by shuffle.
        __shared__ uint32_t s_tri[TRACE_WARPS][32];
        __shared__ uint32_t s_owner[TRACE_WARPS][32];
        __shared__ unsigned long long s_best[TRACE_WARPS][32];
        const int wi = threadIdx.x >> 5;
        const bool isT = tracing && tgy != 0;
        const int cnt = isT ? __popc(tgy) : 0;
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
        int slot = incl - cnt;                                  // first queue slot of this lane's items
        const int total = min(__shfl_sync(FULL, incl, 31), 32);
        s_best[wi][lane] = ~0ull;
        while (isT && tgy != 0 && slot < 32) {                  // highest bit first = the sequential test order
          const int tb = 31 - __clz((int)tgy);
          tgy &= ~(1u << tb);
          s_tri[wi][slot] = tgx + (uint32_t)tb;
          s_owner[wi][slot] = (uint32_t)lane;
          ++slot;
        }
        __syncwarp();
        const bool work = lane < total;
        const uint32_t ti = work ? s_tri[wi][lane] : 0u;
        const int owner = work ? (int)s_owner[wi][lane] : lane;
        Ray lr;
        lr.ox = __shfl_sync(FULL, r.ox, owner); lr.oy = __shfl_sync(FULL, r.oy, owner); lr.oz = __shfl_sync(FULL, r.oz, owner);
        const int ot = (threadIdx.x & ~31) + owner;             // the owner's slot of the parked ray fields
        lr.dx = RAY_DX(ot); lr.dy = RAY_DY(ot); lr.dz = RAY_DZ(ot);
        lr.tnear = __shfl_sync(FULL, r.tnear, owner);
        // The winner must not depend on which other rays share the warp (an owner's items may be split over two steps
        // when the queue is full): a triangle is a candidate when it passes the test against the ray's ORIGINAL tfar and
        // its final t is <= the owner's current hit distance; among candidates the smallest t wins, the later item on
        // equal t.  This is the minimum over all tested triangles whatever the batching, so the batched entry points,
        // the packet entry points and the host-pointer pipeline return bit-identical hits for the same ray.  This is
        // spread_record_test (record_tests.cuh), written out: called from here it changes this kernel's code and cost 0.3 %
        // on the headline stream (1346.6 against 1351.1 Mrays/s, four alternating runs, H100 80GB HBM3 at 700 W).
        const float o_tfar = RAY_TFAR(ot);
        const float o_best = __shfl_sync(FULL, tfar_tri, owner);
        const uint32_t o_mask = RAY_MASK(ot);
        float w_t = 0.0f, w_u = 0.0f, w_v = 0.0f;
        unsigned long long key = ~0ull;
        if (work) {
          const uint4* tp = tris + (size_t)ti * 3;
          const uint4 a = __ldg(tp), b = __ldg(tp + 1), c = __ldg(tp + 2);
          if (STATS) ++st_tris;
          TriHit th;
          if ((c.w & o_mask) != 0 &&
              tri_test(lr, o_tfar, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(b.x),
                       __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(c.x), __uint_as_float(c.y), __uint_as_float(c.z), th)) {
            if (OCCLUDED) {   // any hit: one accepted triangle terminates the owner's ray (bvh_intersector1.cpp:186-188)
              s_best[wi][owner] = 0ull;
            } else {
            const float rcpAbsDen = 1.0f / th.absDen;
            const float t = th.T * rcpAbsDen;
            if (t <= o_best) {
              w_t = t; w_u = th.U * rcpAbsDen; w_v = th.V * rcpAbsDen;
              // t <= best holds between -0 and +0 both ways, so the two zeros must share a key for the later item to win: the
              // key is made from t + 0 (-0 + 0 = +0), and the winner's own t, sign included, comes from its lane below
              uint32_t tb32 = __float_as_uint(__fadd_rn(t, 0.0f));
              tb32 ^= (tb32 >> 31) ? 0xFFFFFFFFu : 0x80000000u;   // order-preserving float -> uint
              key = ((unsigned long long)tb32 << 32) | (uint32_t)(31 - lane);
              atomicMin(&s_best[wi][owner], key);
            }
            }
          }
        }
        __syncwarp();
        const unsigned long long best = s_best[wi][lane];       // as owner
        const bool got = isT && best != ~0ull;
        const int win = got ? 31 - (int)(best & 31ull) : lane;  // worker lane that holds the winning item
        const float b_t = __shfl_sync(FULL, w_t, win), b_u = __shfl_sync(FULL, w_u, win), b_v = __shfl_sync(FULL, w_v, win);
        if (got && OCCLUDED) { found = true; ngy = 0; tgy = 0; sp = 0; top_y = 0; }
        else if (got) {
          tfar_tri = b_t;
          hit_u = b_u; hit_v = b_v; hit_tri = s_tri[wi][win];
          found = true;
        }
        __syncwarp();                                           // the queue is reused by the next triangle step
      } else if (tracing && tgy != 0) {
        const int tb = 31 - __clz((int)tgy);
        tgy &= ~(1u << tb);
        const uint32_t ti = tgx + (uint32_t)tb;
        const uint4* tp = tris + (size_t)ti * 3;
        const uint4 a = __ldg(tp), b = __ldg(tp + 1), c = __ldg(tp + 2);
        if (STATS) ++st_tris;
        if constexpr (INST) {
          // an instance record (instance index in a.w, its mask in c.w): enter the instance instead of testing a record.  What is
          // left of the node and leaf groups goes on the stack, then the exit marker.
          if (b.w == kInstRecord) {
            if ((c.w & RAY_MASK(threadIdx.x)) != 0) {   // instance_intersector.cpp:19-22
              const InstRec& ir = p.insts[a.w];
              if (top_y) push_entry(top_x, top_y);
              top_y = 0;
              if (ngy & 0xFF000000u) push_entry(ngx, ngy);
              if (tgy) push_entry(tgx, tgy);
              push_entry(0u, 0u);
              Ray q = full_ray();
              to_object_space(ir, q);
              r.ox = q.ox; r.oy = q.oy; r.oz = q.oz;
              RAY_DX(threadIdx.x) = q.dx; RAY_DY(threadIdx.x) = q.dy; RAY_DZ(threadIdx.x) = q.dz;
              idx = rcp_safe_fast(q.dx); idy = rcp_safe_fast(q.dy); idz = rcp_safe_fast(q.dz);
              oct = (idx < 0.0f ? 1u : 0u) | (idy < 0.0f ? 2u : 0u) | (idz < 0.0f ? 4u : 0u);
              CUR_INST = a.w;
              ngx = __ldg(&ir.child_root); ngy = 0x80000000u;   // the instanced scene's root, entered like the scene root at refill
              tgy = 0;
            }
          } else {
            test_tri(ti, a, b, c);   // one record per step: a second one could be an instance
          }
        } else if (RTK_TRI2) {
          // a second pending triangle of the same lane rides along: its record is fetched together with the first
          // (one latency instead of two) and tested after it, against the tfar the first one left -- the sequential order
          const bool two = tgy != 0;
          const int tb2 = two ? 31 - __clz((int)tgy) : tb;
          const uint32_t ti2 = tgx + (uint32_t)tb2;
          const uint4* tp2 = tris + (size_t)ti2 * 3;
          uint4 a2, b2, c2;
          if (two) { a2 = __ldg(tp2); b2 = __ldg(tp2 + 1); c2 = __ldg(tp2 + 2); }
          test_tri(ti, a, b, c);
          if (two && tgy != 0) {          // (any hit: the first test may have terminated the ray and cleared tgy)
            tgy &= ~(1u << tb2);
            if (STATS) ++st_tris;
            test_tri(ti2, a2, b2, c2);
          }
        } else {
          test_tri(ti, a, b, c);
        }
      }
    }
    // ---- 4. pop or finish
    if (tracing && tgy == 0 && (ngy & 0xFF000000u) == 0) {
      if (top_y) { ngx = top_x; ngy = top_y; top_y = 0; }
      else if (sp > 0) {
        const uint2 e = pop_entry();
        ngx = e.x; ngy = e.y;
        if constexpr (INST) {
          if ((e.y & 0xFF000000u) == 0) {   // a leaf group, or the exit marker of an instance
            ngy = 0;
            if (e.y) { tgx = e.x; tgy = e.y; }
            else {   // back in world space: the ray from the ray buffer, its reciprocal and octant as the refill set them up
              IO::load(static_cast<const char*>(p.rays), ray_index, r);
              RAY_DX(threadIdx.x) = r.dx; RAY_DY(threadIdx.x) = r.dy; RAY_DZ(threadIdx.x) = r.dz;
              idx = rcp_safe_fast(r.dx); idy = rcp_safe_fast(r.dy); idz = rcp_safe_fast(r.dz);
              oct = (idx < 0.0f ? 1u : 0u) | (idy < 0.0f ? 2u : 0u) | (idz < 0.0f ? 4u : 0u);
              CUR_INST = kInvalidID;
            }
          }
        }
      }
      else state = DONE;
    }
  }
  if (GATHER == 2) {   // every block is complete by now and has left; this only covers a block that never filled
    const uint32_t* ss = s_slot[threadIdx.x >> 5];
    if (ss[0] != kNoBlock && ss[1]) flush_block(ss[0], ss[1]);
    if (ss[2] != kNoBlock && ss[3]) flush_block(ss[2], ss[3]);
  }
  if (STATS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      st_rays += __shfl_xor_sync(FULL, st_rays, o);
      st_nodes += __shfl_xor_sync(FULL, st_nodes, o);
      st_tris += __shfl_xor_sync(FULL, st_tris, o);
    }
    if (lane == 0) { atomicAdd(&p.stat[0], st_rays); atomicAdd(&p.stat[1], st_nodes); atomicAdd(&p.stat[2], st_tris); }
  }
}

#undef hit_u
#undef hit_v
#undef hit_tri
#undef ray_index
#undef CURVE_NG
#undef CUR_INST
#undef HIT_INST
#undef RAY_DX
#undef RAY_DY
#undef RAY_DZ
#undef RAY_MASK
#undef RAY_TFAR

static int g_num_sms = 0;
static Tuning g_tuning;
Tuning& tuning() { return g_tuning; }

template <int K, bool OCCLUDED>
static int launch_k(TraceParams p, cudaStream_t st) {
  if (p.n == 0) return 0;
  if (p.n > 0x40000000ull) {   // the kernel indexes rays with 32 bits: longer streams run as consecutive 2^30-ray launches
    const unsigned long long chunk = 0x40000000ull;   // a multiple of every packet width and of the 32-ray block
    for (unsigned long long first = 0; first < p.n; first += chunk) {
      TraceParams q = p;
      q.n = (p.n - first) < chunk ? (p.n - first) : chunk;
      q.rays = static_cast<char*>(p.rays) + first * RayIO<K, OCCLUDED>::kRayBytes;
      if (p.valid) q.valid = p.valid + first;
      if (p.compact_out) q.compact_out = static_cast<char*>(p.compact_out) + first * 32;
      if (p.stage) q.stage = static_cast<char*>(p.stage) + first * 32;
      const int r = launch_k<K, OCCLUDED>(q, st);
      if (r != 0) return r;
    }
    return 0;
  }
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  p.tri_batch_min = p.curves == 2 ? g_tuning.curve_batch_min : p.curves ? g_tuning.point_batch_min : g_tuning.tri_batch_min;
  p.tri_wait_max = p.curves == 2 ? g_tuning.curve_wait_max : p.curves ? g_tuning.point_wait_max : g_tuning.tri_wait_max;
  p.refill_min = g_tuning.refill_min;
  // persistent grid: a multiple of the SM count, capped by the work available
  const unsigned long long need = (p.n + TRACE_THREADS - 1) / TRACE_THREADS;
  const unsigned long long cap = (unsigned long long)g_num_sms * (p.curves == 2 ? g_tuning.curve_blocks_per_sm : g_tuning.blocks_per_sm);
  const unsigned blocks = (unsigned)(need < cap ? need : cap);
  // tiny launches (single-record API calls read a mapped pinned host record) skip the bulk prefetch
  p.use_prefetch = (p.n >= 1024 && g_tuning.use_tma) ? 1 : 0;
  // kernel variant: bit 0 GENERAL (instances / quads), bit 1 ROBUST, bit 2 STATS; closest-hit Moeller-Trumbore triangle
  // scenes (no bit 0 / 1) run the SPREAD instantiation -- the pending triangles of all lanes are tested by the whole warp
  constexpr bool CLOSEST = !OCCLUDED;
  constexpr bool CAN_GATHER = (K == 1 && CLOSEST);
  const int variant = (p.stat ? 4 : 0) | (p.robust ? 2 : 0) | (p.descs ? 1 : 0);
  const int g = general_of(p.descs, p.curves);
  if (p.excl_off) {   // filter-callback passes (rtcore_shim.cpp trace_filtered): K == 1 closest hit, no gather, no statistics
    if (!(K == 1 && CLOSEST) || !p.excl_idx || !p.win || p.insts) return (int)cudaErrorInvalidValue;
    constexpr bool FI = (K == 1 && CLOSEST);   // only these instantiations carry the exclusion code
    switch (g * 2 + (p.robust ? 1 : 0)) {
#define RTK_FILTER(RB, GE) trace_kernel<K, OCCLUDED, false, RB, GE, 0, false, FI><<<blocks, TRACE_THREADS, 0, st>>>(p); break
      case 0: RTK_FILTER(false, 0);
      case 1: RTK_FILTER(true, 0);
      case 2: RTK_FILTER(false, 1);
      case 3: RTK_FILTER(true, 1);
      case 4: RTK_FILTER(false, 2);
      case 5: RTK_FILTER(true, 2);
#undef RTK_FILTER
    }
    count_launch();
    return (int)cudaGetLastError();
  }
  if (p.insts) {   // instance traversal: the INST instantiations, GENERAL 1 or 2
    const int gmode = (CAN_GATHER && p.compact_out) ? ((g_tuning.gather_mode == 0 || !p.stage) ? 1 : 2) : 0;
    switch ((variant >> 1) + 4 * gmode + (g == 2 ? 12 : 0)) {
#define RTK_INST(ST, RB, GE, GA) trace_kernel<K, OCCLUDED, ST, RB, GE, (CAN_GATHER ? GA : 0), false, false, true><<<blocks, TRACE_THREADS, 0, st>>>(p); break
#define RTK_INST4(GE, GA)                                              \
      case (GE == 2 ? 12 : 0) + 4 * GA + 0: RTK_INST(false, false, GE, GA); \
      case (GE == 2 ? 12 : 0) + 4 * GA + 1: RTK_INST(false, true, GE, GA);  \
      case (GE == 2 ? 12 : 0) + 4 * GA + 2: RTK_INST(true, false, GE, GA);  \
      case (GE == 2 ? 12 : 0) + 4 * GA + 3: RTK_INST(true, true, GE, GA);
      RTK_INST4(1, 0)
      RTK_INST4(1, 1)
      RTK_INST4(1, 2)
      RTK_INST4(2, 0)
      RTK_INST4(2, 1)
      RTK_INST4(2, 2)
#undef RTK_INST4
#undef RTK_INST
    }
    count_launch();
    return (int)cudaGetLastError();
  }
  if (g == 2) {   // scenes with curve or point records: the GENERAL = 2 instantiations
    const int gmode = (CAN_GATHER && p.compact_out) ? ((g_tuning.gather_mode == 0 || !p.stage) ? 1 : 2) : 0;
    switch ((variant >> 1) + 4 * gmode) {
#define RTK_CURVE(ST, RB, GA) trace_kernel<K, OCCLUDED, ST, RB, 2, (CAN_GATHER ? GA : 0), false><<<blocks, TRACE_THREADS, 0, st>>>(p); break
#define RTK_CURVE4(GA)                         \
      case 4 * GA + 0: RTK_CURVE(false, false, GA); \
      case 4 * GA + 1: RTK_CURVE(false, true, GA);  \
      case 4 * GA + 2: RTK_CURVE(true, false, GA);  \
      case 4 * GA + 3: RTK_CURVE(true, true, GA);
      RTK_CURVE4(0)
      RTK_CURVE4(1)
      RTK_CURVE4(2)
#undef RTK_CURVE4
#undef RTK_CURVE
    }
    count_launch();
    return (int)cudaGetLastError();
  }
  const int gather = (CAN_GATHER && p.compact_out) ? ((g_tuning.gather_mode == 0 || !p.stage) ? 1 : 2) : 0;
  const bool spread = (CLOSEST ? g_tuning.tri_spread : g_tuning.tri_spread_occluded) && !p.robust && !p.descs;
  switch (variant + 8 * gather + (spread ? 32 : 0)) {
#define RTK_LAUNCH(ST, RB, IN, GA, SP) trace_kernel<K, OCCLUDED, ST, RB, (IN ? 1 : 0), (CAN_GATHER ? GA : 0), SP><<<blocks, TRACE_THREADS, 0, st>>>(p); break
#define RTK_LAUNCH8(GA)                                          \
    case 8 * GA + 0: RTK_LAUNCH(false, false, false, GA, false); \
    case 8 * GA + 1: RTK_LAUNCH(false, false, true, GA, false);  \
    case 8 * GA + 2: RTK_LAUNCH(false, true, false, GA, false);  \
    case 8 * GA + 3: RTK_LAUNCH(false, true, true, GA, false);   \
    case 8 * GA + 4: RTK_LAUNCH(true, false, false, GA, false);  \
    case 8 * GA + 5: RTK_LAUNCH(true, false, true, GA, false);   \
    case 8 * GA + 6: RTK_LAUNCH(true, true, false, GA, false);   \
    case 8 * GA + 7: RTK_LAUNCH(true, true, true, GA, false);    \
    case 32 + 8 * GA + 0: RTK_LAUNCH(false, false, false, GA, true); \
    case 32 + 8 * GA + 4: RTK_LAUNCH(true, false, false, GA, true);
    RTK_LAUNCH8(0)
    RTK_LAUNCH8(1)
    RTK_LAUNCH8(2)
#undef RTK_LAUNCH8
#undef RTK_LAUNCH
  }
  count_launch();
  return (int)cudaGetLastError();
}

int launch_trace(const TraceParams& p, int occluded, int K, cudaStream_t st) {
  switch (K) {
    case 1: return occluded ? launch_k<1, true>(p, st) : launch_k<1, false>(p, st);
    case 4: return occluded ? launch_k<4, true>(p, st) : launch_k<4, false>(p, st);
    case 8: return occluded ? launch_k<8, true>(p, st) : launch_k<8, false>(p, st);
    case 16: return occluded ? launch_k<16, true>(p, st) : launch_k<16, false>(p, st);
  }
  return (int)cudaErrorInvalidValue;
}

}  // namespace rtk
