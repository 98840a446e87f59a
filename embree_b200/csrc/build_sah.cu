// build_sah.cu -- top-down binned-SAH construction of the binary build tree, device-wide, level by level.
//
// Replaces kernels/builders/bvh_builder_sah.h:216-313 (recurse), heuristic_binning.h:17-110 (BinMapping),
// :210-260 (bin), :339-393 (best) and heuristic_binning_array_aligned.h:137-172 (partition), which the reference
// runs as a task recursion with parallel binning above 3072 primitives.  Here every tree level is a handful of
// launches over a work list of segments ("tasks") of the Morton-sorted primitive array:
//   * LARGE segments (> kBlockCap prims): many CTAs per segment -- per-CTA shared-memory bins flushed with atomics
//     into per-segment global bins, one warp per segment sweeps the 3 x 32 bins for the best split, then a chunked
//     partition into the other half of a ping-pong buffer using atomic range reservation;
//   * BLOCK segments (<= kBlockCap): one CTA owns the segment: bins in shared memory, primitive ids staged in
//     shared memory, in-place stable partition;
//   * WARP segments (<= kWarpCap): same routine with a 32-thread group, four segments per CTA.
// Differences to the reference, on purpose: always 32 bins (one per lane; the reference uses min(32, 4+0.05N)),
// cost in primitives rather than blocks of 4 (our leaves are single-triangle slots of a BVH8 node), splitting
// continues down to single primitives and the 8-wide collapse (rt_core.cuh select_children) decides the leaves.
// Fallback when no bin split exists (all centres coincide): split the segment in the middle
// (heuristic_binning_array_aligned.h performFallbackSplit).
#include <stdio.h>

#include <algorithm>

#include "rtk_device.h"

namespace rtk {

constexpr int kBins = 32;
constexpr uint32_t kBlockCap = 8192;  // ids + bin stash of one segment fit 64 KB of shared memory
constexpr uint32_t kWarpCap = 64;
constexpr uint32_t kChunk = 2048;     // primitives per CTA in the LARGE phase

struct SahTask {
  uint32_t begin, end;   // segment of the primitive-id array
  uint32_t node;         // Node2 to complete (its bounds/first/count/parent were written by the parent)
  uint32_t buf;          // which ping-pong half holds the segment
  float clo[3], chi[3];  // centroid (lower+upper) bounds of the segment
};

struct SahCounters {
  uint32_t n_large, n_block, n_warp;  // next-level list sizes
  uint32_t node_tail;                 // internal Node2 allocation (root = 0)
  uint32_t n_chunks, pad[3];
};

// per LARGE task scratch: global bins + split decision + partition cursors
struct LargeScratch {
  int lo[3][kBins][3], hi[3][kBins][3];  // ordered-int encoded bin bounds
  uint32_t cnt[3][kBins];
  int dim, pos;                          // chosen split (dim < 0: positional fallback)
  uint32_t nl;
  float lbox[6], rbox[6];
  uint32_t lcur, rcur;                   // reservation cursors of the partition
  int lc_lo[3], lc_hi[3], rc_lo[3], rc_hi[3];  // child centroid bounds (ordered ints)
  uint32_t chunk0;                       // first chunk id of this task
};

constexpr int kOrdPosInf = 0x7F800000;            // f2ord(+inf)
constexpr int kOrdNegInf = (int)0x807FFFFF;       // f2ord(-inf)

struct BinMap { float lo[3], scale[3]; };
__device__ __forceinline__ BinMap make_map(const float clo[3], const float chi[3]) {
  BinMap m;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float ext = chi[a] - clo[a];
    m.lo[a] = clo[a];
    m.scale[a] = ext > 1e-34f ? (0.99f * kBins) / ext : 0.0f;   // heuristic_binning.h:25-29
  }
  return m;
}
__device__ __forceinline__ int bin_of(const BinMap& m, float c, int a) {
  const int b = (int)floorf((c - m.lo[a]) * m.scale[a]);
  return min(max(b, 0), kBins - 1);
}

__device__ __forceinline__ float box_half_area(const float b[6]) {
  const float dx = b[3] - b[0], dy = b[4] - b[1], dz = b[5] - b[2];
  return dx * (dy + dz) + dy * dz;
}

// One warp: sweep the 32 bins of axis `a` (lane = bin) and return the best (cost, pos) with left/right boxes and the
// left count.  Bins given as ordered ints.  cost = lA*lN + rA*rN over split planes p in [1,31] with both sides non-empty.
struct SweepResult { float cost; int pos; uint32_t nl; float lbox[6], rbox[6]; };

__device__ __forceinline__ SweepResult sweep_axis(const int* lo /*[kBins][3]*/, const int* hi, const uint32_t* cnt) {
  const int lane = threadIdx.x & 31;
  float b[6];
#pragma unroll
  for (int k = 0; k < 3; ++k) { b[k] = ord2f(lo[lane * 3 + k]); b[3 + k] = ord2f(hi[lane * 3 + k]); }
  uint32_t c = cnt[lane];
  // inclusive prefix (left) and suffix (right) of boxes / counts
  float L[6], R[6];
  uint32_t lc = c, rc = c;
#pragma unroll
  for (int k = 0; k < 6; ++k) { L[k] = b[k]; R[k] = b[k]; }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t ylc = __shfl_up_sync(0xFFFFFFFFu, lc, o), yrc = __shfl_down_sync(0xFFFFFFFFu, rc, o);
    float yl[6], yr[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { yl[k] = __shfl_up_sync(0xFFFFFFFFu, L[k], o); yr[k] = __shfl_down_sync(0xFFFFFFFFu, R[k], o); }
    if (lane >= o) {
      lc += ylc;
#pragma unroll
      for (int k = 0; k < 3; ++k) { L[k] = fminf(L[k], yl[k]); L[3 + k] = fmaxf(L[3 + k], yl[3 + k]); }
    }
    if (lane + o < 32) {
      rc += yrc;
#pragma unroll
      for (int k = 0; k < 3; ++k) { R[k] = fminf(R[k], yr[k]); R[3 + k] = fmaxf(R[3 + k], yr[3 + k]); }
    }
  }
  // split plane p = lane: left = prefix of lane-1, right = suffix of lane
  float Lp[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) Lp[k] = __shfl_up_sync(0xFFFFFFFFu, L[k], 1);
  const uint32_t lcp = __shfl_up_sync(0xFFFFFFFFu, lc, 1);
  float cost = INFINITY;
  if (lane >= 1 && lcp > 0 && rc > 0) cost = box_half_area(Lp) * (float)lcp + box_half_area(R) * (float)rc;
  // argmin over lanes (ties -> lowest plane, like the reference's strict '<' scan from the left)
  float best = cost;
  int bl = lane;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float oc = __shfl_xor_sync(0xFFFFFFFFu, best, o);
    const int ol = __shfl_xor_sync(0xFFFFFFFFu, bl, o);
    if (oc < best || (oc == best && ol < bl)) { best = oc; bl = ol; }
  }
  SweepResult r;
  r.cost = best; r.pos = bl;
  r.nl = __shfl_sync(0xFFFFFFFFu, lcp, bl);
#pragma unroll
  for (int k = 0; k < 6; ++k) { r.lbox[k] = __shfl_sync(0xFFFFFFFFu, Lp[k], bl); r.rbox[k] = __shfl_sync(0xFFFFFFFFu, R[k], bl); }
  return r;
}

// Write a child Node2 and, when it still has to be split, append its task to the list of its size class.
// Returns the child's node id.  Leaves (one primitive) live at id n-1+position.
__device__ uint32_t emit_child(Node2* nodes, uint32_t n, uint32_t parent, uint32_t begin, uint32_t end, uint32_t buf,
                               const float box[6], const float clo[3], const float chi[3], SahCounters* ctr,
                               SahTask* out_large, SahTask* out_block, SahTask* out_warp) {
  const uint32_t count = end - begin;
  uint32_t id;
  if (count == 1) id = n - 1 + begin;
  else id = atomicAdd(&ctr->node_tail, 1u);
  Node2& nd = nodes[id];
  nd.lox = box[0]; nd.loy = box[1]; nd.loz = box[2];
  nd.hix = box[3]; nd.hiy = box[4]; nd.hiz = box[5];
  nd.first = begin; nd.count = count; nd.parent = parent; nd.pad = buf;
  if (count == 1) { nd.left = (int32_t)begin; nd.right = -1; return id; }
  SahTask t;
  t.begin = begin; t.end = end; t.node = id; t.buf = buf;
#pragma unroll
  for (int a = 0; a < 3; ++a) { t.clo[a] = clo[a]; t.chi[a] = chi[a]; }
  if (count > kBlockCap) out_large[atomicAdd(&ctr->n_large, 1u)] = t;
  else if (count > kWarpCap) out_block[atomicAdd(&ctr->n_block, 1u)] = t;
  else out_warp[atomicAdd(&ctr->n_warp, 1u)] = t;
  return id;
}

// ---------------------------------------------------------------------------------------------------------------------
// BLOCK / WARP segments: one thread group owns the segment
// ---------------------------------------------------------------------------------------------------------------------
template <int NT>
__device__ __forceinline__ void group_sync() {
  if (NT == 32) __syncwarp(); else __syncthreads();
}

struct GroupSmem {          // per group
  int lo[3][kBins][3], hi[3][kBins][3];
  uint32_t cnt[3][kBins];
  int c_lo[2][3], c_hi[2][3];   // child centroid bounds
  float lbox[6], rbox[6];
  int dim, pos;
  uint32_t nl;
  uint32_t scan[8];             // warp partial sums of the partition scan
  uint32_t run_l, run_r;
};

// NT threads per group, GROUPS groups per CTA, CAP = max segment size; ids/bins stash: CAP * 8 bytes per group (dynamic smem)
template <int NT, int GROUPS, uint32_t CAP>
__global__ void __launch_bounds__(NT* GROUPS) sah_group_kernel(const SahTask* __restrict__ tasks, uint32_t ntasks,
                                                               const PrimRef* __restrict__ prims, uint32_t* idsA, uint32_t* idsB,
                                                               Node2* nodes, uint32_t n, SahCounters* ctr, SahTask* out_large,
                                                               SahTask* out_block, SahTask* out_warp, uint32_t small_max) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int group = threadIdx.x / NT, tid = threadIdx.x % NT, lane = threadIdx.x & 31, gwarp = tid >> 5;
  GroupSmem* gs = reinterpret_cast<GroupSmem*>(smem_raw) + group;
  uint32_t* stash = reinterpret_cast<uint32_t*>(smem_raw + sizeof(GroupSmem) * GROUPS) + (size_t)group * CAP * 2;
  uint32_t* sid = stash;          // primitive ids of the segment
  uint32_t* sbin = stash + CAP;   // packed bins: x | y<<5 | z<<10
  for (uint32_t ti = blockIdx.x * GROUPS + group; ti < ntasks; ti += gridDim.x * GROUPS) {
    const SahTask t = tasks[ti];
    uint32_t* ids = t.buf ? idsB : idsA;
    const uint32_t count = t.end - t.begin;
    // ---- tiny segments (warp groups only): no binning.  7/8 of all split tasks of a build are at the last three
    // levels; a full 3 x 32-bin sweep for 2..4 primitives costs ~3000 warp instructions and decides almost nothing.
    if (NT == 32 && count <= small_max) {
      // object-median split along the longest centroid axis.  The lanes first put the segment into a canonical order
      // (centre along that axis, primitive id as tie-break), so the result depends only on the SET of primitives --
      // the LARGE-phase partition reserves ranges with atomics and leaves the order inside a segment run-dependent.
      const uint32_t nl = count / 2;
      const bool in = (uint32_t)lane < count;
      float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
      uint32_t id = 0xFFFFFFFFu;
      if (in) {
        id = ids[t.begin + lane];
        const float4 plo = __ldg(reinterpret_cast<const float4*>(&prims[id]));
        const float4 phi = __ldg(reinterpret_cast<const float4*>(&prims[id]) + 1);
        lo[0] = plo.x; lo[1] = plo.y; lo[2] = plo.z; hi[0] = phi.x; hi[1] = phi.y; hi[2] = phi.z;
      }
      const float ex = t.chi[0] - t.clo[0], ey = t.chi[1] - t.clo[1], ez = t.chi[2] - t.clo[2];
      const int ax = (ex >= ey && ex >= ez) ? 0 : (ey >= ez ? 1 : 2);
      const float key = in ? (ax == 0 ? lo[0] + hi[0] : (ax == 1 ? lo[1] + hi[1] : lo[2] + hi[2])) : INFINITY;
      uint32_t rank = 0;
      for (uint32_t j = 0; j < count; ++j) {
        const float kj = __shfl_sync(0xFFFFFFFFu, key, (int)j);
        const uint32_t ij = __shfl_sync(0xFFFFFFFFu, id, (int)j);
        if (kj < key || (kj == key && ij < id)) ++rank;
      }
      __syncwarp();
      if (in) ids[t.begin + rank] = id;
      const bool left = in && rank < nl;
      float lb[6], rb[6], lcl[3], lch[3], rcl[3], rch[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float c = lo[k] + hi[k];
        float a0 = (in && left) ? lo[k] : INFINITY, a1 = (in && left) ? hi[k] : -INFINITY;
        float b0 = (in && !left) ? lo[k] : INFINITY, b1 = (in && !left) ? hi[k] : -INFINITY;
        float c0 = (in && left) ? c : INFINITY, c1 = (in && left) ? c : -INFINITY;
        float d0 = (in && !left) ? c : INFINITY, d1 = (in && !left) ? c : -INFINITY;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a0 = fminf(a0, __shfl_xor_sync(0xFFFFFFFFu, a0, o)); a1 = fmaxf(a1, __shfl_xor_sync(0xFFFFFFFFu, a1, o));
          b0 = fminf(b0, __shfl_xor_sync(0xFFFFFFFFu, b0, o)); b1 = fmaxf(b1, __shfl_xor_sync(0xFFFFFFFFu, b1, o));
          c0 = fminf(c0, __shfl_xor_sync(0xFFFFFFFFu, c0, o)); c1 = fmaxf(c1, __shfl_xor_sync(0xFFFFFFFFu, c1, o));
          d0 = fminf(d0, __shfl_xor_sync(0xFFFFFFFFu, d0, o)); d1 = fmaxf(d1, __shfl_xor_sync(0xFFFFFFFFu, d1, o));
        }
        lb[k] = a0; lb[3 + k] = a1; rb[k] = b0; rb[3 + k] = b1; lcl[k] = c0; lch[k] = c1; rcl[k] = d0; rch[k] = d1;
      }
      __syncwarp();
      if (lane == 0) {
        const uint32_t l = emit_child(nodes, n, t.node, t.begin, t.begin + nl, t.buf, lb, lcl, lch, ctr, out_large, out_block, out_warp);
        const uint32_t r = emit_child(nodes, n, t.node, t.begin + nl, t.end, t.buf, rb, rcl, rch, ctr, out_large, out_block, out_warp);
        nodes[t.node].left = (int32_t)l;
        nodes[t.node].right = (int32_t)r;
      }
      __syncwarp();
      continue;
    }
    const BinMap map = make_map(t.clo, t.chi);
    // ---- clear bins
    for (int i = tid; i < 3 * kBins; i += NT) {
      (&gs->cnt[0][0])[i] = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) { (&gs->lo[0][0][0])[i * 3 + k] = kOrdPosInf; (&gs->hi[0][0][0])[i * 3 + k] = kOrdNegInf; }
    }
    if (tid < 6) { (&gs->c_lo[0][0])[tid] = kOrdPosInf; (&gs->c_hi[0][0])[tid] = kOrdNegInf; }
    group_sync<NT>();
    // ---- pass 1: bin
    for (uint32_t i = tid; i < count; i += NT) {
      const uint32_t id = ids[t.begin + i];
      const float4 plo = __ldg(reinterpret_cast<const float4*>(&prims[id]));
      const float4 phi = __ldg(reinterpret_cast<const float4*>(&prims[id]) + 1);
      const float lo[3] = {plo.x, plo.y, plo.z}, hi[3] = {phi.x, phi.y, phi.z};
      uint32_t packed = 0;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const int b = bin_of(map, lo[a] + hi[a], a);
        packed |= (uint32_t)b << (5 * a);
        atomicAdd(&gs->cnt[a][b], 1u);
#pragma unroll
        for (int k = 0; k < 3; ++k) { atomicMin(&gs->lo[a][b][k], f2ord(lo[k])); atomicMax(&gs->hi[a][b][k], f2ord(hi[k])); }
      }
      sid[i] = id; sbin[i] = packed;
    }
    group_sync<NT>();
    // ---- sweep: first warp of the group, axes in turn
    if (gwarp == 0) {
      float best = INFINITY;
      int bdim = -1;
      SweepResult br;
      br.pos = 0; br.nl = 0;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (map.scale[a] == 0.0f) continue;   // zero-sized dimension (heuristic_binning.h:375-377)
        const SweepResult r = sweep_axis(&gs->lo[a][0][0], &gs->hi[a][0][0], &gs->cnt[a][0]);
        if (r.cost < best) { best = r.cost; bdim = a; br = r; }
      }
      if (lane == 0) {
        gs->dim = bdim; gs->pos = br.pos;
        gs->nl = bdim >= 0 ? br.nl : count / 2;   // positional fallback: first half goes left
#pragma unroll
        for (int k = 0; k < 6; ++k) { gs->lbox[k] = br.lbox[k]; gs->rbox[k] = br.rbox[k]; }
        gs->run_l = 0; gs->run_r = 0;
      }
    }
    group_sync<NT>();
    const int dim = gs->dim, pos = gs->pos;
    const uint32_t nl = gs->nl;
    // ---- pass 2: stable in-place partition (all reads come from the shared-memory stash) + child bounds
    int flo[2][3], fhi[2][3];   // per-thread centroid bounds of (left,right), ordered ints
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < 3; ++k) { flo[s][k] = kOrdPosInf; fhi[s][k] = kOrdNegInf; }
    for (uint32_t base = 0; base < count; base += NT) {
      const uint32_t i = base + tid;
      const bool in = i < count;
      bool left = false;
      uint32_t id = 0;
      if (in) {
        id = sid[i];
        left = dim >= 0 ? (int)((sbin[i] >> (5 * dim)) & 31u) < pos : i < nl;
      }
      const uint32_t bl = __ballot_sync(0xFFFFFFFFu, in && left), br = __ballot_sync(0xFFFFFFFFu, in && !left);
      const uint32_t lt = (1u << lane) - 1u;
      uint32_t offl = __popc(bl & lt), offr = __popc(br & lt);
      if (NT > 32) {
        if (lane == 0) gs->scan[gwarp] = (uint32_t)__popc(bl) | ((uint32_t)__popc(br) << 16);
        __syncthreads();
        for (int w = 0; w < gwarp; ++w) { const uint32_t v = gs->scan[w]; offl += v & 0xFFFFu; offr += v >> 16; }
      }
      const uint32_t rl = gs->run_l, rr = gs->run_r;
      if (in) {
        const uint32_t dst = left ? (t.begin + rl + offl) : (t.begin + nl + rr + offr);
        ids[dst] = id;
        const float4 plo = __ldg(reinterpret_cast<const float4*>(&prims[id]));
        const float4 phi = __ldg(reinterpret_cast<const float4*>(&prims[id]) + 1);
        const float lo3[3] = {plo.x, plo.y, plo.z}, hi3[3] = {phi.x, phi.y, phi.z};
        const int s = left ? 0 : 1;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int c = f2ord(lo3[k] + hi3[k]);
          flo[s][k] = min(flo[s][k], c); fhi[s][k] = max(fhi[s][k], c);
        }
      }
      group_sync<NT>();
      if (NT > 32) {
        if (tid == 0) {
          uint32_t tl = 0, tr = 0;
          for (int w = 0; w < NT / 32; ++w) { const uint32_t v = gs->scan[w]; tl += v & 0xFFFFu; tr += v >> 16; }
          gs->run_l = rl + tl; gs->run_r = rr + tr;
        }
      } else if (lane == 0) { gs->run_l = rl + __popc(bl); gs->run_r = rr + __popc(br); }
      group_sync<NT>();
    }
    // reduce child centroid bounds: warp shuffle, then shared atomics
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        int a = flo[s][k], b = fhi[s][k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a = min(a, __shfl_xor_sync(0xFFFFFFFFu, a, o)); b = max(b, __shfl_xor_sync(0xFFFFFFFFu, b, o));
        }
        if (lane == 0) { atomicMin(&gs->c_lo[s][k], a); atomicMax(&gs->c_hi[s][k], b); }
      }
    group_sync<NT>();
    if (tid == 0) {
      float lb[6], rb[6], lcl[3], lch[3], rcl[3], rch[3];
#pragma unroll
      for (int k = 0; k < 6; ++k) { lb[k] = gs->lbox[k]; rb[k] = gs->rbox[k]; }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        lcl[k] = ord2f(gs->c_lo[0][k]); lch[k] = ord2f(gs->c_hi[0][k]);
        rcl[k] = ord2f(gs->c_lo[1][k]); rch[k] = ord2f(gs->c_hi[1][k]);
      }
      if (dim < 0) {
        // all centres coincide (or NaN-free degenerate): both children get the parent's box, which is conservative
        const Node2& self = nodes[t.node];
        lb[0] = rb[0] = self.lox; lb[1] = rb[1] = self.loy; lb[2] = rb[2] = self.loz;
        lb[3] = rb[3] = self.hix; lb[4] = rb[4] = self.hiy; lb[5] = rb[5] = self.hiz;
      }
      const uint32_t l = emit_child(nodes, n, t.node, t.begin, t.begin + nl, t.buf, lb, lcl, lch, ctr, out_large, out_block, out_warp);
      const uint32_t r = emit_child(nodes, n, t.node, t.begin + nl, t.end, t.buf, rb, rcl, rch, ctr, out_large, out_block, out_warp);
      nodes[t.node].left = (int32_t)l;
      nodes[t.node].right = (int32_t)r;
    }
    group_sync<NT>();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// LARGE segments
// ---------------------------------------------------------------------------------------------------------------------
__global__ void sah_large_setup(const SahTask* __restrict__ tasks, uint32_t ntasks, LargeScratch* scr, uint32_t* chunk_task,
                                SahCounters* ctr) {
  // single CTA: clear scratch, assign chunk ranges
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (uint32_t t = 0; t < ntasks; ++t) { scr[t].chunk0 = run; run += (tasks[t].end - tasks[t].begin + kChunk - 1) / kChunk; }
    ctr->n_chunks = run;
  }
  __syncthreads();
  for (uint32_t t = 0; t < ntasks; ++t) {
    LargeScratch& s = scr[t];
    for (int i = threadIdx.x; i < 3 * kBins; i += blockDim.x) {
      (&s.cnt[0][0])[i] = 0;
      for (int k = 0; k < 3; ++k) { (&s.lo[0][0][0])[i * 3 + k] = kOrdPosInf; (&s.hi[0][0][0])[i * 3 + k] = kOrdNegInf; }
    }
    if (threadIdx.x < 3) {
      s.lc_lo[threadIdx.x] = s.rc_lo[threadIdx.x] = kOrdPosInf;
      s.lc_hi[threadIdx.x] = s.rc_hi[threadIdx.x] = kOrdNegInf;
    }
    if (threadIdx.x == 0) { s.lcur = 0; s.rcur = 0; }
    const uint32_t nch = (tasks[t].end - tasks[t].begin + kChunk - 1) / kChunk;
    for (uint32_t c = threadIdx.x; c < nch; c += blockDim.x) chunk_task[s.chunk0 + c] = t;
  }
}

__global__ void __launch_bounds__(256) sah_large_bin(const SahTask* __restrict__ tasks, const uint32_t* __restrict__ chunk_task,
                                                     LargeScratch* scr, const PrimRef* __restrict__ prims,
                                                     const uint32_t* __restrict__ idsA, const uint32_t* __restrict__ idsB) {
  __shared__ int slo[3][kBins][3], shi[3][kBins][3];
  __shared__ uint32_t scnt[3][kBins];
  const uint32_t ti = chunk_task[blockIdx.x];
  const SahTask t = tasks[ti];
  LargeScratch& s = scr[ti];
  const uint32_t* ids = t.buf ? idsB : idsA;
  const BinMap map = make_map(t.clo, t.chi);
  for (int i = threadIdx.x; i < 3 * kBins; i += 256) {
    (&scnt[0][0])[i] = 0;
    for (int k = 0; k < 3; ++k) { (&slo[0][0][0])[i * 3 + k] = kOrdPosInf; (&shi[0][0][0])[i * 3 + k] = kOrdNegInf; }
  }
  __syncthreads();
  const uint32_t c0 = t.begin + (blockIdx.x - s.chunk0) * kChunk, c1 = min(c0 + kChunk, t.end);
  for (uint32_t i = c0 + threadIdx.x; i < c1; i += 256) {
    const uint32_t id = ids[i];
    const float4 plo = __ldg(reinterpret_cast<const float4*>(&prims[id]));
    const float4 phi = __ldg(reinterpret_cast<const float4*>(&prims[id]) + 1);
    const float lo[3] = {plo.x, plo.y, plo.z}, hi[3] = {phi.x, phi.y, phi.z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int b = bin_of(map, lo[a] + hi[a], a);
      atomicAdd(&scnt[a][b], 1u);
#pragma unroll
      for (int k = 0; k < 3; ++k) { atomicMin(&slo[a][b][k], f2ord(lo[k])); atomicMax(&shi[a][b][k], f2ord(hi[k])); }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * kBins; i += 256) {
    const uint32_t c = (&scnt[0][0])[i];
    if (c) {
      atomicAdd(&(&s.cnt[0][0])[i], c);
      for (int k = 0; k < 3; ++k) {
        atomicMin(&(&s.lo[0][0][0])[i * 3 + k], (&slo[0][0][0])[i * 3 + k]);
        atomicMax(&(&s.hi[0][0][0])[i * 3 + k], (&shi[0][0][0])[i * 3 + k]);
      }
    }
  }
}

__global__ void __launch_bounds__(128) sah_large_split(const SahTask* __restrict__ tasks, uint32_t ntasks, LargeScratch* scr) {
  const uint32_t ti = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (ti >= ntasks) return;
  const int lane = threadIdx.x & 31;
  const SahTask t = tasks[ti];
  LargeScratch& s = scr[ti];
  const BinMap map = make_map(t.clo, t.chi);
  float best = INFINITY;
  int bdim = -1;
  SweepResult br;
  br.pos = 0; br.nl = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (map.scale[a] == 0.0f) continue;
    const SweepResult r = sweep_axis(&s.lo[a][0][0], &s.hi[a][0][0], &s.cnt[a][0]);
    if (r.cost < best) { best = r.cost; bdim = a; br = r; }
  }
  if (lane == 0) {
    s.dim = bdim; s.pos = br.pos;
    s.nl = bdim >= 0 ? br.nl : (t.end - t.begin) / 2;
    for (int k = 0; k < 6; ++k) { s.lbox[k] = br.lbox[k]; s.rbox[k] = br.rbox[k]; }
  }
}

__global__ void __launch_bounds__(256) sah_large_partition(const SahTask* __restrict__ tasks, const uint32_t* __restrict__ chunk_task,
                                                           LargeScratch* scr, const PrimRef* __restrict__ prims,
                                                           uint32_t* idsA, uint32_t* idsB) {
  __shared__ uint32_t wl[8], wr[8], basel, baser;
  __shared__ int c_lo[2][3], c_hi[2][3];
  const uint32_t ti = chunk_task[blockIdx.x];
  const SahTask t = tasks[ti];
  LargeScratch& s = scr[ti];
  const uint32_t* in = t.buf ? idsB : idsA;
  uint32_t* out = t.buf ? idsA : idsB;
  const BinMap map = make_map(t.clo, t.chi);
  const int dim = s.dim, pos = s.pos;
  const uint32_t nl = s.nl;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < 6) { (&c_lo[0][0])[threadIdx.x] = kOrdPosInf; (&c_hi[0][0])[threadIdx.x] = kOrdNegInf; }
  const uint32_t c0 = t.begin + (blockIdx.x - s.chunk0) * kChunk, c1 = min(c0 + kChunk, t.end);
  // each thread owns kChunk/256 consecutive-strided items; two passes: count, then reserve + write
  constexpr int ITEMS = kChunk / 256;
  uint32_t id[ITEMS];
  bool left[ITEMS], in_range[ITEMS];
  uint32_t myl = 0, myr = 0;
  int flo[2][3], fhi[2][3];
#pragma unroll
  for (int sd = 0; sd < 2; ++sd)
#pragma unroll
    for (int k = 0; k < 3; ++k) { flo[sd][k] = kOrdPosInf; fhi[sd][k] = kOrdNegInf; }
#pragma unroll
  for (int j = 0; j < ITEMS; ++j) {
    const uint32_t i = c0 + j * 256 + threadIdx.x;
    in_range[j] = i < c1;
    left[j] = false; id[j] = 0;
    if (in_range[j]) {
      id[j] = in[i];
      const float4 plo = __ldg(reinterpret_cast<const float4*>(&prims[id[j]]));
      const float4 phi = __ldg(reinterpret_cast<const float4*>(&prims[id[j]]) + 1);
      const float c[3] = {plo.x + phi.x, plo.y + phi.y, plo.z + phi.z};
      left[j] = dim >= 0 ? bin_of(map, c[dim], dim) < pos : (i - t.begin) < nl;
      const int sd = left[j] ? 0 : 1;
#pragma unroll
      for (int k = 0; k < 3; ++k) { const int o = f2ord(c[k]); flo[sd][k] = min(flo[sd][k], o); fhi[sd][k] = max(fhi[sd][k], o); }
      if (left[j]) ++myl; else ++myr;
    }
  }
  // block exclusive scan of (myl, myr) in thread order: positions inside the chunk's reserved ranges
  uint32_t xl = myl, xr = myr;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t yl = __shfl_up_sync(0xFFFFFFFFu, xl, o), yr = __shfl_up_sync(0xFFFFFFFFu, xr, o);
    if (lane >= o) { xl += yl; xr += yr; }
  }
  if (lane == 31) { wl[warp] = xl; wr[warp] = xr; }
  __syncthreads();
  uint32_t offl = xl - myl, offr = xr - myr;
  for (int w = 0; w < warp; ++w) { offl += wl[w]; offr += wr[w]; }
  if (threadIdx.x == 255) {
    basel = atomicAdd(&s.lcur, offl + myl);
    baser = atomicAdd(&s.rcur, offr + myr);
  }
  __syncthreads();
  const uint32_t bl = t.begin + basel, br = t.begin + nl + baser;
#pragma unroll
  for (int j = 0; j < ITEMS; ++j) {
    if (!in_range[j]) continue;
    if (left[j]) out[bl + offl++] = id[j]; else out[br + offr++] = id[j];
  }
  // child centroid bounds
#pragma unroll
  for (int sd = 0; sd < 2; ++sd)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      int a = flo[sd][k], b = fhi[sd][k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { a = min(a, __shfl_xor_sync(0xFFFFFFFFu, a, o)); b = max(b, __shfl_xor_sync(0xFFFFFFFFu, b, o)); }
      if (lane == 0) { atomicMin(&c_lo[sd][k], a); atomicMax(&c_hi[sd][k], b); }
    }
  __syncthreads();
  if (threadIdx.x < 3) {
    const int k = threadIdx.x;
    atomicMin(&s.lc_lo[k], c_lo[0][k]); atomicMax(&s.lc_hi[k], c_hi[0][k]);
    atomicMin(&s.rc_lo[k], c_lo[1][k]); atomicMax(&s.rc_hi[k], c_hi[1][k]);
  }
}

__global__ void __launch_bounds__(128) sah_large_emit(const SahTask* __restrict__ tasks, uint32_t ntasks, const LargeScratch* scr,
                                                      Node2* nodes, uint32_t n, SahCounters* ctr, SahTask* out_large,
                                                      SahTask* out_block, SahTask* out_warp) {
  const uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if (ti >= ntasks) return;
  const SahTask t = tasks[ti];
  const LargeScratch& s = scr[ti];
  float lb[6], rb[6], lcl[3], lch[3], rcl[3], rch[3];
  for (int k = 0; k < 6; ++k) { lb[k] = s.lbox[k]; rb[k] = s.rbox[k]; }
  for (int k = 0; k < 3; ++k) { lcl[k] = ord2f(s.lc_lo[k]); lch[k] = ord2f(s.lc_hi[k]); rcl[k] = ord2f(s.rc_lo[k]); rch[k] = ord2f(s.rc_hi[k]); }
  if (s.dim < 0) {
    const Node2& self = nodes[t.node];
    lb[0] = rb[0] = self.lox; lb[1] = rb[1] = self.loy; lb[2] = rb[2] = self.loz;
    lb[3] = rb[3] = self.hix; lb[4] = rb[4] = self.hiy; lb[5] = rb[5] = self.hiz;
  }
  const uint32_t nb = t.buf ^ 1u;  // the partition wrote into the other half of the ping-pong buffer
  const uint32_t l = emit_child(nodes, n, t.node, t.begin, t.begin + s.nl, nb, lb, lcl, lch, ctr, out_large, out_block, out_warp);
  const uint32_t r = emit_child(nodes, n, t.node, t.begin + s.nl, t.end, nb, rb, rcl, rch, ctr, out_large, out_block, out_warp);
  nodes[t.node].left = (int32_t)l;
  nodes[t.node].right = (int32_t)r;
}

__global__ void sah_init(Node2* nodes, uint32_t n, const float* bounds6, const float* cent6, SahTask* lists[3], SahCounters* ctr) {
  Node2& root = nodes[0];
  root.lox = bounds6[0]; root.loy = bounds6[1]; root.loz = bounds6[2];
  root.hix = bounds6[3]; root.hiy = bounds6[4]; root.hiz = bounds6[5];
  root.first = 0; root.count = n; root.parent = 0xFFFFFFFFu; root.pad = 0; root.left = 0; root.right = 0;
  SahTask t;
  t.begin = 0; t.end = n; t.node = 0; t.buf = 0;
  for (int a = 0; a < 3; ++a) { t.clo[a] = cent6[a]; t.chi[a] = cent6[3 + a]; }
  ctr->n_large = ctr->n_block = ctr->n_warp = 0; ctr->node_tail = 1; ctr->n_chunks = 0;
  if (n > kBlockCap) { lists[0][0] = t; ctr->n_large = 1; }
  else if (n > kWarpCap) { lists[1][0] = t; ctr->n_block = 1; }
  else { lists[2][0] = t; ctr->n_warp = 1; }
}

// single-primitive leaves: Node2 at id n-1+j for every position j; parent/bounds come from emit_child, the
// position->primitive mapping is read by the collapse from the ping-pong half recorded in `pad`.
// (nothing to do here: emit_child wrote the leaves.)

#define CKS(x)                                                                                        \
  do {                                                                                                \
    cudaError_t e_ = (x);                                                                             \
    if (e_ != cudaSuccess) {                                                                          \
      snprintf(errmsg, 256, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return (int)e_;                                                                                 \
    }                                                                                                 \
  } while (0)

// ids: Morton-sorted primitive ids (half A); idsB: scratch half of the ping-pong buffer.
// scene_bounds / cent_bounds: 6 floats each on the HOST.
int build_sah_tree(const PrimRef* prims, uint32_t* idsA, uint32_t* idsB, uint32_t n, Node2* nodes, const float* scene_bounds,
                   const float* cent_bounds, cudaStream_t st, char* errmsg) {
  const size_t max_tasks = (size_t)n / 2 + 2;
  SahTask* lists[2][3] = {};
  SahCounters* d_ctr = nullptr;
  LargeScratch* d_scr = nullptr;
  uint32_t* d_chunk_task = nullptr;
  float* d_b = nullptr;
  SahTask** d_lists = nullptr;
  const size_t max_large = (size_t)n / kBlockCap + 2;
  const size_t max_chunks = (size_t)n / kChunk + max_large + 2;
  int rc = 0;
  auto cleanup = [&]() {
    for (int p = 0; p < 2; ++p) for (int k = 0; k < 3; ++k) if (lists[p][k]) cudaFreeAsync(lists[p][k], st);
    if (d_ctr) cudaFreeAsync(d_ctr, st);
    if (d_scr) cudaFreeAsync(d_scr, st);
    if (d_chunk_task) cudaFreeAsync(d_chunk_task, st);
    if (d_b) cudaFreeAsync(d_b, st);
    if (d_lists) cudaFreeAsync(d_lists, st);
  };
#define CKC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { snprintf(errmsg, 256, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); cleanup(); return (int)e_; } } while (0)
  for (int p = 0; p < 2; ++p) {
    CKC(cudaMallocAsync(reinterpret_cast<void**>(&lists[p][0]), max_large * sizeof(SahTask), st));
    CKC(cudaMallocAsync(reinterpret_cast<void**>(&lists[p][1]), ((size_t)n / kWarpCap + 2) * sizeof(SahTask), st));
    CKC(cudaMallocAsync(reinterpret_cast<void**>(&lists[p][2]), max_tasks * sizeof(SahTask), st));
  }
  CKC(cudaMallocAsync(reinterpret_cast<void**>(&d_ctr), sizeof(SahCounters), st));
  CKC(cudaMallocAsync(reinterpret_cast<void**>(&d_scr), max_large * sizeof(LargeScratch), st));
  CKC(cudaMallocAsync(reinterpret_cast<void**>(&d_chunk_task), max_chunks * 4, st));
  CKC(cudaMallocAsync(reinterpret_cast<void**>(&d_b), 12 * sizeof(float), st));
  CKC(cudaMallocAsync(reinterpret_cast<void**>(&d_lists), 3 * sizeof(SahTask*), st));
  float hb[12];
  for (int k = 0; k < 6; ++k) { hb[k] = scene_bounds[k]; hb[6 + k] = cent_bounds[k]; }
  CKC(cudaMemcpyAsync(d_b, hb, sizeof hb, cudaMemcpyHostToDevice, st));
  CKC(cudaMemcpyAsync(d_lists, lists[0], 3 * sizeof(SahTask*), cudaMemcpyHostToDevice, st));
  sah_init<<<1, 1, 0, st>>>(nodes, n, d_b, d_b + 6, d_lists, d_ctr);
  count_launch();

  constexpr int BLOCK_NT = 256, WARP_GROUPS = 4;
  const size_t smem_block = sizeof(GroupSmem) + (size_t)kBlockCap * 8;
  const size_t smem_warp = (sizeof(GroupSmem) + (size_t)kWarpCap * 8) * WARP_GROUPS;
  CKC(cudaFuncSetAttribute(sah_group_kernel<BLOCK_NT, 1, kBlockCap>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_block));
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);

  int cur = 0;
  SahCounters hc;
  for (int level = 0;; ++level) {
    CKC(cudaMemcpyAsync(&hc, d_ctr, sizeof hc, cudaMemcpyDeviceToHost, st));
    CKC(cudaStreamSynchronize(st));
    const uint32_t nL = hc.n_large, nB = hc.n_block, nW = hc.n_warp;
    if (nL + nB + nW == 0) break;
    if (level > 4096) { snprintf(errmsg, 256, "SAH build did not terminate"); cleanup(); return -1; }
    if (nL > max_large) { snprintf(errmsg, 256, "internal: large task overflow"); cleanup(); return -1; }
    // reset the next-level counters (keep node_tail)
    CKC(cudaMemsetAsync(d_ctr, 0, 3 * sizeof(uint32_t), st));
    SahTask** in = lists[cur];
    SahTask** out = lists[cur ^ 1];
    if (nL) {
      sah_large_setup<<<1, 256, 0, st>>>(in[0], nL, d_scr, d_chunk_task, d_ctr);
      uint32_t nchunks = 0;
      CKC(cudaMemcpyAsync(&nchunks, &d_ctr->n_chunks, 4, cudaMemcpyDeviceToHost, st));
      CKC(cudaStreamSynchronize(st));
      sah_large_bin<<<nchunks, 256, 0, st>>>(in[0], d_chunk_task, d_scr, prims, idsA, idsB);
      sah_large_split<<<(nL * 32 + 127) / 128, 128, 0, st>>>(in[0], nL, d_scr);
      sah_large_partition<<<nchunks, 256, 0, st>>>(in[0], d_chunk_task, d_scr, prims, idsA, idsB);
      sah_large_emit<<<(nL + 127) / 128, 128, 0, st>>>(in[0], nL, d_scr, nodes, n, d_ctr, out[0], out[1], out[2]);
      count_launch(5);
    }
    if (nB) {
      const uint32_t grid = std::min<uint32_t>(nB, (uint32_t)sms * 8);
      sah_group_kernel<BLOCK_NT, 1, kBlockCap><<<grid, BLOCK_NT, smem_block, st>>>(in[1], nB, prims, idsA, idsB, nodes, n, d_ctr,
                                                                                  out[0], out[1], out[2], 0u);
      count_launch();
    }
    if (nW) {
      const uint32_t grid = std::min<uint32_t>((nW + WARP_GROUPS - 1) / WARP_GROUPS, (uint32_t)sms * 32);
      sah_group_kernel<32, WARP_GROUPS, kWarpCap><<<grid, 32 * WARP_GROUPS, smem_warp, st>>>(in[2], nW, prims, idsA, idsB, nodes, n,
                                                                                             d_ctr, out[0], out[1], out[2], (uint32_t)tuning().sah_small);
      count_launch();
    }
    CKC(cudaGetLastError());
    cur ^= 1;
  }
  CKC(cudaStreamSynchronize(st));
  cleanup();
  return rc;
}

}  // namespace rtk
