// TEST TOOL: kernels that trace from device code with argument filters (include/embree4_b200_device.cuh), compiled as a user
// would (build.sh: nvcc for sm_90a, default floating-point flags, -I include only), plus host C callbacks with the same rules for
// the host-pointer entry points.  tests/test_device_filter.py and scripts/device_filter_bench.py drive the extern "C" functions
// with ctypes.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "embree4_b200.h"
#include "embree4_b200_device.cuh"

namespace {

constexpr int kThreads = 128;
// hair_geometry_device.h:71-74: hair_Kt = 0.8f * hair_K
__host__ __device__ inline float hair_kt(int k) { return k == 0 ? 0.8f * 0.8f : k == 1 ? 0.8f * 0.57f : 0.8f * 0.32f; }

// The accept / reject rule of tests/filter_cases.py rejects(): one candidate in four, from its ids alone, so the final hit does
// not depend on the order in which a traversal offers the candidates.
__host__ __device__ inline bool rejects(uint32_t geomID, uint32_t primID, uint32_t instID) {
  const uint32_t h = primID * 2654435761u + geomID * 40503u + (instID == RTC_INVALID_GEOMETRY_ID ? 0u : (instID + 1u) * 97u);
  return ((h >> 7) & 3u) == 0u;
}
// What the hit-editing filters write into an accepted hit: u and v swapped, Ng negated, instPrimID tagged with the primID.
__host__ __device__ inline void edit_hit(float& ngx, float& ngy, float& ngz, float& u, float& v, uint32_t primID, uint32_t& instPrimID) {
  const float t = u; u = v; v = t;
  ngx = -ngx; ngy = -ngy; ngz = -ngz;
  instPrimID = primID ^ 0x5A5A0000u;
}

// One call as the recording filter saw it: words 0-11 the RTCRay, 12-20 the RTCHit, 21-22 context instID / instPrimID,
// 23 the thread's ray index, 24-25 geometryUserPtr, 26 the decision (1 accepted)
struct Record { uint32_t w[32]; };

// The per-thread context: RTCRayQueryContext first, then this tool's fields (the hair tutorial's RayQueryContext layout).
struct ThreadContext {
  RTCRayQueryContext base;
  float T[3];               // transparency of the hair shadow filter
  uint32_t ray;             // index of the thread's ray
  Record* rec; unsigned* rec_count; unsigned rec_cap;   // recording filter
  float* T_by_id;           // hair filter with per-ray state indexed by ray.id
};

enum Filter { F_NONE = 0, F_ACCEPT = 1, F_RULE = 2, F_EDIT = 3, F_RECORD = 4, F_HAIR = 5, F_HAIR_ID = 6, F_TFAR = 7 };

__device__ void accept_filter(const RTCFilterFunctionNArguments*) {}
__device__ void rule_filter(const RTCFilterFunctionNArguments* a) {
  const RTCHit* h = reinterpret_cast<const RTCHit*>(a->hit);
  if (rejects(h->geomID, h->primID, h->instID[0])) a->valid[0] = 0;
}
__device__ void edit_filter(const RTCFilterFunctionNArguments* a) {
  RTCHit* h = reinterpret_cast<RTCHit*>(a->hit);
  if (rejects(h->geomID, h->primID, h->instID[0])) { a->valid[0] = 0; return; }
  edit_hit(h->Ng_x, h->Ng_y, h->Ng_z, h->u, h->v, h->primID, h->instPrimID[0]);
}
// the rule, and an accepted hit pulls ray.tfar in by one ulp: the distance written and culled against is the filter's, not the
// candidate's (a shrink that no other candidate's t falls into, so the result does not depend on the order of the candidates)
__device__ void tfar_filter(const RTCFilterFunctionNArguments* a) {
  const RTCHit* h = reinterpret_cast<const RTCHit*>(a->hit);
  if (rejects(h->geomID, h->primID, h->instID[0])) { a->valid[0] = 0; return; }
  RTCRay* r = reinterpret_cast<RTCRay*>(a->ray);
  r->tfar = nextafterf(r->tfar, 0.0f);
}
__device__ void record_filter(const RTCFilterFunctionNArguments* a) {
  const RTCHit* h = reinterpret_cast<const RTCHit*>(a->hit);
  const bool ok = !rejects(h->geomID, h->primID, h->instID[0]);
  ThreadContext* c = reinterpret_cast<ThreadContext*>(a->context);
  const unsigned k = atomicAdd(c->rec_count, 1u);
  if (k < c->rec_cap) {
    Record r;
    memset(&r, 0, sizeof r);
    memcpy(r.w, a->ray, 48);
    memcpy(r.w + 12, a->hit, 36);
    r.w[21] = c->base.instID[0]; r.w[22] = c->base.instPrimID[0]; r.w[23] = c->ray;
    const unsigned long long up = (unsigned long long)(uintptr_t)a->geometryUserPtr;
    r.w[24] = (uint32_t)up; r.w[25] = (uint32_t)(up >> 32); r.w[26] = ok ? 1u : 0u;
    c->rec[k] = r;
  }
  if (!ok) a->valid[0] = 0;
}
// occlusionFilter of hair_geometry_device.cpp:208-238, its transparency in the extended context
__device__ void hair_filter(const RTCFilterFunctionNArguments* a) {
  if (!a->valid[0]) return;
  ThreadContext* c = reinterpret_cast<ThreadContext*>(a->context);
  float T[3];
  for (int k = 0; k < 3; ++k) { T[k] = hair_kt(k) * c->T[k]; c->T[k] = T[k]; }
  if (fmaxf(T[0], fmaxf(T[1], T[2])) > 0.02f) a->valid[0] = 0;
}
// the same filter with the transparency in a global array indexed by ray.id: the host path can run it in one batched call
__device__ void hair_id_filter(const RTCFilterFunctionNArguments* a) {
  if (!a->valid[0]) return;
  float* Tp = reinterpret_cast<ThreadContext*>(a->context)->T_by_id + 3 * (size_t)reinterpret_cast<const RTCRay*>(a->ray)->id;
  float T[3];
  for (int k = 0; k < 3; ++k) { T[k] = hair_kt(k) * Tp[k]; Tp[k] = T[k]; }
  if (fmaxf(T[0], fmaxf(T[1], T[2])) > 0.02f) a->valid[0] = 0;
}

__device__ RTCFilterFunctionN pick(int which) {   // the addresses are taken in device code
  switch (which) {
    case F_ACCEPT: return accept_filter;
    case F_RULE: return rule_filter;
    case F_EDIT: return edit_filter;
    case F_RECORD: return record_filter;
    case F_HAIR: return hair_filter;
    case F_HAIR_ID: return hair_id_filter;
    case F_TFAR: return tfar_filter;
    default: return nullptr;
  }
}

struct Launch {   // what every thread's arguments and context are made of
  int which; unsigned flags, feature_mask; int with_ctx; unsigned seedI, seedP;
  Record* rec; unsigned* rec_count; unsigned rec_cap;
  float* T_out;          // F_HAIR: the context's transparency after the query, 3 floats per ray
  float* T_by_id;        // F_HAIR_ID
  unsigned* ctx_after;   // with_ctx: the context's instID / instPrimID after the query, 2 per ray
};

// one thread per ray; RTCIntersectArguments / RTCOccludedArguments and the context live in the thread's own memory
template <bool OCCLUDED>
__global__ void filter_kernel(const RTCB200DeviceTraversable t, void* recs, size_t n, const Launch L) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ThreadContext c;
  c.base.instID[0] = L.seedI; c.base.instPrimID[0] = L.seedP;
  c.T[0] = c.T[1] = c.T[2] = 1.0f;
  c.ray = (uint32_t)i; c.rec = L.rec; c.rec_count = L.rec_count; c.rec_cap = L.rec_cap; c.T_by_id = L.T_by_id;
  if (OCCLUDED) {
    RTCOccludedArguments args;
    rtcInitOccludedArguments(&args);
    args.flags = (RTCRayQueryFlags)L.flags; args.feature_mask = (RTCFeatureFlags)L.feature_mask;
    args.context = L.with_ctx ? &c.base : nullptr; args.filter = pick(L.which);
    rtcb200TraversableOccluded1<RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS>(t, static_cast<RTCRay*>(recs) + i, &args);
  } else {
    RTCIntersectArguments args;
    rtcInitIntersectArguments(&args);
    args.flags = (RTCRayQueryFlags)L.flags; args.feature_mask = (RTCFeatureFlags)L.feature_mask;
    args.context = L.with_ctx ? &c.base : nullptr; args.filter = pick(L.which);
    rtcb200TraversableIntersect1<RTC_FEATURE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS>(t, static_cast<RTCRayHit*>(recs) + i, &args);
  }
  if (L.T_out) { L.T_out[3 * i] = c.T[0]; L.T_out[3 * i + 1] = c.T[1]; L.T_out[3 * i + 2] = c.T[2]; }
  if (L.ctx_after) { L.ctx_after[2 * i] = c.base.instID[0]; L.ctx_after[2 * i + 1] = c.base.instPrimID[0]; }
}

unsigned blocks_for(size_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// host callbacks: lane l of field f of an SoA block of N lanes
inline uint32_t& word(void* p, unsigned N, int f, unsigned l) { return static_cast<uint32_t*>(p)[(size_t)f * N + l]; }
inline float& fword(void* p, unsigned N, int f, unsigned l) { return reinterpret_cast<float*>(static_cast<uint32_t*>(p))[(size_t)f * N + l]; }
float* g_host_T_by_id = nullptr;

}  // namespace

extern "C" {

int devfilter_query(const RTCB200DeviceTraversable* t, int occluded, void* d_recs, size_t n, int which, unsigned flags, unsigned feature_mask,
                    int with_ctx, unsigned seedI, unsigned seedP, void* d_rec, unsigned* d_rec_count, unsigned rec_cap, float* d_T_out,
                    float* d_T_by_id, unsigned* d_ctx_after, void* stream) {
  if (n == 0) return 0;
  cudaSetDevice(t->device);
  const Launch L{which, flags, feature_mask, with_ctx, seedI, seedP, static_cast<Record*>(d_rec), d_rec_count, rec_cap, d_T_out, d_T_by_id, d_ctx_after};
  if (occluded) filter_kernel<true><<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_recs, n, L);
  else filter_kernel<false><<<blocks_for(n), kThreads, 0, (cudaStream_t)stream>>>(*t, d_recs, n, L);
  return (int)cudaGetLastError();
}

// the rule, the hit-editing rule and the per-id hair filter as host callbacks (any N; the library calls them with N == 1)
void devfilter_host_rule(const RTCFilterFunctionNArguments* a) {
  for (unsigned l = 0; l < a->N; ++l)
    if (a->valid[l] == -1 && rejects(word(a->hit, a->N, 6, l), word(a->hit, a->N, 5, l), word(a->hit, a->N, 7, l))) a->valid[l] = 0;
}
void devfilter_host_edit(const RTCFilterFunctionNArguments* a) {
  const unsigned N = a->N;
  for (unsigned l = 0; l < N; ++l) {
    if (a->valid[l] != -1) continue;
    if (rejects(word(a->hit, N, 6, l), word(a->hit, N, 5, l), word(a->hit, N, 7, l))) { a->valid[l] = 0; continue; }
    edit_hit(fword(a->hit, N, 0, l), fword(a->hit, N, 1, l), fword(a->hit, N, 2, l), fword(a->hit, N, 3, l), fword(a->hit, N, 4, l),
             word(a->hit, N, 5, l), word(a->hit, N, 8, l));
  }
}
void devfilter_host_tfar(const RTCFilterFunctionNArguments* a) {
  for (unsigned l = 0; l < a->N; ++l) {
    if (a->valid[l] != -1) continue;
    if (rejects(word(a->hit, a->N, 6, l), word(a->hit, a->N, 5, l), word(a->hit, a->N, 7, l))) { a->valid[l] = 0; continue; }
    fword(a->ray, a->N, 8, l) = nextafterf(fword(a->ray, a->N, 8, l), 0.0f);
  }
}
void devfilter_host_hair_id(const RTCFilterFunctionNArguments* a) {
  for (unsigned l = 0; l < a->N; ++l) {
    if (a->valid[l] == 0) continue;
    float* Tp = g_host_T_by_id + 3 * (size_t)word(a->ray, a->N, 10, l);
    float T[3];
    for (int k = 0; k < 3; ++k) { T[k] = hair_kt(k) * Tp[k]; Tp[k] = T[k]; }
    if (fmaxf(T[0], fmaxf(T[1], T[2])) > 0.02f) a->valid[l] = 0;
  }
}
void devfilter_set_host_T_by_id(float* T) { g_host_T_by_id = T; }
int devfilter_record_words() { return (int)(sizeof(Record) / 4); }

}  // extern "C"
