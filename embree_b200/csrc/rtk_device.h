// rtk_device.h -- internal interface between the host shim (rtcore_shim.cpp) and the CUDA code
// (build.cu, trace.cu).  Plain structs and status codes only; no exceptions cross this boundary.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "rt_core.cuh"

namespace rtk {

// what the leaf records of a GeomDesc are and which test they take (build.cu primref_gen / leaf_pack, trace.cu curve_record_test)
enum PrimKind : uint32_t {
  PRIM_TRIANGLE = 0,        // triangle or quad mesh (a quad is stored as two triangle records)
  PRIM_ROUND_LINEAR = 1,    // cone-sphere segment
  PRIM_FLAT_LINEAR = 2,     // ray-facing ribbon segment
  PRIM_FLAT_CUBIC = 3,      // tessellated ribbon, one record per segment
  PRIM_ROUND_CUBIC = 4,     // sweep, one record per first-level sub-segment
  PRIM_SPHERE = 5,          // point kinds: point_test's point type is kind - PRIM_SPHERE
  PRIM_DISC = 6,            // ray-facing disc
  PRIM_ORIENTED_DISC = 7,   // disc with a normal (in `tangents`, stride `tstride`)
};
// The kernels write `kind >= PRIM_SPHERE` out instead of calling point_record: even inlined, the call changes how the compiler lays
// out their if-chains over the kinds.
RT_HD constexpr bool curve_record(uint32_t kind) { return kind >= PRIM_ROUND_LINEAR && kind <= PRIM_ROUND_CUBIC; }
RT_HD constexpr bool point_record(uint32_t kind) { return kind >= PRIM_SPHERE; }   // PRIM_ORIENTED_DISC is the last kind

// one enabled triangle mesh, buffers already resident on the device (raw bytes, caller's stride honoured:
// kernels/common/buffer.h BufferView semantics)
struct GeomDesc {
  const uint8_t* verts;  // first vertex (byteOffset applied)
  const uint8_t* idx;    // first index triple
  uint64_t vstride, istride;
  uint32_t nverts, ntris;   // ntris = 2 * quads for a quad mesh (each half is one record)
  uint32_t geomID, mask;
  // instancing (RTC_GEOMETRY_TYPE_INSTANCE, flattened at commit): this mesh is seen through the instance transform
  // xfm = (vx | vy | vz | p) columns of local2world (places the triangles in the world-space BVH), w2l its inverse
  // (takes the ray to the object-space triangle records); hits report instID and must also pass inst_mask.
  uint32_t has_xfm = 0, instID = 0xFFFFFFFFu, inst_mask = 0xFFFFFFFFu, skip_bounds = 0;
  // quad mesh (RTC_GEOMETRY_TYPE_QUAD): idx holds 4 indices per primitive; local prim 2q / 2q+1 are the halves
  // (v0,v1,v3) / (v2,v1,v3) of quad q exactly as quad_intersector_moeller.h:190-200 splits them.
  uint32_t is_quad = 0;
  // round linear curves (RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE): verts = float4 (xyz, radius), idx = first vertex of each
  // segment, ntris = segments; `flags` = one neighbour-flag byte per segment (device).  The vertex buffer stays resident
  // after the build: the trace kernel fetches the neighbour vertices from it.
  uint32_t kind = PRIM_TRIANGLE;   // PrimKind of the records
  const uint8_t* flags = nullptr;
  // flat cubic curves (RTC_GEOMETRY_TYPE_FLAT_BEZIER / _BSPLINE / _CATMULL_ROM / _HERMITE_CURVE): idx = first of the four
  // control vertices (Hermite: of the two vertex / tangent pairs), `basis` = rt_core.cuh CurveBasis of the control points,
  // `tess` = tessellation rate N, `basis_tab` = device table [8][N + 1] of the basis / derivative weights at u = j / N,
  // `tangents` = the resident float4 tangent buffer of a Hermite geometry (converted to Bezier control points on load).
  uint32_t basis = 0, tess = 4, hermite = 0;
  const float* basis_tab = nullptr;
  const uint8_t* tangents = nullptr;
  uint64_t tstride = 0;
  float xfm[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
  float w2l[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
};

#if defined(__CUDACC__)
// the four control points of the flat cubic curve whose index-buffer entry is `vid` (CurveGeometry::gather,
// scene_curves.h:107-113; Hermite: HermiteCurveT's conversion to Bezier control points, hermite_curve.h:19-20)
__device__ __forceinline__ void load_cubic_cp(const GeomDesc& g, uint32_t vid, CurveVtx cp[4]) {
  if (g.hermite) {
    const float4 p0 = __ldg(reinterpret_cast<const float4*>(g.verts + (size_t)vid * g.vstride));
    const float4 p1 = __ldg(reinterpret_cast<const float4*>(g.verts + (size_t)(vid + 1) * g.vstride));
    const float4 t0 = __ldg(reinterpret_cast<const float4*>(g.tangents + (size_t)vid * g.tstride));
    const float4 t1 = __ldg(reinterpret_cast<const float4*>(g.tangents + (size_t)(vid + 1) * g.tstride));
    const float k = 1.0f / 3.0f;
    cp[0] = CurveVtx{p0.x, p0.y, p0.z, p0.w};
    cp[1] = CurveVtx{fma_rn(k, t0.x, p0.x), fma_rn(k, t0.y, p0.y), fma_rn(k, t0.z, p0.z), fma_rn(k, t0.w, p0.w)};
    cp[2] = CurveVtx{fma_rn(-k, t1.x, p1.x), fma_rn(-k, t1.y, p1.y), fma_rn(-k, t1.z, p1.z), fma_rn(-k, t1.w, p1.w)};
    cp[3] = CurveVtx{p1.x, p1.y, p1.z, p1.w};
    return;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(g.verts + (size_t)(vid + k) * g.vstride));
    cp[k] = CurveVtx{q.x, q.y, q.z, q.w};
  }
}
#endif

enum BuilderKind : uint32_t { BUILDER_LBVH = 0, BUILDER_SAH = 1 };

struct SceneGPU {
  int device = 0;
  Node8* nodes = nullptr;
  TriRec* tris = nullptr;
  uint32_t num_nodes = 0, num_tris = 0;
  uint32_t root_valid = 0;              // 0: empty scene -> queries return immediately
  int robust = 0;                       // RTC_SCENE_FLAG_ROBUST: leaf records are (v0, v1, v2), Pluecker intersector
  int general = 0;                      // scene has instances, quads or curves: records carry a descriptor index instead of geomID
  int curves = 0;                       // scene has curve or point records: 2 curve records among them, 1 point records only
  GeomDesc* d_descs = nullptr;          // device copy of the mesh descriptors (kept while general)
  uint32_t num_descs = 0;               // entries of d_descs
  float bounds[6] = {0, 0, 0, 0, 0, 0};  // lower xyz, upper xyz of all valid triangles (world space, instances flattened)
  float api_bounds[6] = {0, 0, 0, 0, 0, 0};  // the same without instanced triangles
  double build_ms = 0, sah_cost = 0;
  uint32_t builder = 0, max_depth = 0;
  unsigned long long* d_stat = nullptr;  // [3] rays, nodes, tris (device)
  size_t node_capacity = 0, tri_capacity = 0;
  // kept by build_scene for refit_scene: record -> global primitive index, number of primitives (valid or not) the
  // scene was built from, and the node id where every BVH8 level starts (levels[l] .. levels[l+1])
  uint32_t* tri_src = nullptr;
  uint32_t total_prims = 0;
  std::vector<uint32_t> levels;
  // two-level assembly (assemble_scene): where each sub-BVH lives in the arrays, its counts at layout time, its (relocated) root node
  std::vector<uint32_t> sub_node_off, sub_tri_off, sub_nodes, sub_tris;
  std::vector<Node8> sub_root;
  std::vector<const void*> sub_id;      // which sub-BVH object occupies each slot (a different one there is copied even if the counts match)
  uint32_t top_cap = 0;                 // nodes reserved at the start of the array for the top level
  bool is_sub = false;                  // a per-mesh BVH of a two-level scene: never traced on its own (no stat counters)
};

// ---- two-level scenes (kernels/bvh/bvh_builder_twolevel.cpp:35-240: dynamic scenes keep one BVH per mesh and rebuild only what
// changed).  Every mesh is built on its own (build_scene / refit_scene on a one-mesh SceneGPU, kept by the host shim); assemble_scene
// places the sub-BVHs in ONE node / record array -- node and record indices relocated by the mesh's offsets -- under a small top-level
// BVH8 built on the host over the mesh boxes, whose lowest nodes hold COPIES of the meshes' root nodes (children of a node must be
// consecutive), so the trace kernel runs unchanged.  `dirty[i]`: sub i was rebuilt / refitted since the last assembly.  The layout
// is reused while every sub keeps its node and record counts (then only dirty subs are copied again); otherwise everything is laid out anew.
int assemble_scene(SceneGPU& top, SceneGPU* const* subs, int nsubs, const uint8_t* dirty, cudaStream_t stream, char* errmsg);

// Build the BVH8 over `ngeoms` meshes.  Returns cudaSuccess (0) or a CUDA error code; `errmsg` (>=256 B) gets text.
int build_scene(SceneGPU& s, const GeomDesc* geoms, int ngeoms, BuilderKind kind, cudaStream_t stream, char* errmsg);
// Refit the committed BVH to moved vertices (same meshes, same primitive counts, no instances); s.builder becomes 2.
int refit_scene(SceneGPU& s, const GeomDesc* geoms, int ngeoms, cudaStream_t stream, char* errmsg);
void free_scene(SceneGPU& s);

struct TraceParams {
  const Node8* nodes;
  const TriRec* tris;
  uint32_t root_valid;
  void* rays;            // RTCRayHit[] / RTCRay[] / RTCRayHitK[] / RTCRayK[]  (device-accessible)
  const int* valid;      // per lane, -1 active; NULL = all active (always NULL for K == 1)
  unsigned long long n;  // number of rays = records * K
  uint32_t instID, instPrimID;
  unsigned long long* stat;  // non-NULL -> counting kernel
  // optional second output (K == 1 closest-hit only): one 32-byte record per ray {tfar, Ng.xyz, u, v, primID, geomID}
  // written when the ray terminates.  May point into a PEER GPU's memory (NVLink): this is how the multi-GPU
  // hit gather is fused into the trace kernel instead of being a separate collective.
  void* compact_out = nullptr;
  void* stage = nullptr;   // gather mode 1: local staging buffer with the same indexing (n x 32 B)
  int tri_batch_min = 8, tri_wait_max = 4, refill_min = 4, use_prefetch = 1;  // filled by launch_trace from tuning()
  const GeomDesc* descs = nullptr;  // non-NULL: instanced scene, record.geomID slot holds a descriptor index
  int curves = 0;                   // the scene holds curve or point records (descs != NULL): 2 curves among them, 1 points only
  uint32_t top_nodes = 0;           // nodes in the first three BVH8 levels (RTK_TOP_SMEM experiment)
  int robust = 0;  // scene built with RTC_SCENE_FLAG_ROBUST: triangle records hold v0,v1,v2, Pluecker test
  // filter-callback passes (K == 1 closest hit): per-ray lists of rejected record indices (excl_off has n + 1 entries) and
  // the per-ray output of the winning record index (0xFFFFFFFF on a miss)
  const uint32_t* excl_off = nullptr;
  const uint32_t* excl_idx = nullptr;
  uint32_t* win = nullptr;
};
// occluded: 0 = closest hit (rtcIntersect*), 1 = any hit (rtcOccluded*); K in {1,4,8,16}
int launch_trace(const TraceParams& p, int occluded, int K, cudaStream_t stream);

// run-time tuning knobs (defaults = shipped configuration; overridable through rtcb200SetTuning / RTCB200_* env)
struct Tuning {
  int collapse_policy = 3;   // 0/1/2 greedy variants (rt_core.cuh select_children), 3 = SAH-optimal dynamic programme
  int c_node = 100, c_tri = 50;  // DP cost of a BVH8 node visit / a triangle test, in 1/100
  int tri_batch_min = 8;     // triangle step when >= this many lanes have triangles pending (or no lane has a node, or after tri_wait_max deferrals)
  int tri_wait_max = 4;
  // the same two keys for scenes with curve records: a curve test costs 10-100x a triangle test, so it pays to wait until more
  // lanes have one pending (scripts/hair_tune.py sweeps both on the fur ball of bench.py); scenes of points only take their own
  // pair.  Curve scenes also run with fewer CTAs per SM (curve_blocks_per_sm).
  int curve_batch_min = 32, curve_wait_max = 24;
  int point_batch_min = 24, point_wait_max = 16;
  int blocks_per_sm = 8;
  int curve_blocks_per_sm = 6;
  int use_tma = 1;
  int refill_min = 4;
  int gather_mode = 1;       // fused hit gather: 0 = one 32-byte store per record, 1 = blocks staged in shared memory, 1 KB stores
  int tri_spread = 1;        // warp-wide triangle redistribution in the trace kernel (trace.cu SPREAD; closest-hit triangle scenes)
  int tri_spread_occluded = 1;   // the same redistribution in the any-hit kernels (a hit ends the owner's ray)
  int sah_small = 4;         // SAH builder: segments of <= this many primitives are split in the middle (no binning)
};
Tuning& tuning();

void set_pool_keep_bytes(unsigned long long bytes);   // release threshold of the stream-ordered pool the builds allocate from
unsigned long long launch_count();
void count_launch(unsigned n = 1);

}  // namespace rtk
