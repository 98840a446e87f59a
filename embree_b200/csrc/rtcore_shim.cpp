// rtcore_shim.cpp -- host side of the drop-in boundary: the Embree 4 object model (device / buffer / geometry /
// scene handles, reference counts, the sticky-first-error convention, the geometry commit state machine) and the
// extern "C" rtc* entry points declared in include/embree4_b200.h, in front of the CUDA code in build.cu / trace.cu.
//
// Mirrors (reference paths): kernels/common/rtcore.cpp (entry points), rtcore.h:23-74 (error funnel),
// device.cpp:263-330 (error slots), geometry.cpp:97-135 (modCounter / MODIFIED / COMMITTED),
// scene_triangle_mesh.cpp:35-147 (buffer validation), scene.cpp:762-1040 + scene_verify.cpp:11-22 (commit),
// buffer.h:16-97 (shared vs owned memory).  There is NO CPU traversal or build in this file or anywhere in the
// library: if CUDA is unavailable, rtcNewDevice fails with RTC_ERROR_UNKNOWN and returns NULL.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/embree4_b200.h"
#include "interp.cuh"
#include "rtk_device.h"
#include "transform_format.cuh"

namespace {

struct ApiError {
  RTCError code;
  std::string msg;
};
[[noreturn]] void fail(RTCError c, const char* m) { throw ApiError{c, m}; }

struct ErrSlot {
  RTCError code = RTC_ERROR_NONE;
  std::string msg;
};

struct DeviceImpl;
thread_local ErrSlot t_noDeviceError;                               // errors with no device (device.cpp:288-310)
thread_local std::unordered_map<const DeviceImpl*, ErrSlot> t_err;  // per device, per thread (device.cpp:263-286)

struct RefCounted {
  std::atomic<long> rc{1};
  virtual ~RefCounted() {}
  void retain() { rc.fetch_add(1); }
  void release() { if (rc.fetch_sub(1) == 1) delete this; }
};

std::mutex g_deviceMutex;  // device create/retain/release take a global lock (rtcore.cpp:17,23)

struct DeviceImpl : RefCounted {
  int gpu = 0;
  int verbose = 0;
  RTCErrorFunction errFn = nullptr;
  void* errPtr = nullptr;
  RTCMemoryMonitorFunction memFn = nullptr;
  void* memPtr = nullptr;
  cudaDeviceProp prop{};
  void report(RTCError code, const char* msg) {
    if (verbose >= 1) fprintf(stderr, "Embree(b200): %s, (%s)\n", rtcGetErrorString(code), msg ? msg : "");
    if (errFn) errFn(errPtr, code, msg);
    ErrSlot& s = t_err[this];
    if (s.code == RTC_ERROR_NONE) { s.code = code; if (msg && *msg) s.msg = msg; }
  }
  void use() const { cudaSetDevice(gpu); }
};

void process_error(DeviceImpl* d, RTCError code, const char* msg) {
  if (!d) {
    if (t_noDeviceError.code == RTC_ERROR_NONE) { t_noDeviceError.code = code; if (msg && *msg) t_noDeviceError.msg = msg; }
    return;
  }
  d->report(code, msg);
}

#define API_BEGIN try {
#define API_END(dev)                                                                     \
  }                                                                                      \
  catch (std::bad_alloc&) { process_error(dev, RTC_ERROR_OUT_OF_MEMORY, "out of memory"); } \
  catch (ApiError & e) { process_error(dev, e.code, e.msg.c_str()); }                    \
  catch (std::exception & e) { process_error(dev, RTC_ERROR_UNKNOWN, e.what()); }        \
  catch (...) { process_error(dev, RTC_ERROR_UNKNOWN, "unknown exception caught"); }
#define VERIFY_HANDLE(h) if ((h) == nullptr) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid argument")

void cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    char buf[256];
    snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(e));
    if (e == cudaErrorMemoryAllocation) fail(RTC_ERROR_OUT_OF_MEMORY, buf);
    fail(RTC_ERROR_UNKNOWN, buf);
  }
}

struct BufferImpl : RefCounted {
  DeviceImpl* dev;
  char* ptr = nullptr;
  size_t bytes = 0;
  bool shared = false;
  bool device = false;   // rtcb200SetSharedGeometryBufferDevice: `ptr` is the caller's memory on the library's GPU, not the host's
  BufferImpl(DeviceImpl* d, size_t n, void* user) : dev(d), bytes(n), shared(user != nullptr) {
    dev->retain();
    if (user) ptr = static_cast<char*>(user);
    else {
      const size_t padded = (n + 15) & ~size_t(15);  // owned memory is 16-byte rounded (buffer.h:29-30)
      if (posix_memalign(reinterpret_cast<void**>(&ptr), 64, padded ? padded : 16) != 0) throw std::bad_alloc();
      memset(ptr, 0, padded ? padded : 16);
    }
  }
  ~BufferImpl() override {
    if (!shared) free(ptr);
    dev->release();
  }
};

struct BufferView {
  BufferImpl* buf = nullptr;
  size_t offset = 0, stride = 0, count = 0;
  RTCFormat format = RTC_FORMAT_UNDEFINED;
  void set(BufferImpl* b, size_t off, size_t st, size_t n, RTCFormat f) {
    if (b) b->retain();
    if (buf) buf->release();
    buf = b; offset = off; stride = st; count = n; format = f;
  }
  const char* data() const { return buf && buf->ptr ? buf->ptr + offset : nullptr; }   // NULL: an empty device view
  bool on_device() const { return buf && buf->device; }
  // how a device copy of the view's bytes is made
  cudaMemcpyKind copy_kind() const { return on_device() ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice; }
  ~BufferView() { if (buf) buf->release(); }
};

enum class GeomState { MODIFIED, COMMITTED };
// The record kind a geometry type is built into and, for a cubic curve, the basis of its control points (a Hermite curve is converted
// to Bezier control points on load).  Triangles, quads, instances and the types this back-end does not support answer PRIM_TRIANGLE.
struct PrimType { rtk::PrimKind kind; rtk::CurveBasis basis; };
PrimType prim_type(RTCGeometryType t) {
  switch (t) {
    case RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE: return {rtk::PRIM_ROUND_LINEAR, rtk::BASIS_BEZIER};
    case RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE: return {rtk::PRIM_FLAT_LINEAR, rtk::BASIS_BEZIER};
    case RTC_GEOMETRY_TYPE_FLAT_BEZIER_CURVE: case RTC_GEOMETRY_TYPE_FLAT_HERMITE_CURVE: return {rtk::PRIM_FLAT_CUBIC, rtk::BASIS_BEZIER};
    case RTC_GEOMETRY_TYPE_FLAT_BSPLINE_CURVE: return {rtk::PRIM_FLAT_CUBIC, rtk::BASIS_BSPLINE};
    case RTC_GEOMETRY_TYPE_FLAT_CATMULL_ROM_CURVE: return {rtk::PRIM_FLAT_CUBIC, rtk::BASIS_CATMULL_ROM};
    case RTC_GEOMETRY_TYPE_ROUND_BEZIER_CURVE: case RTC_GEOMETRY_TYPE_ROUND_HERMITE_CURVE: return {rtk::PRIM_ROUND_CUBIC, rtk::BASIS_BEZIER};
    case RTC_GEOMETRY_TYPE_ROUND_BSPLINE_CURVE: return {rtk::PRIM_ROUND_CUBIC, rtk::BASIS_BSPLINE};
    case RTC_GEOMETRY_TYPE_ROUND_CATMULL_ROM_CURVE: return {rtk::PRIM_ROUND_CUBIC, rtk::BASIS_CATMULL_ROM};
    case RTC_GEOMETRY_TYPE_SPHERE_POINT: return {rtk::PRIM_SPHERE, rtk::BASIS_BEZIER};
    case RTC_GEOMETRY_TYPE_DISC_POINT: return {rtk::PRIM_DISC, rtk::BASIS_BEZIER};
    case RTC_GEOMETRY_TYPE_ORIENTED_DISC_POINT: return {rtk::PRIM_ORIENTED_DISC, rtk::BASIS_BEZIER};
    default: return {rtk::PRIM_TRIANGLE, rtk::BASIS_BEZIER};
  }
}
bool curve_geometry(RTCGeometryType t) { return rtk::curve_record(prim_type(t).kind); }
bool is_linear_curve(RTCGeometryType t) { const rtk::PrimKind k = prim_type(t).kind; return k == rtk::PRIM_ROUND_LINEAR || k == rtk::PRIM_FLAT_LINEAR; }
bool point_geometry(RTCGeometryType t) { return rtk::point_record(prim_type(t).kind); }
bool is_hermite(RTCGeometryType t) { return t == RTC_GEOMETRY_TYPE_FLAT_HERMITE_CURVE || t == RTC_GEOMETRY_TYPE_ROUND_HERMITE_CURVE; }
// number of live geometries that have a filter callback or accept the arguments' filter: while it is zero (and the
// query carries no filter) no query looks at the geometries at all
std::atomic<long> g_filterGeoms{0};

struct SceneImpl;
void release_scene_ref(SceneImpl* s);
// frees `bufs` on `st`, after the work enqueued there that may still read them
void release_buffers(std::vector<void*>& bufs, cudaStream_t st) {
  for (void* p : bufs) cudaFreeAsync(p, st);
  bufs.clear();
}

struct GeometryImpl : RefCounted {
  DeviceImpl* dev;
  RTCGeometryType type = RTC_GEOMETRY_TYPE_TRIANGLE;
  SceneImpl* instScene = nullptr;                       // RTC_GEOMETRY_TYPE_INSTANCE: the instanced scene (retained)
  float xfm[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};  // local2world columns vx | vy | vz | p (AffineSpace3fa)
  float w2l[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};  // world2local0 = rcp(local2world) (scene_instance.cpp:153)
  void update_world2local();
  BufferView vertices, indices, flags;   // flags: RTC_BUFFER_TYPE_FLAGS of a curve geometry (optional)
  BufferView tangents;                   // RTC_BUFFER_TYPE_TANGENT of a Hermite curve geometry
  int tessellationRate = 4;              // flat cubic curves (scene_curves.cpp:27,247)
  std::vector<BufferView> attribs;
  unsigned mask = 1;  // reference default (geometry.cpp:48)
  bool enabled = true;
  RTCBuildQuality quality = RTC_BUILD_QUALITY_MEDIUM;
  void* userPtr = nullptr;
  // filter callbacks (geometry.h:269-270,481-482; geometry.cpp:142-156): host functions, run by trace_filtered()
  RTCFilterFunctionN intersectFilter = nullptr, occludedFilter = nullptr;
  bool argFilterEnabled = false;
  GeomState state = GeomState::MODIFIED;
  unsigned modCounter = 1;
  // bumped by every set or update of the index buffer: a REFIT keeps the primitives that were valid at the last build, so new
  // indices must rebuild (the reference refits only while the index buffer's version is unchanged: bvh_refit.cpp:184-192,
  // scene_triangle_mesh.h:261-263)
  unsigned indexVersion = 0;
  // identity that survives address reuse: caches keyed by the GeometryImpl* (kept per-mesh BVHs, the refit topology) compare it, because a
  // geometry released and another one allocated at the same address with the same modCounter must not be taken for the old one
  static std::atomic<unsigned long long>& serial_source() { static std::atomic<unsigned long long> n{0}; return n; }
  const unsigned long long serial = serial_source().fetch_add(1) + 1;
  explicit GeometryImpl(DeviceImpl* d) : dev(d) { dev->retain(); }
  ~GeometryImpl() override { if (has_filter()) g_filterGeoms.fetch_sub(1); if (instScene) release_scene_ref(instScene); dev->release(); }
  bool has_filter() const { return intersectFilter || occludedFilter || argFilterEnabled; }
  template <typename F> void set_filter(F&& change) {
    const bool before = has_filter();
    change();
    const bool after = has_filter();
    if (after != before) g_filterGeoms.fetch_add(after ? 1 : -1);
  }
  void update() { ++modCounter; state = GeomState::MODIFIED; }  // geometry.cpp:97-101
};

struct SceneImpl : RefCounted {
  DeviceImpl* dev;
  std::mutex geomMutex;     // attach/detach are thread safe (README.md:921-924)
  std::mutex commitMutex;
  std::vector<GeometryImpl*> geoms;      // index == geomID
  std::vector<unsigned> committedCounter;  // modCounter snapshot of the last commit (scene.cpp:878-884)
  // Instances are flattened into this scene's BVH at commit, so a re-committed CHILD scene must make the parent's next
  // rtcCommitScene rebuild (the reference traverses the child BVH live and sees child edits without this): every
  // successful commit bumps `generation`, and the parent remembers the generation of each instanced scene it baked in.
  std::atomic<unsigned long long> generation{0};
  std::vector<unsigned long long> committedChildGen;
  // topology signature of the last full build (geometry, geomID, primitive / vertex counts, index buffer version): a later commit whose enabled
  // geometries all ask for RTC_BUILD_QUALITY_REFIT and match it refits the BVH instead of rebuilding (bvh_refit.cpp)
  // (the geomID too: a refit keeps the descriptor table of the build, which maps the records of quads and curves to their geomIDs)
  struct TopoEntry {
    GeometryImpl* g; unsigned geomID; size_t nprims, nverts; unsigned long long serial; unsigned indexVersion;
    bool operator==(const TopoEntry& o) const {
      return g == o.g && geomID == o.geomID && nprims == o.nprims && nverts == o.nverts && serial == o.serial && indexVersion == o.indexVersion;
    }
  };
  std::vector<TopoEntry> builtTopology;
  RTCBuildQuality builtQuality = RTC_BUILD_QUALITY_MEDIUM;
  RTCSceneFlags builtFlags = RTC_SCENE_FLAG_NONE;
  RTCSceneFlags flags = RTC_SCENE_FLAG_NONE;
  RTCBuildQuality quality = RTC_BUILD_QUALITY_MEDIUM;
  bool flagsModified = true;  // forces the first commit (scene_verify.cpp:11-22 isModified())
  bool everCommitted = false;
  RTCProgressMonitorFunction progFn = nullptr;
  void* progPtr = nullptr;
  rtk::SceneGPU gpu;
  float apiBounds[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};  // what rtcGetSceneBounds reports
  std::vector<void*> deviceBuffers;  // uploaded vertex/index bytes of the current commit
  std::vector<void*> residentBuffers;  // curve vertex buffers: read by the trace kernel, live until the next commit
  // which of them hold a curve geometry's vertices and (Hermite) tangents: batched interpolation reads them instead of a second copy
  struct CurveCopy { const uint8_t* verts = nullptr; const uint8_t* tangents = nullptr; };
  std::unordered_map<const GeometryImpl*, CurveCopy> residentCurves;
  // batched interpolation (rtcb200InterpolateHits*): one table per (buffer type, slot) asked for since the last commit and the device
  // copies of the buffers it reads; built by the first call that needs it, freed by the next commit and with the scene
  struct InterpTable { RTCBufferType type; unsigned slot; rtk::InterpEntry* d_table; uint32_t nentries; std::vector<void*> buffers; };
  std::vector<InterpTable> interpTables;
  // device-side argument filters and shading getters (rtcb200GetSceneDeviceTraversable): (geomID, instID or invalid) of every
  // descriptor of the last commit, and the geometry snapshots the getter uploaded since then (geometry_snapshot: header,
  // per-record table, per-geomID block in one allocation) with the bytes of the newest after its header -- reused while they are
  // unchanged; the next commit frees them all, and so does releasing the scene
  std::vector<std::pair<uint32_t, uint32_t>> descIds;
  std::vector<void*> geomTables;
  std::vector<unsigned char> lastGeomTable;
  void free_geom_tables(cudaStream_t st) {
    release_buffers(geomTables, st);
    lastGeomTable.clear();
  }
  void free_interp(cudaStream_t st) {
    for (InterpTable& t : interpTables) {
      cudaFreeAsync(t.d_table, st);
      release_buffers(t.buffers, st);
    }
    interpTables.clear();
  }
  // BVHs kept across commits, rebuilt only when what they were built from changed (taken and put back by KeptBvhs):
  // - two-level scenes (RTC_SCENE_FLAG_DYNAMIC with several triangle meshes; bvh_builder_twolevel.cpp:35-240): one per mesh, rebuilt
  //   or refitted only when that mesh's modCounter moved (scene.cpp:878-884, bvh_builder_twolevel.h:174-177).  Keyed by (geometry,
  //   geomID): the records hold the geomID, and attaching under another ID leaves modCounter alone, so a geometry moved to another ID,
  //   or attached under two, gets a BVH of its own per ID (the reference keys its builders by objectID and drops them on detach:
  //   bvh_builder_twolevel.cpp:80-106,230,287-306, scene.cpp:743-760).
  // - instance traversal (commit_instanced): one per instanced scene, keyed by (scene, 0), built by this scene with its own flags and
  //   quality from the instanced scene's geometries, and kept while that scene's generation is the same.  The entry holds a reference
  //   to the instanced scene (so its address names it while the entry lives) and the device buffers the trace kernel reads through
  //   the BVH's descriptors (curve vertices, basis tables).
  // Either is also rebuilt when this scene's ROBUST flag or quality changed.
  struct KeptBvh {
    rtk::SceneGPU gpu;
    RTCBuildQuality sceneQuality = RTC_BUILD_QUALITY_MEDIUM; int robust = 0;
    // the mesh it was built from: GeometryImpl::serial (0: none yet), modCounter, index buffer version and counts
    unsigned long long serial = 0; unsigned modCounter = 0, indexVersion = 0; size_t nprims = 0, nverts = 0;
    // the instanced scene and the generation it was built from (~0: none yet), the BVH's descriptors and the buffers they point at
    SceneImpl* scene = nullptr; unsigned long long generation = ~0ull;
    std::vector<rtk::GeomDesc> descs;
    std::vector<void*> resident;
    std::unordered_map<const GeometryImpl*, CurveCopy> curves;
    void release(cudaStream_t st);   // frees the BVH and the buffers on `st`
    ~KeptBvh();
  };
  using KeptMap = std::map<std::pair<const void*, unsigned>, std::unique_ptr<KeptBvh>>;
  KeptMap meshBvhs, sceneBvhs;
  bool statCounters = false;
  double lastTraceMs = -1.0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // Commits on a stream (rtcb200CommitSceneWithStream): `committed` is recorded on the commit stream when a commit has enqueued its
  // work.  While `pending`, that work may still run: the library's streams and a Device call's stream wait for the event on the
  // device (wait_on), readers on the host wait for it and take what the commit left for them (settle).  A refit that did not wait
  // left its root box and time in refitStaging[lastRefit]; the other blocks may still be read by earlier refits on the device.
  cudaEvent_t committed = nullptr;
  bool pending = false;
  std::vector<rtk::RefitStaging> refitStaging;
  int lastRefit = -1;
  explicit SceneImpl(DeviceImpl* d) : dev(d) { dev->retain(); gpu.device = d->gpu; }
  ~SceneImpl() override {
    dev->use();
    if (pending) cudaEventSynchronize(committed);
    for (GeometryImpl* g : geoms) if (g) g->release();
    release_buffers(deviceBuffers, 0);
    release_buffers(residentBuffers, 0);
    free_interp(0);
    free_geom_tables(0);
    meshBvhs.clear();
    sceneBvhs.clear();
    rtk::free_scene(gpu);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (committed) cudaEventDestroy(committed);
    for (rtk::RefitStaging& b : refitStaging) {
      cudaFreeHost(b.host);
      cudaEventDestroy(b.t0);
      cudaEventDestroy(b.t1);
    }
    dev->release();
  }
  void wait_on(cudaStream_t st) const {
    if (pending) cuda_check(cudaStreamWaitEvent(st, committed, 0), "wait for the stream commit");
  }
  void settle() {
    if (!pending) return;
    dev->use();
    cuda_check(cudaEventSynchronize(committed), "stream commit");
    if (lastRefit >= 0) {
      rtk::resolve_refit(gpu, refitStaging[lastRefit]);
      for (int a = 0; a < 6; ++a) apiBounds[a] = gpu.api_bounds[a];   // a refitted scene has no instances (set_api_bounds)
      lastRefit = -1;
    }
    pending = false;
  }
  // Keeps `blocks` staging blocks of at least `bytes` for refits that do not wait.  Called after a build, which waited anyway: a pinned
  // allocation may wait for the device.
  void reserve_refit_staging(size_t bytes, size_t blocks) {
    for (rtk::RefitStaging& b : refitStaging)
      if (b.cap < bytes) {
        cuda_check(cudaEventSynchronize(b.t1), "refit staging");
        cudaFreeHost(b.host); b.host = nullptr; b.cap = 0;
        cuda_check(cudaHostAlloc(&b.host, bytes, cudaHostAllocDefault), "cudaHostAlloc(refit staging)");
        b.cap = bytes;
      }
    while (refitStaging.size() < blocks) {
      rtk::RefitStaging b;
      cuda_check(cudaEventCreate(&b.t0), "cudaEventCreate");
      cuda_check(cudaEventCreate(&b.t1), "cudaEventCreate");
      cuda_check(cudaHostAlloc(&b.host, bytes, cudaHostAllocDefault), "cudaHostAlloc(refit staging)");
      b.cap = bytes;
      refitStaging.push_back(b);
    }
  }
  // a staging block of at least `bytes` that no refit on the device still reads, or -1 (the refit then waits).  A block whose results
  // settle() has not taken yet may be taken: the refit it serves replaces them.
  int free_refit_staging(size_t bytes) {
    for (size_t i = 0; i < refitStaging.size(); ++i)
      if (refitStaging[i].cap >= bytes && cudaEventQuery(refitStaging[i].t1) == cudaSuccess) return (int)i;
    return -1;
  }
  bool isModified() {
    if (flagsModified) return true;
    for (size_t i = 0; i < geoms.size(); ++i) {
      const unsigned cur = geoms[i] ? geoms[i]->modCounter : 0u;
      const unsigned old = i < committedCounter.size() ? committedCounter[i] : 0u;
      if (cur != old) return true;
      if (geoms[i] && geoms[i]->instScene) {
        const unsigned long long g = i < committedChildGen.size() ? committedChildGen[i] : ~0ull;
        if (geoms[i]->instScene->generation.load() != g) return true;
      }
    }
    return geoms.size() != committedCounter.size();
  }
};

void release_scene_ref(SceneImpl* s) { s->release(); }
void SceneImpl::KeptBvh::release(cudaStream_t st) {
  rtk::free_scene(gpu, st);
  release_buffers(resident, st);
}
SceneImpl::KeptBvh::~KeptBvh() {
  release(0);
  if (scene) scene->release();
}
// drops the kept BVHs of `m`, their memory freed on `st`
void clear_kept(SceneImpl::KeptMap& m, cudaStream_t st) {
  for (auto& kv : m) kv.second->release(st);
  m.clear();
}

// rcp(AffineSpace3fa) = (il, -(il * p)), il = adjoint / det (affinespace.h:83, linearspace3.h:44-51).  The reference runs
// this once per commit in its lowest-ISA (non-FMA) code, so the products below must stay unfused: volatile keeps a
// contracting host compiler from fusing them.
void GeometryImpl::update_world2local() {
  const float *vx = xfm, *vy = xfm + 3, *vz = xfm + 6, *p = xfm + 9;
  auto cross = [](const float* a, const float* b, float* o) {
    for (int i = 0; i < 3; ++i) {
      const int j = (i + 1) % 3, k = (i + 2) % 3;
      volatile float m0 = a[j] * b[k], m1 = a[k] * b[j];
      o[i] = m0 - m1;
    }
  };
  float c0[3], c1[3], c2[3];
  cross(vy, vz, c0); cross(vz, vx, c1); cross(vx, vy, c2);
  volatile float d0 = vx[0] * c0[0], d1 = vx[1] * c0[1], d2 = vx[2] * c0[2];
  volatile float d01 = d0 + d1;
  const float det = d01 + d2;
  for (int a = 0; a < 3; ++a) { w2l[3 * a] = c0[a] / det; w2l[3 * a + 1] = c1[a] / det; w2l[3 * a + 2] = c2[a] / det; }
  for (int a = 0; a < 3; ++a) {
    volatile float m0 = p[0] * w2l[a], m1 = p[1] * w2l[3 + a], m2 = p[2] * w2l[6 + a];
    volatile float s12 = m1 + m2;
    w2l[9 + a] = -(m0 + s12);
  }
}

DeviceImpl* D(RTCDevice h) { return reinterpret_cast<DeviceImpl*>(h); }
BufferImpl* B(RTCBuffer h) { return reinterpret_cast<BufferImpl*>(h); }
GeometryImpl* G(RTCGeometry h) { return reinterpret_cast<GeometryImpl*>(h); }
SceneImpl* S(RTCScene h) { return reinterpret_cast<SceneImpl*>(h); }

// "key=value,key=value" device configuration (state.cpp:263-457); unknown keys are accepted and ignored
void parse_config(DeviceImpl* d, const char* cfg) {
  if (!cfg) return;
  std::string s(cfg);
  size_t pos = 0;
  while (pos < s.size()) {
    size_t end = s.find_first_of(",; ", pos);
    if (end == std::string::npos) end = s.size();
    const std::string tok = s.substr(pos, end - pos);
    const size_t eq = tok.find('=');
    if (eq != std::string::npos) {
      const std::string k = tok.substr(0, eq), v = tok.substr(eq + 1);
      if (k == "verbose") d->verbose = atoi(v.c_str());
      else if (k == "gpu") d->gpu = atoi(v.c_str());
      else if (k == "pool_keep_mb") rtk::set_pool_keep_bytes((unsigned long long)atoll(v.c_str()) << 20);
    }
    pos = end + 1;
  }
}

// ---- commit: upload the enabled meshes and build on the device (scene.cpp:828-887) --------------------------

// The uploads of one commit: the descriptors the build takes and the device copies of the geometries' buffers.  A geometry instanced
// many times is uploaded once; every instance adds its own descriptor.
struct CommitUpload {
  SceneImpl* s;
  cudaStream_t st;   // the commit stream: allocations, copies and the flag kernel are enqueued there
  std::vector<rtk::GeomDesc> descs;
  std::unordered_map<GeometryImpl*, rtk::GeomDesc> uploaded;   // descriptor of every uploaded geometry, before geomID and instance
  // where buffers the trace kernel reads go, and which of them hold curve vertices: the scene's, or those of a kept instanced scene's BVH
  std::vector<void*>* resident;
  std::unordered_map<const GeometryImpl*, SceneImpl::CurveCopy>* curves;
  CommitUpload(SceneImpl* scene, cudaStream_t stream) : s(scene), st(stream), resident(&scene->residentBuffers), curves(&scene->residentCurves) {}

  // `bytes` of device memory (at least a 16-byte placeholder), freed right after the build or, `resident`, kept for the trace kernel
  // until the next commit
  uint8_t* alloc(size_t bytes, bool resident, const char* what) {
    void* p = nullptr;
    cuda_check(cudaMallocAsync(&p, bytes ? bytes : 16, st), (std::string("cudaMallocAsync(") + what + ")").c_str());
    (resident ? *this->resident : s->deviceBuffers).push_back(p);
    return static_cast<uint8_t*>(p);
  }
  // device copy of `bytes` at `src`, host memory or (`kind` device-to-device) the caller's device memory; the build reads the same
  // fresh allocation either way
  const uint8_t* copy(const void* src, size_t bytes, bool resident, const char* what, cudaMemcpyKind kind = cudaMemcpyHostToDevice) {
    uint8_t* p = alloc(bytes, resident, what);
    if (bytes) cuda_check(cudaMemcpyAsync(p, src, bytes, kind, st), (std::string("upload ") + what).c_str());
    return p;
  }
  const uint8_t* copy(const BufferView& v, size_t bytes, bool resident, const char* what) {
    return v.data() ? copy(v.data(), bytes, resident, what, v.copy_kind()) : alloc(bytes, resident, what);   // an empty device view: nothing to copy
  }

  // Adds the descriptor of `g` as `geomID`, seen through the instance `inst` (`instID` in its scene) when that is not null.  False when
  // `g` has no primitives.
  bool upload_geometry(GeometryImpl* g, uint32_t geomID, const GeometryImpl* inst = nullptr, uint32_t instID = RTC_INVALID_GEOMETRY_ID) {
    auto it = uploaded.find(g);
    if (it == uploaded.end()) {
      rtk::GeomDesc d{};
      if (!copy_geometry(g, d)) return false;
      it = uploaded.emplace(g, d).first;
    }
    rtk::GeomDesc d = it->second;
    d.geomID = geomID;
    // an instanced geometry: its records stay in OBJECT space (the trace kernel takes the ray there), the builder boxes them in world
    // space, the API bounds come from the instance box
    if (inst) {
      d.has_xfm = 1; d.instID = instID; d.inst_mask = inst->mask; d.skip_bounds = 1;
      memcpy(d.xfm, inst->xfm, sizeof d.xfm);
      memcpy(d.w2l, inst->w2l, sizeof d.w2l);
    }
    descs.push_back(d);
    return true;
  }

  // Validates `g` and uploads its buffers into `d`; false when it has no primitives.
  bool copy_geometry(GeometryImpl* g, rtk::GeomDesc& d) {
    const PrimType pt = prim_type(g->type);
    const size_t nverts = g->vertices.count, nprims = g->indices.count;
    d.kind = pt.kind; d.mask = g->mask;
    d.vstride = g->vertices.stride; d.istride = g->indices.stride; d.nverts = (uint32_t)nverts;
    if (rtk::point_record(pt.kind)) {
      // point primitives (scene_points.cpp): float4 vertices (centre, radius), one primitive per vertex; oriented discs carry one
      // float3 normal per vertex (GeomDesc.tangents / tstride hold that buffer).  They share the curve kernels (GENERAL == 2).
      if (nverts == 0 || !g->vertices.buf) return false;
      const bool oriented = pt.kind == rtk::PRIM_ORIENTED_DISC;
      if (oriented && !g->tangents.buf) fail(RTC_ERROR_INVALID_OPERATION, "normal buffer not set");
      if (oriented && g->tangents.count != nverts) fail(RTC_ERROR_INVALID_OPERATION, "number of normals must match number of vertices");
      if (nverts > 0x7FFFFFFFull) fail(RTC_ERROR_INVALID_OPERATION, "point geometry too large");
      d.verts = copy(g->vertices, (nverts - 1) * g->vertices.stride + 16, false, "point vertices");
      if (oriented) {
        d.tangents = copy(g->tangents, (nverts - 1) * g->tangents.stride + 12, false, "point normals");
        d.tstride = g->tangents.stride;
      }
      d.ntris = (uint32_t)nverts;
      return true;
    }
    if (nprims == 0 || !g->indices.buf) return false;
    if (!g->vertices.buf) fail(RTC_ERROR_INVALID_OPERATION, "vertex buffer not set");
    // curves: the float4 vertex buffer stays resident (the trace kernel reads neighbours / control points from it), one index per curve
    const size_t curveVertBytes = nverts ? (nverts - 1) * g->vertices.stride + 16 : 16, curveIdxBytes = (nprims - 1) * g->indices.stride + 4;
    if (pt.kind == rtk::PRIM_ROUND_LINEAR || pt.kind == rtk::PRIM_FLAT_LINEAR) {
      // linear curves (scene_line_segments.cpp): one index per segment, neighbour flags from the application or derived from the
      // index buffer as LineSegments::commit does (:209-232), computed on the device from the copies (rtk::linear_curve_flags)
      if (nprims > 0x3FFFFFFFull || nverts > 0x3FFFFFFFull) fail(RTC_ERROR_INVALID_OPERATION, "curve geometry too large");
      if (g->flags.buf && g->flags.count != nprims) fail(RTC_ERROR_INVALID_OPERATION, "flags buffer must hold one entry per segment");
      d.verts = copy(g->vertices, curveVertBytes, true, "curve vertices");
      (*curves)[g].verts = d.verts;
      d.idx = copy(g->indices, curveIdxBytes, false, "curve indices");
      const uint8_t* app = g->flags.buf ? copy(g->flags, (nprims - 1) * g->flags.stride + 1, false, "curve flags") : nullptr;
      uint8_t* fl = alloc(nprims, false, "curve neighbour flags");
      cuda_check((cudaError_t)rtk::linear_curve_flags(d.idx, d.istride, app, g->flags.stride, (uint32_t)nprims, fl, st), "curve flags launch");
      d.flags = fl;
      d.ntris = (uint32_t)nprims;
      return true;
    }
    if (rtk::curve_record(pt.kind)) {
      // cubic curves (scene_curves.cpp): float4 control vertices, one index per curve (first control vertex), Hermite adds float4
      // tangents; the basis weights at the tessellation points are tabulated here as the reference tabulates them
      const bool hermite = is_hermite(g->type);
      if (hermite && !g->tangents.buf) fail(RTC_ERROR_INVALID_OPERATION, "tangent buffer not set");
      if (hermite && g->tangents.count != nverts) fail(RTC_ERROR_INVALID_OPERATION, "number of tangents must match number of vertices");   // scene_curves.cpp commit
      d.tess = (uint32_t)g->tessellationRate;
      const size_t segs = rtk::prims_per_curve(d);
      if (nprims * segs > 0x7FFFFFFFull || nverts > 0xFFFFFFFFull) fail(RTC_ERROR_INVALID_OPERATION, "curve geometry too large");
      d.verts = copy(g->vertices, curveVertBytes, true, "curve vertices");
      (*curves)[g].verts = d.verts;
      d.idx = copy(g->indices, curveIdxBytes, false, "curve indices");
      if (hermite) {
        d.tangents = copy(g->tangents, nverts ? (nverts - 1) * g->tangents.stride + 16 : 16, true, "curve tangents");
        (*curves)[g].tangents = d.tangents;
        d.tstride = g->tangents.stride; d.hermite = 1;
      }
      d.basis = pt.basis;
      float tab[8 * (rtk::kMaxTess + 1)];
      rtk::curve_basis_table(d.basis, g->tessellationRate, tab);
      d.basis_tab = reinterpret_cast<const float*>(copy(tab, sizeof(float) * 8 * (g->tessellationRate + 1), true, "curve basis table"));
      cuda_check(cudaStreamSynchronize(st), "upload curve basis table");   // `tab` is on the stack
      d.ntris = (uint32_t)(nprims * segs);
      return true;
    }
    const bool quad = g->type == RTC_GEOMETRY_TYPE_QUAD;
    const size_t ntris = quad ? 2 * nprims : nprims;   // a quad contributes its two halves (quad_intersector_moeller.h:190-200)
    if (ntris > 0x7FFFFFFFull || nverts > 0xFFFFFFFFull) fail(RTC_ERROR_INVALID_OPERATION, "mesh too large");
    d.verts = copy(g->vertices, nverts ? (nverts - 1) * g->vertices.stride + 12 : 0, false, "vertices");
    d.idx = copy(g->indices, (nprims - 1) * g->indices.stride + (quad ? 16 : 12), false, "indices");
    d.ntris = (uint32_t)ntris; d.is_quad = quad ? 1 : 0;
    return true;
  }

  // RTC_GEOMETRY_TYPE_INSTANCE (kernels/geometry/instance_intersector.cpp:15-38): flattened here -- every mesh of the instanced scene
  // enters the top-level BVH through the instance transform; hits report the instance id, the CHILD scene's geomID / primID and an
  // object-space Ng exactly as the reference's two-level traversal does.  Grows `bounds` by the instance box and returns the
  // generation of the instanced scene it baked in.
  unsigned long long upload_instance(GeometryImpl* inst, uint32_t instID, float bounds[6]) {
    const unsigned long long gen = instanced_generation(inst);
    upload_scene(inst->instScene, inst, instID);
    add_instance_bounds(inst, bounds);
    return gen;
  }

  // Adds every enabled geometry of the instanced scene `child` under its geomID, seen through `inst` when that is not null.
  void upload_scene(SceneImpl* child, const GeometryImpl* inst = nullptr, uint32_t instID = RTC_INVALID_GEOMETRY_ID) {
    std::vector<GeometryImpl*> cgeoms;
    { std::lock_guard<std::mutex> lg(child->geomMutex); cgeoms = child->geoms; }
    for (size_t cid = 0; cid < cgeoms.size(); ++cid) {
      GeometryImpl* cg = cgeoms[cid];
      if (!cg || !cg->enabled) continue;
      if (cg->type == RTC_GEOMETRY_TYPE_INSTANCE)   // RTC_MAX_INSTANCE_LEVEL_COUNT == 1, as in the reference's default build
        fail(RTC_ERROR_INVALID_OPERATION, "multi-level instancing is not supported (RTC_MAX_INSTANCE_LEVEL_COUNT is 1)");
      upload_geometry(cg, (uint32_t)cid, inst, instID);
    }
  }

  // the generation of the scene the instance `inst` instances, which must have been committed
  static unsigned long long instanced_generation(const GeometryImpl* inst) {
    if (!inst->instScene) fail(RTC_ERROR_INVALID_OPERATION, "instance has no instanced scene");
    if (!inst->instScene->everCommitted) fail(RTC_ERROR_INVALID_OPERATION, "instanced scene not committed");
    return inst->instScene->generation.load();
  }

  // grows `bounds` by the instance box as the reference computes it: xfmBounds(local2world, child scene bounds) (affinespace.h:106-118)
  static void add_instance_bounds(const GeometryImpl* inst, float bounds[6]) {
    const float* cb = inst->instScene->apiBounds;
    if (cb[0] <= cb[3])
      for (int c = 0; c < 8; ++c) {
        const float x = (c & 4) ? cb[3] : cb[0], y = (c & 2) ? cb[4] : cb[1], z = (c & 1) ? cb[5] : cb[2];
        for (int a = 0; a < 3; ++a) {
          const float w = fmaf(x, inst->xfm[a], fmaf(y, inst->xfm[3 + a], fmaf(z, inst->xfm[6 + a], inst->xfm[9 + a])));
          bounds[a] = fminf(bounds[a], w); bounds[3 + a] = fmaxf(bounds[3 + a], w);
        }
      }
  }
};

// Two-level scenes: a DYNAMIC scene of several plain triangle meshes keeps one BVH per mesh (the reference's two-level builder for
// dynamic scenes) -- a commit rebuilds / refits only the meshes that changed and re-assembles the top level.  `possible`: the scene is
// such a scene; `chosen`: this commit takes the two-level path.
struct TwoLevelChoice { bool possible, chosen; };
TwoLevelChoice choose_two_level(const SceneImpl* s, const std::vector<GeometryImpl*>& geoms) {
  size_t nmeshes = 0;
  bool plain = true;
  for (GeometryImpl* g : geoms) if (g && g->enabled) { plain = plain && g->type == RTC_GEOMETRY_TYPE_TRIANGLE; ++nmeshes; }
  const bool possible = plain && nmeshes >= 2 && (s->flags & RTC_SCENE_FLAG_DYNAMIC);
  if (!possible || getenv("RTCB200_NO_TWOLEVEL")) return {possible, false};
  // Which regime is cheaper for THIS commit?  Cost model: rebuilding one BVH over everything costs ~1.5 ms + 2.5 ns per
  // triangle (device build plus the vertex upload at PCIe speed), the two-level commit ~1 ms + (0.5 ms + 2.5 ns per triangle)
  // per mesh modified since the last commit (bench.py extras.dynamic_scene_two_level times both paths).  When most meshes move every frame (tutorials/dynamic_scene) one rebuild wins; when a few of
  // many move, the two-level path does -- meshes that have no kept BVH yet are built then, a one-time investment.
  double total = 0.0, two = 1.0;
  for (size_t id = 0; id < geoms.size(); ++id) {
    GeometryImpl* g = geoms[id];
    if (!g || !g->enabled) continue;
    const double tris = (double)g->indices.count;
    total += tris;
    const bool modified = !s->everCommitted || id >= s->committedCounter.size() || s->committedCounter[id] != g->modCounter;
    if (modified) two += 0.5 + tris * 2.5e-6;
  }
  return {possible, two < 1.5 + total * 2.5e-6};
}

// quality -> builder (scene.cpp:163-206: LOW = Morton two-level builder, MEDIUM/HIGH = SAH)
rtk::BuilderKind builder_kind(const SceneImpl* s) { return s->quality == RTC_BUILD_QUALITY_LOW ? rtk::BUILDER_LBVH : rtk::BUILDER_SAH; }

// SceneGPU::curves of a BVH over `descs`: 2 with curve records among them, 1 with point records only, 0 with neither -- the two kinds
// take different leaf-test batching and grid (rtk::Tuning)
int curves_level(const std::vector<rtk::GeomDesc>& descs) {
  int level = 0;
  for (const rtk::GeomDesc& d : descs) level = std::max(level, d.kind == rtk::PRIM_TRIANGLE ? 0 : rtk::curve_record(d.kind) ? 2 : 1);
  return level;
}

// rtcGetSceneBounds: the scene's own primitives and the instance boxes
void set_api_bounds(SceneImpl* s, const float instBounds[6]) {
  for (int a = 0; a < 3; ++a) {
    s->apiBounds[a] = fminf(s->gpu.api_bounds[a], instBounds[a]);
    s->apiBounds[3 + a] = fmaxf(s->gpu.api_bounds[3 + a], instBounds[3 + a]);
  }
}

// A failed allocation stays the runtime's last error: cleared here, or the next commit's launch checks would report it again.
[[noreturn]] void build_failed(int code, const char* msg) {
  cudaGetLastError();
  fail(code == (int)cudaErrorMemoryAllocation ? RTC_ERROR_OUT_OF_MEMORY : RTC_ERROR_UNKNOWN, msg);
}

// a successful commit: what it committed (scene.cpp:878-884), the generation instancing scenes compare, and the staging block of
// a refit that did not wait (-1: none, the scene's bounds and times are final)
void finish_commit(SceneImpl* s, const std::vector<GeometryImpl*>& geoms, const std::vector<unsigned long long>& childGen, int refitBlock = -1) {
  s->lastRefit = refitBlock;
  {
    std::lock_guard<std::mutex> lg(s->geomMutex);
    s->committedCounter.assign(geoms.size(), 0u);
    for (size_t i = 0; i < geoms.size(); ++i) s->committedCounter[i] = geoms[i] ? geoms[i]->modCounter : 0u;
    s->committedChildGen = childGen;
    s->generation.fetch_add(1);
    // geometries attached while we were building keep the scene modified
    s->flagsModified = false;
    s->everCommitted = true;
  }
  if (s->progFn) s->progFn(s->progPtr, 1.0);
}

// May a REFIT commit of a DYNAMIC scene refit BVH `b` and still find what the reference finds?  The reference refits only in a
// DYNAMIC scene of LOW quality (scene.cpp:158-194: any other quality takes the STATIC SAH builder, which rebuilds on every commit;
// LOW takes the two-level builder whose per-mesh RefitBuilder refits, bvh_builder_twolevel_internal.h:297).  Its refit keeps the
// primitives of its last build, which dropped the invalid ones (TriangleMesh::buildBounds, scene_triangle_mesh.h:195-207), so a
// triangle made valid by a later vertex update stays unhittable there -- and here.  At any other quality the reference rebuilds: a
// refit here gives the same hits unless the last build dropped a primitive, and then this commit rebuilds too.
bool refit_keeps_reference_hits(const SceneImpl* s, const rtk::SceneGPU& b) {
  return s->quality == RTC_BUILD_QUALITY_LOW || b.num_tris == b.total_prims;
}

// The kept BVHs of one commit.  take() hands out the cached entry for (obj, id), or a new one.  When the commit ends, however it
// ends, every entry handed out goes back into the cache: one rebuilt before a later failure is kept, not lost with its buffers, and
// its SceneGPU::content tells the next assembly that the copy in the scene's arrays is stale.  done(), called once the commit has
// succeeded, drops the cached entries it did not take.
struct KeptBvhs {
  SceneImpl::KeptMap& cache;
  SceneImpl::KeptMap taken;
  int device;
  cudaStream_t st;   // the commit stream, where the dropped entries are freed
  KeptBvhs(SceneImpl::KeptMap& c, int dev, cudaStream_t stream) : cache(c), device(dev), st(stream) {}
  ~KeptBvhs() { for (auto& kv : taken) cache[kv.first] = std::move(kv.second); }
  SceneImpl::KeptBvh* take(const void* obj, unsigned id) {
    std::unique_ptr<SceneImpl::KeptBvh>& e = taken[{obj, id}];
    if (e) return e.get();
    auto it = cache.find({obj, id});
    if (it != cache.end()) { e = std::move(it->second); cache.erase(it); }
    else { e.reset(new SceneImpl::KeptBvh()); e->gpu.device = device; e->gpu.is_sub = true; }
    return e.get();
  }
  void done() { clear_kept(cache, st); }
};

void commit_two_level(SceneImpl* s, const std::vector<GeometryImpl*>& geoms, cudaStream_t cs) {
  const int robust = (s->flags & RTC_SCENE_FLAG_ROBUST) ? 1 : 0;
  CommitUpload up(s, cs);
  KeptBvhs kept(s->meshBvhs, s->dev->gpu, cs);
  std::vector<rtk::SceneGPU*> order;
  size_t rebuilt = 0;
  char err[256];
  {   // many fresh per-mesh BVHs keep their memory: grow the stream-ordered pool once instead of once per mesh (~ms each)
    size_t fresh_tris = 0, fresh_n = 0;
    for (size_t id = 0; id < geoms.size(); ++id) {
      GeometryImpl* g = geoms[id];
      if (g && g->enabled && !s->meshBvhs.count({g, (unsigned)id})) { fresh_tris += g->indices.count; ++fresh_n; }
    }
    if (fresh_n >= 8) {
      void* prime = nullptr;
      const size_t bytes = fresh_tris * 400 + (size_t)fresh_n * (1u << 16);     // nodes + records + the build's temporaries, generously
      if (cudaMallocAsync(&prime, bytes, cs) == cudaSuccess) cudaFreeAsync(prime, cs);
      else cudaGetLastError();
    }
  }
  for (size_t id = 0; id < geoms.size(); ++id) {
    GeometryImpl* g = geoms[id];
    if (!g || !g->enabled) continue;
    SceneImpl::KeptBvh* e = kept.take(g, (unsigned)id);
    order.push_back(&e->gpu);
    // only a changed mesh is uploaded and built again (a new entry has no serial)
    if (e->serial == g->serial && e->modCounter == g->modCounter && e->sceneQuality == s->quality && e->robust == robust && e->gpu.device == s->dev->gpu)
      continue;
    e->gpu.robust = robust; e->gpu.general = 0; e->gpu.curves = 0;
    int r = 0;
    if (!up.upload_geometry(g, (uint32_t)id)) {   // no triangles: an empty sub-BVH
      rtk::free_scene(e->gpu, cs);
      for (int a = 0; a < 3; ++a) { e->gpu.bounds[a] = INFINITY; e->gpu.bounds[3 + a] = -INFINITY; }
    } else if (e->serial == g->serial && g->quality == RTC_BUILD_QUALITY_REFIT && e->gpu.root_valid && e->nprims == g->indices.count &&
               e->nverts == g->vertices.count && e->indexVersion == g->indexVersion && refit_keeps_reference_hits(s, e->gpu) &&
               e->sceneQuality == s->quality && e->robust == robust)
      r = rtk::refit_scene(e->gpu, &up.descs.back(), 1, cs, err);
    else
      r = rtk::build_scene(e->gpu, &up.descs.back(), 1, builder_kind(s), cs, err);
    if (r != 0) build_failed(r, err);
    e->serial = g->serial; e->modCounter = g->modCounter; e->sceneQuality = s->quality; e->robust = robust; e->nprims = g->indices.count; e->nverts = g->vertices.count;
    e->indexVersion = g->indexVersion;
    ++rebuilt;
  }
  kept.done();            // meshes that are no longer attached or enabled
  s->gpu.general = 0; s->gpu.curves = 0; s->gpu.robust = robust;
  if (s->gpu.d_descs) { cudaFreeAsync(s->gpu.d_descs, cs); s->gpu.d_descs = nullptr; }
  if (s->gpu.tri_src) { cudaFreeAsync(s->gpu.tri_src, cs); s->gpu.tri_src = nullptr; }
  const int r = rtk::assemble_scene(s->gpu, order.data(), (int)order.size(), cs, err);
  release_buffers(s->deviceBuffers, cs);
  if (r != 0) { rtk::free_scene(s->gpu, cs); build_failed(r, err); }
  s->builtTopology.clear();
  for (int a = 0; a < 6; ++a) s->apiBounds[a] = s->gpu.api_bounds[a];
  if (s->dev->verbose >= 2)
    fprintf(stderr, "[b200] commit (two-level): %zu meshes, %zu rebuilt or refitted, %u nodes, %u tris, assembly %.3f ms\n", order.size(),
            rebuilt, s->gpu.num_nodes, s->gpu.num_tris, s->gpu.build_ms);
  finish_commit(s, geoms, std::vector<unsigned long long>(geoms.size(), 0ull));
}

// Does every buffer a refit of `geoms` reads live in GPU memory?  Then its copies need no pageable memory and the refit need not wait.
bool refit_reads_device_views_only(const std::vector<GeometryImpl*>& geoms) {
  for (GeometryImpl* g : geoms)
    if (g && g->enabled && !(g->vertices.on_device() && g->indices.on_device())) return false;
  return true;
}

// one BVH over everything, instances flattened into it.  `wait`: a refit waits for the device too (rtcCommitScene).
void commit_single(SceneImpl* s, const std::vector<GeometryImpl*>& geoms, bool twoLevelPossible, cudaStream_t cs, bool wait) {
  // the kept per-mesh BVHs stay only while the scene could return to the two-level path (they are compared by modCounter then)
  if (!twoLevelPossible) clear_kept(s->meshBvhs, cs);
  CommitUpload up(s, cs);
  std::vector<unsigned long long> childGen(geoms.size(), 0ull);   // generation of every instanced scene as baked in below
  bool instanced = false;
  float instBounds[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (size_t id = 0; id < geoms.size(); ++id) {
    GeometryImpl* g = geoms[id];
    if (!g || !g->enabled) continue;
    if (g->type != RTC_GEOMETRY_TYPE_INSTANCE) up.upload_geometry(g, (uint32_t)id);
    else { instanced = true; childGen[id] = up.upload_instance(g, (uint32_t)id, instBounds); }
  }
  bool quads = false;
  for (const rtk::GeomDesc& d : up.descs) quads |= d.is_quad != 0;
  s->gpu.curves = curves_level(up.descs);
  s->gpu.general = (instanced || quads || s->gpu.curves) ? 1 : 0;
  s->gpu.robust = (s->flags & RTC_SCENE_FLAG_ROBUST) ? 1 : 0;   // scene.cpp:181-188: Triangle4v + Pluecker
  char errmsg[256];
  // REFIT (geometry build quality, rtcore_geometry.h; kernels/bvh/bvh_refit.cpp): same meshes, same counts, moved vertices
  std::vector<SceneImpl::TopoEntry> topo;
  bool wantRefit = !instanced && !s->gpu.curves && !up.descs.empty();
  for (size_t id = 0; id < geoms.size(); ++id) {
    GeometryImpl* g = geoms[id];
    if (!g || !g->enabled) continue;
    topo.push_back({g, (unsigned)id, g->indices.count, g->vertices.count, g->serial, g->indexVersion});
    wantRefit = wantRefit && g->quality == RTC_BUILD_QUALITY_REFIT;
  }
  // only a DYNAMIC scene refits: the reference rebuilds every other scene on each commit (scene.cpp:807-810)
  const bool canRefit = wantRefit && (s->flags & RTC_SCENE_FLAG_DYNAMIC) && s->gpu.root_valid && refit_keeps_reference_hits(s, s->gpu) &&
                        s->everCommitted && topo == s->builtTopology && s->builtQuality == s->quality && s->builtFlags == s->flags;
  // a refit from device views on a stream commit enqueues its work and returns: its root box and time are taken at settle()
  const size_t stagingBytes = rtk::refit_staging_bytes((int)up.descs.size());
  const int block = canRefit && !wait && refit_reads_device_views_only(geoms) ? s->free_refit_staging(stagingBytes) : -1;
  int r;
  if (canRefit) r = rtk::refit_scene(s->gpu, up.descs.data(), (int)up.descs.size(), cs, errmsg, block >= 0 ? &s->refitStaging[block] : nullptr);
  else {
    r = rtk::build_scene(s->gpu, up.descs.data(), (int)up.descs.size(), builder_kind(s), cs, errmsg);
    s->builtTopology = topo; s->builtQuality = s->quality; s->builtFlags = s->flags;
  }
  // vertex/index copies are only needed during the build (triangles are baked into the leaf records)
  release_buffers(s->deviceBuffers, cs);
  if (r != 0) {
    rtk::free_scene(s->gpu, cs);
    build_failed(r, errmsg);
  }
  // the blocks the next refits take (with frames in flight, one each); a later refit finds none free only when more frames are in
  // flight than this, and then waits
  if (!canRefit && wantRefit && (s->flags & RTC_SCENE_FLAG_DYNAMIC)) s->reserve_refit_staging(stagingBytes, 4);
  if (s->gpu.general)   // the build uploads the descriptors in this order (rtk::SceneGPU::d_descs)
    for (const rtk::GeomDesc& d : up.descs) s->descIds.push_back({d.geomID, d.has_xfm ? d.instID : RTC_INVALID_GEOMETRY_ID});
  set_api_bounds(s, instBounds);
  if (block >= 0) {
    if (s->dev->verbose >= 2)
      fprintf(stderr, "[b200] commit: %u tris, %u nodes, builder=refit, enqueued on the commit stream without a host wait\n", s->gpu.num_tris, s->gpu.num_nodes);
    finish_commit(s, geoms, childGen, block);
    return;
  }
  if (s->dev->verbose >= 2)
    fprintf(stderr, "[b200] commit%s: %u tris, %u nodes (%.1f MB) + %.1f MB tris, builder=%s, %.3f ms (%.1f Mprim/s), SAH %.2f, depth %u\n",
            instanced ? " (instances flattened)" : "", s->gpu.num_tris, s->gpu.num_nodes, s->gpu.num_nodes * sizeof(rtk::Node8) * 1e-6, s->gpu.num_tris * sizeof(rtk::TriRec) * 1e-6,
            s->gpu.builder == rtk::BUILDER_TWO_LEVEL ? "two-level" : s->gpu.builder == rtk::BUILDER_REFIT ? "refit" : s->gpu.builder == rtk::BUILDER_SAH ? "sah" : "lbvh",
            s->gpu.build_ms, s->gpu.build_ms > 0 ? s->gpu.num_tris / s->gpu.build_ms * 1e-3 : 0.0,
            s->gpu.sah_cost, s->gpu.max_depth);
  finish_commit(s, geoms, childGen);
}

// Instance traversal keeps one BVH per instanced scene and a top level over the scene's own primitives and one primitive per
// instance.  Scenes on it are not served by device-side queries or filter callbacks, so a scene is flattened (commit_single, which
// also traces faster) whenever that can be built.  Instance traversal is taken when the flattened copy is beyond what the builder
// takes (kMaxFlatPrims), when its build runs out of memory (commit_scene), or when the application lowered
// rtk::Tuning::instance_flatten_max below the flattened record count (the sum over the instances of the instanced scene's
// records) -- except for a scene with filter callbacks on its geometries or those of its instanced scenes, which is flattened then.
constexpr uint64_t kMaxFlatPrims = 0x7FFFFFFEull;   // build_scene's limit on the primitives of one BVH
bool choose_instance_traversal(const std::vector<GeometryImpl*>& geoms) {
  uint64_t flat = 0;
  bool any = false, filters = false;
  for (GeometryImpl* g : geoms) {
    if (!g || !g->enabled) continue;
    filters |= g->has_filter();
    if (g->type != RTC_GEOMETRY_TYPE_INSTANCE || !g->instScene) continue;
    any = true;
    flat += g->instScene->gpu.num_tris;
    std::lock_guard<std::mutex> lc(g->instScene->geomMutex);
    for (GeometryImpl* cg : g->instScene->geoms) filters |= cg && cg->enabled && cg->has_filter();
  }
  if (!any) return false;
  if (flat > kMaxFlatPrims) return true;
  return !filters && flat > (uint64_t)std::max(0, rtk::tuning().instance_flatten_max);
}
bool has_instances(const std::vector<GeometryImpl*>& geoms) {
  for (GeometryImpl* g : geoms) if (g && g->enabled && g->type == RTC_GEOMETRY_TYPE_INSTANCE && g->instScene) return true;
  return false;
}

void commit_instanced(SceneImpl* s, const std::vector<GeometryImpl*>& geoms, cudaStream_t cs) {
  clear_kept(s->meshBvhs, cs);
  const int robust = (s->flags & RTC_SCENE_FLAG_ROBUST) ? 1 : 0;
  CommitUpload up(s, cs);
  std::vector<unsigned long long> childGen(geoms.size(), 0ull);
  std::vector<std::pair<GeometryImpl*, uint32_t>> insts;
  float instBounds[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (size_t id = 0; id < geoms.size(); ++id) {
    GeometryImpl* g = geoms[id];
    if (!g || !g->enabled) continue;
    if (g->type != RTC_GEOMETRY_TYPE_INSTANCE) { up.upload_geometry(g, (uint32_t)id); continue; }
    childGen[id] = CommitUpload::instanced_generation(g);
    insts.push_back({g, (uint32_t)id});
    CommitUpload::add_instance_bounds(g, instBounds);
  }
  char err[256];
  // one BVH per instanced scene, in the order of first use
  KeptBvhs kept(s->sceneBvhs, s->dev->gpu, cs);
  std::map<SceneImpl*, uint32_t> kidIndex;
  std::vector<SceneImpl::KeptBvh*> order;
  size_t rebuilt = 0;
  for (auto& gi : insts) {
    SceneImpl* c = gi.first->instScene;
    if (kidIndex.count(c)) continue;
    SceneImpl::KeptBvh* e = kept.take(c, 0);
    if (!e->scene) { e->scene = c; c->retain(); }
    kidIndex[c] = (uint32_t)order.size();
    order.push_back(e);
    const unsigned long long gen = childGen[gi.second];
    if (e->generation == gen && e->sceneQuality == s->quality && e->robust == robust) continue;
    e->release(cs);
    e->curves.clear(); e->descs.clear(); e->generation = ~0ull;
    CommitUpload cu(s, cs);
    cu.resident = &e->resident; cu.curves = &e->curves;
    cu.upload_scene(c);
    e->gpu.robust = robust; e->gpu.general = 1; e->gpu.curves = curves_level(cu.descs);
    const int r = rtk::build_scene(e->gpu, cu.descs.data(), (int)cu.descs.size(), builder_kind(s), cs, err);
    if (r != 0) build_failed(r, err);
    e->descs = cu.descs; e->generation = gen; e->sceneQuality = s->quality; e->robust = robust;
    ++rebuilt;
  }
  kept.done();   // instanced scenes no longer instanced here
  for (SceneImpl::KeptBvh* e : order)
    for (auto& kv : e->curves) s->residentCurves[kv.first] = kv.second;

  // descriptors: those of every instanced scene, then the scene's own, then the one of the instances
  std::vector<rtk::GeomDesc> descs;
  std::vector<uint32_t> kidDescOff;
  std::vector<rtk::SceneGPU*> kidGpu;
  uint32_t kidDepth = 0;
  int curves = curves_level(up.descs);
  for (SceneImpl::KeptBvh* e : order) {
    kidDescOff.push_back((uint32_t)descs.size());
    descs.insert(descs.end(), e->descs.begin(), e->descs.end());
    kidGpu.push_back(&e->gpu);
    kidDepth = std::max(kidDepth, e->gpu.max_depth);
    curves = std::max(curves, e->gpu.curves);
  }
  const uint32_t topDescOff = (uint32_t)descs.size();
  uint64_t kidNodes, kidTris;
  const std::vector<rtk::SubSlot> L = rtk::sub_layout(kidGpu.data(), (int)kidGpu.size(), 1, kidNodes, kidTris);
  std::vector<rtk::InstRec> table(insts.size());
  for (size_t i = 0; i < insts.size(); ++i) {
    const GeometryImpl* g = insts[i].first;
    const uint32_t k = kidIndex[g->instScene];
    rtk::InstRec& ir = table[i];
    memset(&ir, 0, sizeof ir);
    memcpy(ir.w2l, g->w2l, sizeof ir.w2l); memcpy(ir.xfm, g->xfm, sizeof ir.xfm);
    ir.instID = insts[i].second; ir.mask = g->mask; ir.child_root = L[k].node_off;
    const rtk::SceneGPU& kg = *kidGpu[k];
    for (int a = 0; a < 3; ++a) {
      ir.lo[a] = kg.root_valid ? kg.bounds[a] : INFINITY;
      ir.hi[a] = kg.root_valid ? kg.bounds[3 + a] : -INFINITY;
    }
  }
  rtk::InstRec* d_insts = nullptr;
  cuda_check(cudaMallocAsync(reinterpret_cast<void**>(&d_insts), std::max<size_t>(table.size(), 1) * sizeof(rtk::InstRec), cs), "cudaMallocAsync(instances)");
  cuda_check(cudaMemcpyAsync(d_insts, table.data(), table.size() * sizeof(rtk::InstRec), cudaMemcpyHostToDevice, cs), "upload instances");
  // the top level: the scene's own primitives and one primitive per instance
  std::vector<rtk::GeomDesc> topDescs = up.descs;
  rtk::GeomDesc id{};
  id.kind = rtk::PRIM_INSTANCE; id.verts = reinterpret_cast<const uint8_t*>(d_insts); id.ntris = (uint32_t)insts.size(); id.skip_bounds = 1;
  topDescs.push_back(id);
  rtk::SceneGPU top;
  top.device = s->dev->gpu; top.is_sub = true; top.robust = robust; top.general = 1;
  int r = rtk::build_scene(top, topDescs.data(), (int)topDescs.size(), builder_kind(s), cs, err);
  release_buffers(s->deviceBuffers, cs);
  // a ray inside an instance holds the top level's entries, its leaf group, the exit marker and the instanced scene's entries
  if (r == 0 && top.max_depth + kidDepth + 2 > (uint32_t)rtk::kStackSize) {
    rtk::free_scene(top, cs); cudaFreeAsync(d_insts, cs);
    snprintf(err, sizeof err, "instance traversal too deep for the traversal stack (%u top-level + %u instanced levels, %d entries)", top.max_depth,
             kidDepth, rtk::kStackSize);
    fail(RTC_ERROR_INVALID_OPERATION, err);
  }
  if (r == 0) r = rtk::assemble_instanced(s->gpu, top, kidGpu.data(), kidDescOff.data(), (int)kidGpu.size(), topDescOff, cs, err);
  const double topMs = top.build_ms;
  const uint32_t topPrims = top.num_tris;
  rtk::free_scene(top, cs);
  if (r != 0) { cudaFreeAsync(d_insts, cs); rtk::free_scene(s->gpu, cs); build_failed(r, err); }
  descs.insert(descs.end(), topDescs.begin(), topDescs.end());
  if (s->gpu.d_descs) cudaFreeAsync(s->gpu.d_descs, cs);
  if (s->gpu.tri_src) { cudaFreeAsync(s->gpu.tri_src, cs); s->gpu.tri_src = nullptr; }
  if (s->gpu.d_insts) cudaFreeAsync(s->gpu.d_insts, cs);
  cuda_check(cudaMallocAsync(reinterpret_cast<void**>(&s->gpu.d_descs), descs.size() * sizeof(rtk::GeomDesc), cs), "cudaMallocAsync(descriptors)");
  cuda_check(cudaMemcpyAsync(s->gpu.d_descs, descs.data(), descs.size() * sizeof(rtk::GeomDesc), cudaMemcpyHostToDevice, cs), "upload descriptors");
  cuda_check(cudaStreamSynchronize(cs), "upload descriptors");   // `descs` is on the stack
  s->gpu.num_descs = (uint32_t)descs.size();
  s->gpu.d_insts = d_insts; s->gpu.num_insts = (uint32_t)insts.size();
  s->gpu.general = 1; s->gpu.curves = curves; s->gpu.robust = robust;
  s->builtTopology.clear();
  set_api_bounds(s, instBounds);   // as flattened
  if (s->dev->verbose >= 2)
    fprintf(stderr, "[b200] commit (instance traversal): %zu instances of %zu scenes, %zu rebuilt, top level %u prims in %.3f ms, %u nodes, %u tris, "
            "depth %u + %u, assembly %.3f ms\n", insts.size(), order.size(), rebuilt, topPrims, topMs, s->gpu.num_nodes, s->gpu.num_tris, s->gpu.max_depth - kidDepth,
            kidDepth, s->gpu.build_ms);
  finish_commit(s, geoms, childGen);
}

// Commits `s` with its device work enqueued on `cs` after the work already there.  `wait` (rtcCommitScene): every path, the refit
// too, waits for its device work before it returns, as it always has.  Otherwise the scene's completion event is recorded after
// the commit's work and stays pending until a reader settles it.
void commit_scene(SceneImpl* s, cudaStream_t cs, bool wait) {
  std::lock_guard<std::mutex> lk(s->commitMutex);
  std::vector<GeometryImpl*> geoms;
  {
    std::lock_guard<std::mutex> lg(s->geomMutex);
    if (!s->isModified()) return;
    geoms = s->geoms;
  }
  for (GeometryImpl* g : geoms)
    if (g && g->enabled && g->state == GeomState::MODIFIED) fail(RTC_ERROR_INVALID_OPERATION, "geometry not committed");
  if (s->progFn && !s->progFn(s->progPtr, 0.0)) fail(RTC_ERROR_CANCELLED, "progress monitor forced termination");
  s->dev->use();
  // the bounds of the instanced scenes are read below; a stream commit of this scene still running is followed on `cs`
  for (GeometryImpl* g : geoms)
    if (g && g->enabled && g->type == RTC_GEOMETRY_TYPE_INSTANCE && g->instScene) g->instScene->settle();
  s->wait_on(cs);
  auto reset = [s, cs] {   // what the last commit (or attempt) uploaded and what was derived from it
    release_buffers(s->deviceBuffers, cs);
    release_buffers(s->residentBuffers, cs);
    s->residentCurves.clear();
    s->free_interp(cs);
    s->free_geom_tables(cs);
    s->descIds.clear();
  };
  reset();
  const TwoLevelChoice twoLevel = choose_two_level(s, geoms);
  if (!twoLevel.chosen && choose_instance_traversal(geoms)) commit_instanced(s, geoms, cs);
  else {
    clear_kept(s->sceneBvhs, cs);
    if (s->gpu.d_insts) { cudaFreeAsync(s->gpu.d_insts, cs); s->gpu.d_insts = nullptr; s->gpu.num_insts = 0; }
    if (twoLevel.chosen) commit_two_level(s, geoms, cs);
    else {
      try {
        commit_single(s, geoms, twoLevel.possible, cs, wait);
      } catch (const ApiError& e) {
        // a flattened copy too large for the card's memory: the scene commits with instance traversal instead, which at this size is
        // the only way it commits at all
        if (e.code != RTC_ERROR_OUT_OF_MEMORY || !has_instances(geoms)) throw;
        reset();
        if (s->dev->verbose >= 2) fprintf(stderr, "[b200] commit: flattening the instances ran out of memory (%s); instance traversal instead\n", e.msg.c_str());
        commit_instanced(s, geoms, cs);
      }
    }
  }
  if (wait) return;
  if (!s->committed) cuda_check(cudaEventCreateWithFlags(&s->committed, cudaEventDisableTiming), "cudaEventCreate");
  cuda_check(cudaEventRecord(s->committed, cs), "record the commit's completion");
  s->pending = true;
}

// ---- query plumbing ----------------------------------------------------------------------------------------------
struct ThreadCtx {  // per calling thread: a stream and a mapped pinned staging record for the single-call path
  int gpu = -1;
  cudaStream_t stream = nullptr;
  static constexpr size_t kStagingBytes = 16384;
  char* staging = nullptr;  // mapped pinned: 1344 B packet + 64 B valid for the single-call path; [2048, 16384) = the filter passes of small queries
  ~ThreadCtx() {
    if (staging) cudaFreeHost(staging);
    if (stream) cudaStreamDestroy(stream);
  }
  void ensure(int g) {
    if (gpu == g && stream) return;
    if (staging) { cudaFreeHost(staging); staging = nullptr; }
    if (stream) { cudaStreamDestroy(stream); stream = nullptr; }
    cudaSetDevice(g);
    cuda_check(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking), "cudaStreamCreate");
    cuda_check(cudaHostAlloc(reinterpret_cast<void**>(&staging), kStagingBytes, cudaHostAllocMapped), "cudaHostAlloc");
    gpu = g;
  }
};
thread_local ThreadCtx t_ctx;

// RTCIntersectArguments / RTCOccludedArguments (rtcore_common.h:335-361, context.h:14-62).  `context->instID` seeds the
// hit's instance ids.  `flags`: RTC_RAY_QUERY_FLAG_COHERENT only selects the reference's coherent packet traverser
// (context.h:41-45) -- a performance hint with identical results, so every value is accepted; a warp here always traces 32
// rays together; RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER makes `filter` apply to every geometry (context.h:48-50).
// `feature_mask`: "should get used in SYCL" (doc/src/api/rtcInitIntersectArguments.md:48); the reference's CPU entry
// points never read it (kernels/common/rtcore.cpp), neither do we.  `filter` is a host function: the host-pointer entry
// points run it through trace_filtered() below, the Device entry points refuse it.  `intersect` / `occluded` belong to
// user geometries, which this back-end does not have.
struct QueryArgs {
  uint32_t instID = RTC_INVALID_GEOMETRY_ID, instPrimID = RTC_INVALID_GEOMETRY_ID;
  RTCFilterFunctionN filter = nullptr;
  bool enforce = false;                  // RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER
  RTCRayQueryContext* ctx = nullptr;     // the caller's context (NULL: a default one is made for the callbacks)
};
template <typename Args>
QueryArgs read_args(const Args* a) {
  QueryArgs q;
  if (!a) return q;
  q.filter = a->filter;
  q.enforce = (a->flags & RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER) != 0;
  q.ctx = a->context;
  if (a->context) { q.instID = a->context->instID[0]; q.instPrimID = a->context->instPrimID[0]; }
  return q;
}

// Does a filter callback apply to some geometry of this scene for this query (filter.h:15-36, :51-71)?
bool filters_apply(SceneImpl* s, const QueryArgs& q, int occluded) {
  if (!q.filter && g_filterGeoms.load(std::memory_order_relaxed) == 0) return false;
  auto applies = [&](const GeometryImpl* g) {
    if (occluded ? g->occludedFilter != nullptr : g->intersectFilter != nullptr) return true;
    return q.filter && (q.enforce || g->argFilterEnabled);
  };
  std::lock_guard<std::mutex> lg(s->geomMutex);
  for (GeometryImpl* g : s->geoms) {
    if (!g || !g->enabled) continue;
    if (g->type != RTC_GEOMETRY_TYPE_INSTANCE) { if (applies(g)) return true; continue; }
    if (!g->instScene) continue;
    std::lock_guard<std::mutex> lc(g->instScene->geomMutex);
    for (GeometryImpl* cg : g->instScene->geoms)
      if (cg && cg->enabled && cg->type != RTC_GEOMETRY_TYPE_INSTANCE && applies(cg)) return true;
  }
  return false;
}

rtk::TraceParams make_params(SceneImpl* s, void* rays, const int* valid, unsigned long long n, uint32_t instID,
                             uint32_t instPrimID) {
  rtk::TraceParams p;
  p.nodes = s->gpu.nodes; p.tris = s->gpu.tris; p.root_valid = s->gpu.root_valid; p.robust = s->gpu.robust;
  p.descs = s->gpu.general ? s->gpu.d_descs : nullptr;
  p.curves = s->gpu.curves;
  p.insts = s->gpu.d_insts;
  p.rays = rays; p.valid = valid; p.n = n; p.instID = instID; p.instPrimID = instPrimID;
  p.stat = s->statCounters ? s->gpu.d_stat : nullptr;
  return p;
}

void require_committed(SceneImpl* s) {
  if (!s->everCommitted) fail(RTC_ERROR_INVALID_OPERATION, "scene not committed");  // scene.cpp:36,65
}

// one synchronous record (single ray or one packet): stage in mapped pinned memory, one launch, one sync
void trace_one(SceneImpl* s, void* rec, size_t recBytes, const int* valid, int K, int occluded, uint32_t instID,
               uint32_t instPrimID) {
  require_committed(s);
  if (!s->gpu.root_valid) return;
  t_ctx.ensure(s->dev->gpu);
  cudaSetDevice(s->dev->gpu);
  s->wait_on(t_ctx.stream);
  memcpy(t_ctx.staging, rec, recBytes);
  int* sv = reinterpret_cast<int*>(t_ctx.staging + 1408);
  if (K > 1) memcpy(sv, valid, 4 * K);
  rtk::TraceParams p = make_params(s, t_ctx.staging, K > 1 ? sv : nullptr, (unsigned long long)K, instID, instPrimID);
  cuda_check((cudaError_t)rtk::launch_trace(p, occluded, K, t_ctx.stream), "trace launch");
  cuda_check(cudaStreamSynchronize(t_ctx.stream), "trace");
  memcpy(rec, t_ctx.staging, recBytes);
}

// batched, device pointers: enqueue only
void trace_device(SceneImpl* s, void* d_rays, const int* d_valid, int K, size_t M, int occluded, uint32_t instID,
                  uint32_t instPrimID, cudaStream_t st, bool timeit, void* compact_out = nullptr) {
  require_committed(s);
  if (!s->gpu.root_valid || M == 0) return;
  cudaSetDevice(s->dev->gpu);
  s->wait_on(st);
  rtk::TraceParams p = make_params(s, d_rays, d_valid, (unsigned long long)M * K, instID, instPrimID);
  p.compact_out = compact_out;
  if (timeit) {
    if (!s->ev0) { cudaEventCreate(&s->ev0); cudaEventCreate(&s->ev1); }
    cudaEventRecord(s->ev0, st);
  }
  cuda_check((cudaError_t)rtk::launch_trace(p, occluded, K, st), "trace launch");
  if (timeit) cudaEventRecord(s->ev1, st);
}

// ---- multi-GPU hit gather into another GPU's memory ------------------------------------------------------------------
// rtcb200Intersect1MGatherDevice: the trace kernel itself delivers one compact 32-byte hit record per ray into
// `compact_out` -- local memory or a peer's memory over NVLink -- so the transfer is spread over the whole launch and no
// separate collective moves hit data.  rtcb200SetTuning("gather_mode", m): 1 (default) writes each record to a local staging
// buffer first and sends complete 32-ray blocks as 1 KB (eight full lines); 0 stores every record on its own as
// one 32-byte sector when its ray terminates (with many peers, rank 0's ingest of single sectors is request-rate bound).
void trace_gather(SceneImpl* s, void* d_rays, size_t M, uint32_t instID, uint32_t instPrimID, cudaStream_t st, void* compact_out) {
  require_committed(s);
  if (M == 0) return;
  if (reinterpret_cast<uintptr_t>(compact_out) & 31) fail(RTC_ERROR_INVALID_ARGUMENT, "compact_out must be 32-byte aligned (one sector per record)");
  cudaSetDevice(s->dev->gpu);
  s->wait_on(st);
  if (!s->ev0) { cudaEventCreate(&s->ev0); cudaEventCreate(&s->ev1); }
  cudaEventRecord(s->ev0, st);
  rtk::TraceParams p = make_params(s, d_rays, nullptr, (unsigned long long)M, instID, instPrimID);
  p.compact_out = compact_out;
  if (rtk::tuning().gather_mode == 1) {   // local staging buffer of the blocked delivery, kept per calling thread and device
    static thread_local struct Stage { int gpu = -1; void* p = nullptr; size_t cap = 0; ~Stage() { if (p) cudaFree(p); } } t_stage;
    if (t_stage.gpu != s->dev->gpu || t_stage.cap < M * 32) {
      if (t_stage.p) { cudaSetDevice(t_stage.gpu); cudaFree(t_stage.p); cudaSetDevice(s->dev->gpu); }
      t_stage.p = nullptr; t_stage.cap = 0; t_stage.gpu = s->dev->gpu;
      cuda_check(cudaMalloc(&t_stage.p, M * 32), "cudaMalloc(gather staging)");
      t_stage.cap = M * 32;
    }
    p.stage = t_stage.p;
  }
  cuda_check((cudaError_t)rtk::launch_trace(p, 0, 1, st), "trace launch");   // empty scene: every ray stores its miss record
  cudaEventRecord(s->ev1, st);
}

// batched, host pointers: chunked H2D -> trace -> D2H pipeline over three streams
// host-buffer pipeline shape (rtcb200SetTuning "host_chunk_log2" / "host_streams"): rays per chunk and chunks in flight
static int g_host_chunk_log2 = 20, g_host_streams = 3;   // scripts/e2e_sweep.py sweeps both
// rtcb200SetTuning("host_d2h_partial", 1): the copy back to the host skips the bytes of a record that a query never changes -- org, tnear,
// dir, time of an RTCRayHit (the first 32 of its 96 bytes), the first eight fields of an RTCRayHitK -- with a pitched copy of the rest.
// Fewer bytes cross PCIe and, with several GPUs per socket, the host's memory controllers -- but the copy engine moves the 64-byte
// rows of a pitched copy slower than one contiguous block (scripts/e2e_partial_ab.py compares both), so it is OFF by default.
static int g_host_d2h_partial = 0;

struct HostPipe {
  int gpu = -1;
  static constexpr int kStreams = 6;   // upper bound; g_host_streams of them are used
  cudaStream_t st[kStreams] = {};
  char* buf[kStreams] = {};
  int* vbuf[kStreams] = {};
  size_t cap = 0, vcap = 0;
  ~HostPipe() { reset(); }
  void reset() {
    for (int i = 0; i < kStreams; ++i) {
      if (buf[i]) cudaFree(buf[i]);
      if (vbuf[i]) cudaFree(vbuf[i]);
      if (st[i]) cudaStreamDestroy(st[i]);
      buf[i] = nullptr; vbuf[i] = nullptr; st[i] = nullptr;
    }
    cap = vcap = 0; gpu = -1;
  }
  void ensure(int g, size_t bytes, size_t vbytes) {
    if (gpu != g) reset();
    cudaSetDevice(g);
    gpu = g;
    for (int i = 0; i < kStreams; ++i)
      if (!st[i]) cuda_check(cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking), "cudaStreamCreate");
    if (bytes > cap) {
      for (int i = 0; i < kStreams; ++i) { if (buf[i]) cudaFree(buf[i]); buf[i] = nullptr; cuda_check(cudaMalloc(&buf[i], bytes), "cudaMalloc(ray chunk)"); }
      cap = bytes;
    }
    if (vbytes > vcap) {
      for (int i = 0; i < kStreams; ++i) { if (vbuf[i]) cudaFree(vbuf[i]); vbuf[i] = nullptr; cuda_check(cudaMalloc(&vbuf[i], vbytes), "cudaMalloc(valid chunk)"); }
      vcap = vbytes;
    }
  }
};
thread_local HostPipe t_pipe;

void trace_host(SceneImpl* s, void* rays, const int* valid, int K, size_t M, size_t recBytes, int occluded,
                uint32_t instID, uint32_t instPrimID) {
  require_committed(s);
  if (!s->gpu.root_valid || M == 0) return;
  const size_t chunkRecs = std::max<size_t>(1, (size_t(1) << g_host_chunk_log2) / K);  // 1 Mi rays per chunk by default
  const int nst = std::min(std::max(g_host_streams, 1), (int)HostPipe::kStreams);
  const size_t chunks = (M + chunkRecs - 1) / chunkRecs;
  const size_t perChunk = std::min(M, chunkRecs);
  t_pipe.ensure(s->dev->gpu, perChunk * recBytes, valid ? perChunk * K * 4 : 0);
  for (int i = 0; i < nst; ++i) s->wait_on(t_pipe.st[i]);
  for (size_t c = 0; c < chunks; ++c) {
    const int b = (int)(c % nst);
    cudaStream_t st = t_pipe.st[b];
    const size_t first = c * chunkRecs, cnt = std::min(chunkRecs, M - first);
    char* h = static_cast<char*>(rays) + first * recBytes;
    // the stream order serialises reuse of buffer b: its previous D2H precedes this H2D
    cuda_check(cudaMemcpyAsync(t_pipe.buf[b], h, cnt * recBytes, cudaMemcpyHostToDevice, st), "H2D rays");
    const int* dvalid = nullptr;
    if (valid) {
      cuda_check(cudaMemcpyAsync(t_pipe.vbuf[b], valid + first * K, cnt * K * 4, cudaMemcpyHostToDevice, st), "H2D valid");
      dvalid = t_pipe.vbuf[b];
    }
    rtk::TraceParams p = make_params(s, t_pipe.buf[b], dvalid, (unsigned long long)cnt * K, instID, instPrimID);
    cuda_check((cudaError_t)rtk::launch_trace(p, occluded, K, st), "trace launch");
    // closest hit: only tfar .. end of the record can have changed (K == 1: bytes 32..95; packets: fields 8..20 = the last 52 K bytes)
    const size_t skip = (!occluded && g_host_d2h_partial) ? (K == 1 ? 32 : (size_t)8 * 4 * K) : 0;
    if (skip)
      cuda_check(cudaMemcpy2DAsync(h + skip, recBytes, t_pipe.buf[b] + skip, recBytes, recBytes - skip, cnt, cudaMemcpyDeviceToHost, st), "D2H rays");
    else
      cuda_check(cudaMemcpyAsync(h, t_pipe.buf[b], cnt * recBytes, cudaMemcpyDeviceToHost, st), "D2H rays");
  }
  for (int i = 0; i < HostPipe::kStreams; ++i) cuda_check(cudaStreamSynchronize(t_pipe.st[i]), "trace");
}

// ---- filter callbacks (kernels/geometry/filter.h:15-84, intersector_epilog.h:264-280, :347-361) ----------------------
// The reference calls the geometry's filter (and / or the arguments' filter) on the host thread for every candidate hit
// it meets during traversal; a rejected candidate (valid[0] = 0) does not shorten the ray and the traversal goes on.  A
// device traversal cannot call into the host, so the same semantics are produced in passes: the FILTER instantiation of
// the trace kernel returns each ray's CLOSEST candidate that no callback has rejected yet, together with the index of
// its leaf record; the callbacks run here with N == 1 (ray.tfar = candidate distance, a separate RTCHit, the context's
// instance ids as during an instanced traversal); an accepted hit is final, a rejected one is appended to the ray's
// exclusion list and the ray is traced again.  Closest hit: the first accepted candidate in distance order is the
// closest accepted hit, which is what the reference's traversal converges to.  Occluded: the ray is occluded iff some
// candidate in [tnear, tfar] is accepted, whatever the order.  Callbacks see every candidate at most once, front to back
// (the reference's order is its traversal order and it may also call them on candidates behind the final hit).
// Packets are processed lane by lane with N == 1, which the callback contract allows (rtcore_common.h:311-324: N is an
// argument precisely because it varies).
struct LaneIO {
  char* base; int K; int occluded;
  size_t packet() const { return (size_t)(occluded ? 12 : 21) * 4 * K + (K == 1 && !occluded ? 12 : 0); }
  uint32_t* field(size_t i, int f) const { return reinterpret_cast<uint32_t*>(base + (i / K) * packet() + ((size_t)f * K + (i % K)) * 4); }
  void load(size_t i, RTCRayHit& r) const {
    uint32_t* d = reinterpret_cast<uint32_t*>(&r);
    for (int f = 0; f < 12; ++f) d[f] = *field(i, f);
    r.hit.Ng_x = r.hit.Ng_y = r.hit.Ng_z = r.hit.u = r.hit.v = 0.0f;
    r.hit.primID = r.hit.geomID = r.hit.instID[0] = RTC_INVALID_GEOMETRY_ID;
    r.hit.instPrimID[0] = RTC_INVALID_GEOMETRY_ID;
  }
  void store_hit(size_t i, const RTCRayHit& r) const {   // copyHitToRay + the distance the callback left in ray.tfar
    const uint32_t* d = reinterpret_cast<const uint32_t*>(&r);
    *field(i, 8) = d[8];
    for (int f = 12; f < 21; ++f) *field(i, f) = d[f];
  }
  void store_tfar(size_t i, float t) const { memcpy(field(i, 8), &t, 4); }
};

GeometryImpl* hit_geometry(SceneImpl* s, const RTCHit& h) {
  std::lock_guard<std::mutex> lg(s->geomMutex);
  const unsigned inst = h.instID[0];
  if (inst != RTC_INVALID_GEOMETRY_ID && inst < s->geoms.size() && s->geoms[inst] && s->geoms[inst]->type == RTC_GEOMETRY_TYPE_INSTANCE &&
      s->geoms[inst]->instScene) {
    SceneImpl* c = s->geoms[inst]->instScene;
    std::lock_guard<std::mutex> lc(c->geomMutex);
    return h.geomID < c->geoms.size() ? c->geoms[h.geomID] : nullptr;
  }
  return h.geomID < s->geoms.size() ? s->geoms[h.geomID] : nullptr;
}

// runIntersectionFilter1 / runOcclusionFilter1 (filter.h:15-84) for one candidate; true = accepted
bool run_filters(GeometryImpl* g, RTCRayHit& r, const QueryArgs& q, int occluded) {
  if (!g) return true;
  RTCFilterFunctionN gfn = occluded ? g->occludedFilter : g->intersectFilter;
  RTCFilterFunctionN afn = (q.filter && (q.enforce || g->argFilterEnabled)) ? q.filter : nullptr;
  if (!gfn && !afn) return true;
  RTCRayQueryContext fallback;
  rtcInitRayQueryContext(&fallback);
  RTCRayQueryContext* ctx = q.ctx ? q.ctx : &fallback;
  const unsigned saveI = ctx->instID[0], saveP = ctx->instPrimID[0];
  ctx->instID[0] = r.hit.instID[0]; ctx->instPrimID[0] = r.hit.instPrimID[0];   // instance_id_stack::push during an instanced traversal
  RTCHit h = r.hit;
  int mask = -1;
  RTCFilterFunctionNArguments fa;
  fa.valid = &mask; fa.geometryUserPtr = g->userPtr; fa.context = ctx;
  fa.ray = reinterpret_cast<RTCRayN*>(&r.ray); fa.hit = reinterpret_cast<RTCHitN*>(&h); fa.N = 1;
  bool ok = true;
  if (gfn) { gfn(&fa); ok = mask != 0; }
  if (ok && afn) { afn(&fa); ok = mask != 0; }
  ctx->instID[0] = saveI; ctx->instPrimID[0] = saveP;
  if (ok) r.hit = h;   // copyHitToRay: what the callback left in the hit is what the caller gets
  return ok;
}

void trace_filtered(SceneImpl* s, void* recs, const int* valid, int K, size_t M, int occluded, const QueryArgs& q) {
  require_committed(s);
  if (!s->gpu.root_valid || M == 0) return;
  t_ctx.ensure(s->dev->gpu);
  cudaSetDevice(s->dev->gpu);
  cudaStream_t st = t_ctx.stream;
  s->wait_on(st);
  const LaneIO io{static_cast<char*>(recs), K, occluded};
  const size_t total = M * (size_t)K, chunk = size_t(1) << 21;
  struct DevBuf {
    void* p = nullptr; size_t cap = 0; cudaStream_t st;
    explicit DevBuf(cudaStream_t s) : st(s) {}
    ~DevBuf() { if (p) cudaFreeAsync(p, st); }
    void* need(size_t bytes) {
      if (bytes > cap) { if (p) cudaFreeAsync(p, st); p = nullptr; cap = 0; cuda_check(cudaMallocAsync(&p, bytes, st), "cudaMallocAsync(filter pass)"); cap = bytes; }
      return p;
    }
  } dRays(st), dOff(st), dIdx(st), dWin(st);
  for (size_t first = 0; first < total; first += chunk) {
    const size_t cnt = std::min(chunk, total - first);
    std::vector<RTCRayHit> work;       // the chunk's active rays as the caller passed them
    std::vector<size_t> src;           // their lane index in the caller's records
    work.reserve(cnt); src.reserve(cnt);
    for (size_t i = first; i < first + cnt; ++i) {
      if (K > 1 && valid && valid[i] != -1) continue;           // inactive lanes stay untouched
      RTCRayHit r;
      io.load(i, r);
      if (occluded && r.ray.tfar < 0.0f) continue;               // already occluded (bvh_intersector1.cpp:128-129)
      work.push_back(r); src.push_back(i);
    }
    std::vector<std::vector<uint32_t>> excl(work.size());
    std::vector<uint32_t> active(work.size()), next;
    for (size_t j = 0; j < active.size(); ++j) active[j] = (uint32_t)j;
    std::vector<RTCRayHit> pass;
    std::vector<uint32_t> off, idx, win;
    while (!active.empty()) {
      const size_t n = active.size();
      pass.resize(n); off.assign(n + 1, 0u); idx.clear(); win.resize(n);
      for (size_t j = 0; j < n; ++j) {
        pass[j] = work[active[j]];
        off[j] = (uint32_t)idx.size();
        idx.insert(idx.end(), excl[active[j]].begin(), excl[active[j]].end());
      }
      off[n] = (uint32_t)idx.size();
      // a single ray or one packet (what a per-pixel caller such as tutorials/hair_geometry issues): the pass runs out of the calling
      // thread's mapped pinned staging block -- no allocation, no copy calls, one launch and one synchronisation, like trace_one
      constexpr size_t kSmallRays = 16, kRaysAt = 2048, kOffAt = kRaysAt + kSmallRays * sizeof(RTCRayHit), kWinAt = kOffAt + 128, kIdxAt = kWinAt + 64;
      if (n <= kSmallRays && kIdxAt + idx.size() * 4 <= ThreadCtx::kStagingBytes) {
        char* sg = t_ctx.staging;
        memcpy(sg + kRaysAt, pass.data(), n * sizeof(RTCRayHit));
        memcpy(sg + kOffAt, off.data(), (n + 1) * 4);
        if (!idx.empty()) memcpy(sg + kIdxAt, idx.data(), idx.size() * 4);
        rtk::TraceParams p = make_params(s, sg + kRaysAt, nullptr, (unsigned long long)n, q.instID, q.instPrimID);
        p.stat = nullptr;
        p.excl_off = reinterpret_cast<const uint32_t*>(sg + kOffAt); p.excl_idx = reinterpret_cast<const uint32_t*>(sg + kIdxAt);
        p.win = reinterpret_cast<uint32_t*>(sg + kWinAt);
        cuda_check((cudaError_t)rtk::launch_trace(p, 0, 1, st), "trace launch");
        cuda_check(cudaStreamSynchronize(st), "trace");
        memcpy(pass.data(), sg + kRaysAt, n * sizeof(RTCRayHit));
        memcpy(win.data(), sg + kWinAt, n * 4);
      } else {
      RTCRayHit* dr = static_cast<RTCRayHit*>(dRays.need(n * sizeof(RTCRayHit)));
      uint32_t* dof = static_cast<uint32_t*>(dOff.need((n + 1) * 4));
      uint32_t* dix = static_cast<uint32_t*>(dIdx.need(std::max<size_t>(idx.size(), 1) * 4));
      uint32_t* dwn = static_cast<uint32_t*>(dWin.need(n * 4));
      cuda_check(cudaMemcpyAsync(dr, pass.data(), n * sizeof(RTCRayHit), cudaMemcpyHostToDevice, st), "H2D rays");
      cuda_check(cudaMemcpyAsync(dof, off.data(), (n + 1) * 4, cudaMemcpyHostToDevice, st), "H2D exclusion offsets");
      if (!idx.empty()) cuda_check(cudaMemcpyAsync(dix, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, st), "H2D exclusion lists");
      rtk::TraceParams p = make_params(s, dr, nullptr, (unsigned long long)n, q.instID, q.instPrimID);
      p.stat = nullptr;
      p.excl_off = dof; p.excl_idx = dix; p.win = dwn;
      cuda_check((cudaError_t)rtk::launch_trace(p, 0, 1, st), "trace launch");
      cuda_check(cudaMemcpyAsync(pass.data(), dr, n * sizeof(RTCRayHit), cudaMemcpyDeviceToHost, st), "D2H rays");
      cuda_check(cudaMemcpyAsync(win.data(), dwn, n * 4, cudaMemcpyDeviceToHost, st), "D2H winning records");
      cuda_check(cudaStreamSynchronize(st), "trace");
      }
      next.clear();
      for (size_t j = 0; j < n; ++j) {
        RTCRayHit& r = pass[j];
        if (r.hit.geomID == RTC_INVALID_GEOMETRY_ID) continue;   // no candidate left: the caller's record stays as it was
        if (run_filters(hit_geometry(s, r.hit), r, q, occluded)) {
          if (occluded) io.store_tfar(src[active[j]], -INFINITY);   // bvh_intersector1.cpp:186-188
          else io.store_hit(src[active[j]], r);
        } else {
          excl[active[j]].push_back(win[j]);
          next.push_back(active[j]);
        }
      }
      active.swap(next);
    }
  }
}

// The filter passes name the rejected hits by record, and one record of an instance-traversal scene serves every instance of its
// instanced scene: those scenes take no filter callbacks yet.
void refuse_filters_on_instance_traversal(SceneImpl* s) {
  if (s->gpu.d_insts)
    fail(RTC_ERROR_INVALID_OPERATION, "filter callbacks are not supported on scenes committed with instance traversal (see rtcb200SetTuning \"instance_flatten_max\")");
}

// one record (single ray or one packet) / M records through host pointers: with or without filter callbacks
template <typename Args>
void query_one(SceneImpl* s, void* rec, size_t bytes, const int* valid, int K, int occluded, const Args* a) {
  const QueryArgs q = read_args(a);
  if (filters_apply(s, q, occluded)) { refuse_filters_on_instance_traversal(s); trace_filtered(s, rec, valid, K, 1, occluded, q); }
  else trace_one(s, rec, bytes, valid, K, occluded, q.instID, q.instPrimID);
}
template <typename Args>
void query_host(SceneImpl* s, void* recs, const int* valid, int K, size_t M, size_t bytes, int occluded, const Args* a) {
  const QueryArgs q = read_args(a);
  if (filters_apply(s, q, occluded)) { refuse_filters_on_instance_traversal(s); trace_filtered(s, recs, valid, K, M, occluded, q); }
  else trace_host(s, recs, valid, K, M, bytes, occluded, q.instID, q.instPrimID);
}
template <typename Args>
QueryArgs device_args(SceneImpl* s, const Args* a, int occluded) {
  const QueryArgs q = read_args(a);
  if (filters_apply(s, q, occluded)) fail(RTC_ERROR_INVALID_OPERATION, "filter callbacks are host functions: use the host-pointer entry points");
  return q;
}


}  // namespace

// =====================================================================================================================
// extern "C" entry points
// =====================================================================================================================
extern "C" {

const char* rtcGetErrorString(enum RTCError e) {
  switch (e) {
    case RTC_ERROR_NONE: return "No error";
    case RTC_ERROR_UNKNOWN: return "Unknown error";
    case RTC_ERROR_INVALID_ARGUMENT: return "Invalid argument";
    case RTC_ERROR_INVALID_OPERATION: return "Invalid operation";
    case RTC_ERROR_OUT_OF_MEMORY: return "Out of memory";
    case RTC_ERROR_UNSUPPORTED_CPU: return "Unsupported CPU";
    case RTC_ERROR_CANCELLED: return "Cancelled";
    case RTC_ERROR_LEVEL_ZERO_RAYTRACING_SUPPORT_MISSING: return "Level Zero raytracing support missing";
  }
  return "Invalid error code";
}

RTCDevice rtcNewDevice(const char* config) {
  std::lock_guard<std::mutex> lk(g_deviceMutex);
  DeviceImpl* d = nullptr;
  API_BEGIN
  d = new DeviceImpl();
  int cur = 0;
  cudaError_t e = cudaGetDevice(&cur);
  if (e != cudaSuccess) { std::string m = std::string("no CUDA device: ") + cudaGetErrorString(e); delete d; d = nullptr; fail(RTC_ERROR_UNKNOWN, m.c_str()); }
  d->gpu = cur;
  parse_config(d, config);
  int count = 0;
  cudaGetDeviceCount(&count);
  if (d->gpu < 0 || d->gpu >= count) { delete d; d = nullptr; fail(RTC_ERROR_INVALID_ARGUMENT, "gpu ordinal out of range"); }
  cuda_check(cudaGetDeviceProperties(&d->prop, d->gpu), "cudaGetDeviceProperties");
  if (d->prop.major != 9 || d->prop.minor != 0) {
    std::string m = std::string("this library contains sm_90a code only; device is ") + d->prop.name;
    delete d; d = nullptr;
    fail(RTC_ERROR_UNKNOWN, m.c_str());
  }
  if (d->verbose >= 1)
    fprintf(stderr, "Embree-API CUDA kernels %s: GPU %d %s, %d SMs, %.0f GB\n", RTC_VERSION_STRING, d->gpu, d->prop.name,
            d->prop.multiProcessorCount, d->prop.totalGlobalMem / 1e9);
  return reinterpret_cast<RTCDevice>(d);
  API_END(nullptr)
  return nullptr;
}
void rtcRetainDevice(RTCDevice h) { API_BEGIN VERIFY_HANDLE(h); std::lock_guard<std::mutex> lk(g_deviceMutex); D(h)->retain(); API_END(D(h)) }
void rtcReleaseDevice(RTCDevice h) { API_BEGIN VERIFY_HANDLE(h); std::lock_guard<std::mutex> lk(g_deviceMutex); if (D(h)->rc.load() == 1) t_err.erase(D(h)); D(h)->release(); API_END(nullptr) }

ssize_t rtcGetDeviceProperty(RTCDevice h, enum RTCDeviceProperty prop) {
  API_BEGIN
  VERIFY_HANDLE(h);
  switch (prop) {  // reference values: kernels/common/device.cpp:461-531
    case RTC_DEVICE_PROPERTY_VERSION: return RTC_VERSION;
    case RTC_DEVICE_PROPERTY_VERSION_MAJOR: return RTC_VERSION_MAJOR;
    case RTC_DEVICE_PROPERTY_VERSION_MINOR: return RTC_VERSION_MINOR;
    case RTC_DEVICE_PROPERTY_VERSION_PATCH: return RTC_VERSION_PATCH;
    case RTC_DEVICE_PROPERTY_NATIVE_RAY4_SUPPORTED:
    case RTC_DEVICE_PROPERTY_NATIVE_RAY8_SUPPORTED:
    case RTC_DEVICE_PROPERTY_NATIVE_RAY16_SUPPORTED: return 1;
    case RTC_DEVICE_PROPERTY_BACKFACE_CULLING_SPHERES_ENABLED:
    case RTC_DEVICE_PROPERTY_BACKFACE_CULLING_CURVES_ENABLED: return 0;
    case RTC_DEVICE_PROPERTY_RAY_MASK_SUPPORTED: return 1;
    case RTC_DEVICE_PROPERTY_BACKFACE_CULLING_ENABLED: return 0;
    case RTC_DEVICE_PROPERTY_FILTER_FUNCTION_SUPPORTED: return 1;  // host-pointer entry points (trace_filtered)
    case RTC_DEVICE_PROPERTY_IGNORE_INVALID_RAYS_ENABLED: return 0;
    case RTC_DEVICE_PROPERTY_COMPACT_POLYS_ENABLED: return 0;
    case RTC_DEVICE_PROPERTY_TRIANGLE_GEOMETRY_SUPPORTED: return 1;
    case RTC_DEVICE_PROPERTY_QUAD_GEOMETRY_SUPPORTED: return 1;
    case RTC_DEVICE_PROPERTY_CURVE_GEOMETRY_SUPPORTED: return 1;   // round linear curves
    case RTC_DEVICE_PROPERTY_SUBDIVISION_GEOMETRY_SUPPORTED:
    case RTC_DEVICE_PROPERTY_USER_GEOMETRY_SUPPORTED:
    case RTC_DEVICE_PROPERTY_POINT_GEOMETRY_SUPPORTED: return 1;   // sphere / disc / oriented disc points
    case RTC_DEVICE_PROPERTY_TASKING_SYSTEM: return 0;
    case RTC_DEVICE_PROPERTY_JOIN_COMMIT_SUPPORTED: return 1;
    case RTC_DEVICE_PROPERTY_PARALLEL_COMMIT_SUPPORTED: return 0;
    case RTC_DEVICE_PROPERTY_CPU_DEVICE: return 0;
    case RTC_DEVICE_PROPERTY_SYCL_DEVICE: return 0;
  }
  fail(RTC_ERROR_INVALID_ARGUMENT, "unknown readable property");
  API_END(D(h))
  return 0;
}
void rtcSetDeviceProperty(RTCDevice h, enum RTCDeviceProperty, ssize_t) {
  API_BEGIN VERIFY_HANDLE(h); fail(RTC_ERROR_INVALID_ARGUMENT, "unknown writable property"); API_END(D(h))
}
enum RTCError rtcGetDeviceError(RTCDevice h) {
  ErrSlot& s = h ? t_err[D(h)] : t_noDeviceError;
  const RTCError e = s.code;
  s.code = RTC_ERROR_NONE;
  return e;
}
const char* rtcGetDeviceLastErrorMessage(RTCDevice h) {
  ErrSlot& s = h ? t_err[D(h)] : t_noDeviceError;
  return s.msg.c_str();
}
void rtcSetDeviceErrorFunction(RTCDevice h, RTCErrorFunction fn, void* p) { API_BEGIN VERIFY_HANDLE(h); D(h)->errFn = fn; D(h)->errPtr = p; API_END(D(h)) }
void rtcSetDeviceMemoryMonitorFunction(RTCDevice h, RTCMemoryMonitorFunction fn, void* p) { API_BEGIN VERIFY_HANDLE(h); D(h)->memFn = fn; D(h)->memPtr = p; API_END(D(h)) }

// ---- buffers ------------------------------------------------------------------------------------------------------
RTCBuffer rtcNewBuffer(RTCDevice h, size_t n) { API_BEGIN VERIFY_HANDLE(h); return reinterpret_cast<RTCBuffer>(new BufferImpl(D(h), n, nullptr)); API_END(D(h)) return nullptr; }
RTCBuffer rtcNewSharedBuffer(RTCDevice h, void* ptr, size_t n) { API_BEGIN VERIFY_HANDLE(h); VERIFY_HANDLE(ptr); return reinterpret_cast<RTCBuffer>(new BufferImpl(D(h), n, ptr)); API_END(D(h)) return nullptr; }
RTCBuffer rtcNewBufferHostDevice(RTCDevice h, size_t n) { return rtcNewBuffer(h, n); }
RTCBuffer rtcNewSharedBufferHostDevice(RTCDevice h, void* p, size_t n) { return rtcNewSharedBuffer(h, p, n); }
void* rtcGetBufferData(RTCBuffer b) { DeviceImpl* d = b ? B(b)->dev : nullptr; API_BEGIN VERIFY_HANDLE(b); return B(b)->ptr; API_END(d) return nullptr; }
void* rtcGetBufferDataDevice(RTCBuffer b) { return rtcGetBufferData(b); }
void rtcCommitBuffer(RTCBuffer b) { DeviceImpl* d = b ? B(b)->dev : nullptr; API_BEGIN VERIFY_HANDLE(b); API_END(d) }
void rtcRetainBuffer(RTCBuffer b) { DeviceImpl* d = b ? B(b)->dev : nullptr; API_BEGIN VERIFY_HANDLE(b); B(b)->retain(); API_END(d) }
void rtcReleaseBuffer(RTCBuffer b) { DeviceImpl* d = b ? B(b)->dev : nullptr; API_BEGIN VERIFY_HANDLE(b); B(b)->release(); API_END(d) }

// ---- geometry -----------------------------------------------------------------------------------------------------
RTCGeometry rtcNewGeometry(RTCDevice h, enum RTCGeometryType type) {
  API_BEGIN
  VERIFY_HANDLE(h);
  if (type != RTC_GEOMETRY_TYPE_TRIANGLE && type != RTC_GEOMETRY_TYPE_QUAD && type != RTC_GEOMETRY_TYPE_INSTANCE && prim_type(type).kind == rtk::PRIM_TRIANGLE)
    fail(RTC_ERROR_INVALID_OPERATION, "only RTC_GEOMETRY_TYPE_TRIANGLE, _QUAD, _ROUND / _FLAT_LINEAR_CURVE, _ROUND / _FLAT_BEZIER / _BSPLINE / _HERMITE / _CATMULL_ROM_CURVE, _SPHERE / _DISC / _ORIENTED_DISC_POINT and _INSTANCE are supported by the CUDA back-end");
  GeometryImpl* g = new GeometryImpl(D(h));
  g->type = type;
  return reinterpret_cast<RTCGeometry>(g);
  API_END(D(h))
  return nullptr;
}
#define GEOM_BEGIN(g) DeviceImpl* dev_ = (g) ? G(g)->dev : nullptr; API_BEGIN VERIFY_HANDLE(g);
#define GEOM_END API_END(dev_)
void rtcRetainGeometry(RTCGeometry g) { GEOM_BEGIN(g) G(g)->retain(); GEOM_END }
void rtcReleaseGeometry(RTCGeometry g) { GEOM_BEGIN(g) G(g)->release(); GEOM_END }
void rtcCommitGeometry(RTCGeometry g) { GEOM_BEGIN(g) ++G(g)->modCounter; G(g)->state = GeomState::COMMITTED; GEOM_END }  // geometry.cpp:103-107
void rtcEnableGeometry(RTCGeometry g) { GEOM_BEGIN(g) if (!G(g)->enabled) { G(g)->enabled = true; ++G(g)->modCounter; } GEOM_END }
void rtcDisableGeometry(RTCGeometry g) { GEOM_BEGIN(g) if (G(g)->enabled) { G(g)->enabled = false; ++G(g)->modCounter; } GEOM_END }
// ---- rtcInterpolate / rtcInterpolateN (scene_triangle_mesh.h:49-105, scene_quad_mesh.h interpolate_impl, scene_line_segments.h:39-75,
// scene_curves.h:535-579, :699-761, geometry.cpp:163-235): host arithmetic on the caller's vertex / attribute buffers, interp.cuh's
// routine that the batched device calls run too.
static rtk::InterpKind interp_kind(RTCGeometryType t, RTCBufferType bt) {
  if (t == RTC_GEOMETRY_TYPE_TRIANGLE) return rtk::INTERP_TRIANGLE;
  if (t == RTC_GEOMETRY_TYPE_QUAD) return rtk::INTERP_QUAD;
  if (is_linear_curve(t)) return rtk::INTERP_LINEAR;
  if (is_hermite(t)) return bt == RTC_BUFFER_TYPE_VERTEX ? rtk::INTERP_HERMITE : rtk::INTERP_HERMITE_ATTRIB;
  if (curve_geometry(t)) return rtk::INTERP_CUBIC;
  return rtk::INTERP_NONE;   // points and instances (geometry.h:400-402)
}
// the buffer an interpolation of `g` reads, or NULL when `g` has no such buffer
static const BufferView* interp_buffer(const GeometryImpl* g, RTCBufferType bt, unsigned slot) {
  const BufferView* bv = nullptr;
  if (bt == RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE) { if (slot < g->attribs.size()) bv = &g->attribs[slot]; }
  else if (bt == RTC_BUFFER_TYPE_VERTEX && slot == 0) bv = &g->vertices;
  return bv && bv->buf ? bv : nullptr;
}
static void interpolate1(GeometryImpl* g, const RTCInterpolateArguments* a) {
  const rtk::InterpKind kind = interp_kind(g->type, a->bufferType);
  if (kind == rtk::INTERP_NONE) fail(RTC_ERROR_INVALID_OPERATION, "operation not supported for this geometry");
  const BufferView* bv = interp_buffer(g, a->bufferType, a->bufferSlot);
  if (!bv || !g->indices.buf || (kind == rtk::INTERP_HERMITE && !g->tangents.buf)) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer");
  if (a->primID >= g->indices.count) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid primitive ID");
  if (bv->on_device() || g->indices.on_device() || (kind == rtk::INTERP_HERMITE && g->tangents.on_device()))
    fail(RTC_ERROR_INVALID_OPERATION, "buffer is in device memory: interpolate with rtcb200InterpolateHits* or rtcb200Interpolate1");
  // dPdv travels with dPdu and the second derivatives with ddPdudu, as in the reference; a curve writes no v-derivative
  const bool curve = rtk::interp_curve(kind);
  float* const out[6] = {a->P, a->dPdu, a->dPdu && !curve ? a->dPdv : nullptr, a->ddPdudu, a->ddPdudu && !curve ? a->ddPdvdv : nullptr,
                         a->ddPdudu && !curve ? a->ddPdudv : nullptr};
  const PrimType pt = prim_type(g->type);
  rtk::interpolate_prim(kind, pt.basis, reinterpret_cast<const uint32_t*>(g->indices.data() + (size_t)a->primID * g->indices.stride),
                        reinterpret_cast<const uint8_t*>(bv->data()), bv->stride, reinterpret_cast<const uint8_t*>(g->tangents.data()),
                        g->tangents.stride, a->u, a->v, a->valueCount, out, 1);
}
void rtcInterpolate(const RTCInterpolateArguments* a) {
  GeometryImpl* g_ = a ? G(a->geometry) : nullptr;
  DeviceImpl* dev_ = g_ ? g_->dev : nullptr;
  API_BEGIN VERIFY_HANDLE(a); VERIFY_HANDLE(a->geometry); interpolate1(g_, a); API_END(dev_)
}
void rtcInterpolateN(const RTCInterpolateNArguments* a) {
  GeometryImpl* g_ = a ? G(a->geometry) : nullptr;
  DeviceImpl* dev_ = g_ ? g_->dev : nullptr;
  API_BEGIN
  VERIFY_HANDLE(a); VERIFY_HANDLE(a->geometry);
  if (a->valueCount > 256) fail(RTC_ERROR_INVALID_OPERATION, "maximally 256 floating point values can be interpolated per vertex");
  const int* valid = static_cast<const int*>(a->valid);
  float P[256], dPdu[256], dPdv[256], d2uu[256], d2vv[256], d2uv[256];
  // a curve has no v-derivatives: they are written as 0 (the reference copies whatever its scratch arrays hold)
  if (rtk::interp_curve(interp_kind(g_->type, a->bufferType))) for (unsigned j = 0; j < 256; ++j) dPdv[j] = d2vv[j] = d2uv[j] = 0.0f;
  for (unsigned i = 0; i < a->N; ++i) {
    if (valid && !valid[i]) continue;
    RTCInterpolateArguments ia;
    ia.geometry = a->geometry; ia.primID = a->primIDs[i]; ia.u = a->u[i]; ia.v = a->v[i]; ia.bufferType = a->bufferType; ia.bufferSlot = a->bufferSlot;
    ia.P = a->P ? P : nullptr; ia.dPdu = a->dPdu ? dPdu : nullptr; ia.dPdv = a->dPdu ? dPdv : nullptr;
    ia.ddPdudu = a->ddPdudu ? d2uu : nullptr; ia.ddPdvdv = a->ddPdudu ? d2vv : nullptr; ia.ddPdudv = a->ddPdudu ? d2uv : nullptr;
    ia.valueCount = a->valueCount;
    interpolate1(g_, &ia);
    for (unsigned j = 0; j < a->valueCount; ++j) {   // SoA outputs: value j of lane i at [j * N + i]
      if (a->P) a->P[j * a->N + i] = P[j];
      if (a->dPdu) { a->dPdu[j * a->N + i] = dPdu[j]; a->dPdv[j * a->N + i] = dPdv[j]; }
      if (a->ddPdudu) { a->ddPdudu[j * a->N + i] = d2uu[j]; a->ddPdvdv[j * a->N + i] = d2vv[j]; a->ddPdudv[j * a->N + i] = d2uv[j]; }
    }
  }
  API_END(dev_)
}

// ---- batched interpolation of hits (rtcb200InterpolateHits*): the scene's interpolation table and its device buffers ----------------
// Builds the entries of one (buffer type, slot) on `st`: one per geomID of `s`, then one block per instanced scene.  Device copies are
// shared between entries that read the same bytes -- host memory, or the caller's device memory copied device-to-device; curve vertex
// and tangent buffers reuse the copies the commit keeps.
static size_t format_bytes(RTCFormat f);
struct InterpTableBuild {
  SceneImpl* s;
  SceneImpl::InterpTable& t;
  cudaStream_t st;
  std::map<std::pair<const char*, size_t>, const uint8_t*> copies;   // (address, bytes) -> device copy

  const uint8_t* upload(const BufferView& v, size_t bytes) {
    const char* src = v.data();
    if (!src || bytes == 0) return nullptr;
    const std::pair<const char*, size_t> key(src, bytes);
    auto it = copies.find(key);
    if (it != copies.end()) return it->second;
    void* p = nullptr;
    cuda_check(cudaMallocAsync(&p, bytes, st), "cudaMallocAsync(interpolation buffer)");
    t.buffers.push_back(p);
    cuda_check(cudaMemcpyAsync(p, src, bytes, v.copy_kind(), st), "upload interpolation buffer");
    return copies[key] = static_cast<const uint8_t*>(p);
  }
  static size_t span(const BufferView& b) { return b.count ? (b.count - 1) * b.stride + format_bytes(b.format) : 0; }

  rtk::InterpEntry entry(const GeometryImpl* g) {
    rtk::InterpEntry e;
    if (!g || !g->enabled) return e;
    const rtk::InterpKind kind = interp_kind(g->type, t.type);
    const BufferView* bv = interp_buffer(g, t.type, t.slot);
    if (kind == rtk::INTERP_NONE || !bv || !g->indices.buf || (kind == rtk::INTERP_HERMITE && !g->tangents.buf)) return e;
    e.kind = kind; e.basis = prim_type(g->type).basis;
    e.nprims = (uint32_t)g->indices.count; e.istride = g->indices.stride;
    e.idx = upload(g->indices, g->indices.count ? (g->indices.count - 1) * g->indices.stride + 4 * rtk::interp_index_count(kind) : 0);
    auto res = s->residentCurves.find(g);
    const bool resident = t.type == RTC_BUFFER_TYPE_VERTEX && res != s->residentCurves.end();
    e.nelems = bv->count; e.dstride = bv->stride;
    e.data = resident && res->second.verts ? res->second.verts : upload(*bv, span(*bv));
    if (kind == rtk::INTERP_HERMITE) {
      e.ntang = g->tangents.count; e.tstride = g->tangents.stride;
      e.tang = resident && res->second.tangents ? res->second.tangents : upload(g->tangents, span(g->tangents));
    }
    return e;
  }

  void build() {
    std::vector<GeometryImpl*> geoms;
    { std::lock_guard<std::mutex> lg(s->geomMutex); geoms = s->geoms; }
    std::vector<rtk::InterpEntry> tab(geoms.size());
    std::unordered_map<SceneImpl*, uint32_t> blocks;   // instanced scene -> first entry of its block
    for (size_t id = 0; id < geoms.size(); ++id) {
      GeometryImpl* g = geoms[id];
      if (!g || g->type != RTC_GEOMETRY_TYPE_INSTANCE) { tab[id] = entry(g); continue; }
      if (!g->enabled || !g->instScene) continue;
      SceneImpl* c = g->instScene;
      std::vector<GeometryImpl*> cgeoms;
      { std::lock_guard<std::mutex> lc(c->geomMutex); cgeoms = c->geoms; }
      auto it = blocks.find(c);
      if (it == blocks.end()) {
        it = blocks.emplace(c, (uint32_t)tab.size()).first;
        for (GeometryImpl* cg : cgeoms) tab.push_back(cg && cg->type != RTC_GEOMETRY_TYPE_INSTANCE ? entry(cg) : rtk::InterpEntry());
      }
      tab[id].kind = rtk::INTERP_INSTANCE; tab[id].sub = it->second; tab[id].nprims = (uint32_t)cgeoms.size();
    }
    t.nentries = (uint32_t)geoms.size();
    void* p = nullptr;
    cuda_check(cudaMallocAsync(&p, std::max<size_t>(tab.size(), 1) * sizeof(rtk::InterpEntry), st), "cudaMallocAsync(interpolation table)");
    t.d_table = static_cast<rtk::InterpEntry*>(p);
    if (!tab.empty()) cuda_check(cudaMemcpyAsync(p, tab.data(), tab.size() * sizeof(rtk::InterpEntry), cudaMemcpyHostToDevice, st), "upload interpolation table");
    cuda_check(cudaStreamSynchronize(st), "upload interpolation table");   // `tab` is a local vector
  }
};

// The argument checks of rtcb200InterpolateHits*; false when there is nothing to launch.
static bool check_interpolate_hits(SceneImpl* s, const RTCB200InterpolateHitsArguments* a) {
  VERIFY_HANDLE(a);
  { std::lock_guard<std::mutex> lg(s->geomMutex); if (!s->everCommitted || s->isModified()) fail(RTC_ERROR_INVALID_OPERATION, "scene not committed"); }
  if (a->valueCount > 256) fail(RTC_ERROR_INVALID_OPERATION, "maximally 256 floating point values can be interpolated per vertex");
  if (a->bufferType == RTC_BUFFER_TYPE_VERTEX ? a->bufferSlot != 0 : a->bufferType != RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer");
  if (!a->dPdu != !a->dPdv) fail(RTC_ERROR_INVALID_ARGUMENT, "dPdu and dPdv must be requested together");
  if (!a->ddPdudu != !a->ddPdvdv || !a->ddPdudu != !a->ddPdudv) fail(RTC_ERROR_INVALID_ARGUMENT, "ddPdudu, ddPdvdv and ddPdudv must be requested together");
  if (a->M && !a->hits) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid argument");
  // a buffer narrower than valueCount floats would be read beyond its elements
  auto check = [&](const GeometryImpl* g) {
    if (!g || !g->enabled || interp_kind(g->type, a->bufferType) == rtk::INTERP_NONE) return;
    const BufferView* bv = interp_buffer(g, a->bufferType, a->bufferSlot);
    if (bv && format_bytes(bv->format) < 4 * (size_t)a->valueCount) fail(RTC_ERROR_INVALID_ARGUMENT, "buffer format holds fewer than valueCount floats");
  };
  std::lock_guard<std::mutex> lg(s->geomMutex);
  for (const GeometryImpl* g : s->geoms) {
    if (!g || g->type != RTC_GEOMETRY_TYPE_INSTANCE) { check(g); continue; }
    if (!g->instScene) continue;
    std::lock_guard<std::mutex> lc(g->instScene->geomMutex);
    for (const GeometryImpl* cg : g->instScene->geoms) check(cg);
  }
  return a->M && a->valueCount && (a->P || a->dPdu || a->ddPdudu);
}

// the scene's interpolation table for (type, slot), built on `st` by the first request since the last commit -- of the batched calls
// or of rtcb200GetSceneDeviceInterpolator, which share it; complete on the device when this returns
static SceneImpl::InterpTable* interp_table(SceneImpl* s, RTCBufferType type, unsigned slot, cudaStream_t st) {
  for (SceneImpl::InterpTable& x : s->interpTables) if (x.type == type && x.slot == slot) return &x;
  s->interpTables.push_back(SceneImpl::InterpTable{type, slot, nullptr, 0, {}});
  SceneImpl::InterpTable* t = &s->interpTables.back();
  try {
    s->wait_on(st);
    InterpTableBuild{s, *t, st, {}}.build();
  }
  catch (...) {   // a partly built table is not kept
    if (t->d_table) cudaFreeAsync(t->d_table, st);
    for (void* p : t->buffers) cudaFreeAsync(p, st);
    s->interpTables.pop_back();
    throw;
  }
  return t;
}

// enqueues the interpolation of `a` (hits and outputs in device memory) on `st`
static void interpolate_hits(SceneImpl* s, const RTCB200InterpolateHitsArguments* a, const RTCRayHit* d_hits, float* const d_out[6], cudaStream_t st) {
  const SceneImpl::InterpTable* t = interp_table(s, a->bufferType, a->bufferSlot, st);
  rtk::InterpParams p;
  p.hits = d_hits; p.M = a->M; p.table = t->d_table; p.nentries = t->nentries; p.valueCount = a->valueCount;
  for (int c = 0; c < 6; ++c) p.out[c] = d_out[c];
  cuda_check((cudaError_t)rtk::launch_interpolate(p, st), "interpolation launch");
}

// scene_curves.cpp:244-249, scene_line_segments.cpp:182-184 (linear curves store the value and never use it: tutorials/hair_geometry
// sets it on every hair set); every other geometry type: "operation not supported for this geometry" (geometry.h:382)
void rtcSetGeometryTessellationRate(RTCGeometry g, float n) {
  GEOM_BEGIN(g)
  if (!curve_geometry(G(g)->type)) fail(RTC_ERROR_INVALID_OPERATION, "operation not supported for this geometry");
  const int r = (int)n;
  G(g)->tessellationRate = r < 1 ? 1 : (r > 16 ? 16 : r);
  G(g)->update();
  GEOM_END
}
void rtcSetGeometryTimeStepCount(RTCGeometry g, unsigned int n) { GEOM_BEGIN(g) if (n != 1) fail(RTC_ERROR_INVALID_OPERATION, "motion blur is not supported by the CUDA back-end"); GEOM_END }
void rtcSetGeometryVertexAttributeCount(RTCGeometry g, unsigned int n) { GEOM_BEGIN(g) G(g)->attribs.resize(n); G(g)->update(); GEOM_END }
void rtcSetGeometryMask(RTCGeometry g, unsigned int mask) { GEOM_BEGIN(g) G(g)->mask = mask; G(g)->update(); GEOM_END }
void rtcSetGeometryBuildQuality(RTCGeometry g, enum RTCBuildQuality q) {
  GEOM_BEGIN(g)
  if (q != RTC_BUILD_QUALITY_LOW && q != RTC_BUILD_QUALITY_MEDIUM && q != RTC_BUILD_QUALITY_HIGH && q != RTC_BUILD_QUALITY_REFIT)
    throw std::runtime_error("invalid build quality");
  G(g)->quality = q; G(g)->update();
  GEOM_END
}

static void set_buffer(GeometryImpl* g, RTCBufferType type, unsigned slot, RTCFormat format, BufferImpl* buf, size_t off, size_t stride, size_t num) {
  // scene_triangle_mesh.cpp:35-80, scene_quad_mesh.cpp:35-80
  if (g->type == RTC_GEOMETRY_TYPE_INSTANCE) fail(RTC_ERROR_INVALID_OPERATION, "operation not supported for this geometry");
  const bool curve = curve_geometry(g->type);   // scene_line_segments.cpp:35-100, scene_curves.cpp:50-140
  if (type == RTC_BUFFER_TYPE_NORMAL) {   // scene_points.cpp:60-71: oriented discs only
    if (g->type != RTC_GEOMETRY_TYPE_ORIENTED_DISC_POINT) fail(RTC_ERROR_INVALID_ARGUMENT, "unknown buffer type");
    if (((size_t)(buf->ptr) + off) & 3 || (stride & 3)) fail(RTC_ERROR_INVALID_OPERATION, "data must be 4 bytes aligned");
    if (format != RTC_FORMAT_FLOAT3) fail(RTC_ERROR_INVALID_OPERATION, "invalid normal buffer format");
    if (slot != 0) fail(RTC_ERROR_INVALID_OPERATION, "invalid normal buffer slot");
    g->tangents.set(buf, off, stride, num, format);
    g->update();
    return;
  }
  if (point_geometry(g->type) && type == RTC_BUFFER_TYPE_INDEX) fail(RTC_ERROR_INVALID_ARGUMENT, "unknown buffer type");   // scene_points.cpp:82
  if (is_hermite(g->type) && type == RTC_BUFFER_TYPE_TANGENT) {
    if (((size_t)(buf->ptr) + off) & 3 || (stride & 3)) fail(RTC_ERROR_INVALID_OPERATION, "data must be 4 bytes aligned");
    if (format != RTC_FORMAT_FLOAT4) fail(RTC_ERROR_INVALID_OPERATION, "invalid tangent buffer format");
    if (slot != 0) fail(RTC_ERROR_INVALID_OPERATION, "invalid tangent buffer slot");
    g->tangents.set(buf, off, stride, num, format);
    g->update();
    return;
  }
  if (is_linear_curve(g->type) && type == RTC_BUFFER_TYPE_FLAGS) {
    if (format != RTC_FORMAT_UCHAR) fail(RTC_ERROR_INVALID_OPERATION, "invalid flag buffer format");
    if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot");
    g->flags.set(buf, off, stride, num, format);
    g->update();
    return;
  }
  if (((size_t)(buf->ptr) + off) & 3 || (stride & 3)) fail(RTC_ERROR_INVALID_OPERATION, "data must be 4 bytes aligned");
  if (num > 0xFFFFFFFFull) fail(RTC_ERROR_INVALID_ARGUMENT, "buffer too large");
  if (type == RTC_BUFFER_TYPE_VERTEX) {
    if (format != ((curve || point_geometry(g->type)) ? RTC_FORMAT_FLOAT4 : RTC_FORMAT_FLOAT3)) fail(RTC_ERROR_INVALID_OPERATION, "invalid vertex buffer format");
    if (stride * num > 16ull * 1024 * 1024 * 1024) fail(RTC_ERROR_INVALID_OPERATION, "vertex buffer can be at most 16GB large");
    if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid vertex buffer slot");
    g->vertices.set(buf, off, stride, num, format);
  } else if (type == RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE) {
    if (format < RTC_FORMAT_FLOAT || format > RTC_FORMAT_FLOAT4 + 12) fail(RTC_ERROR_INVALID_OPERATION, "invalid vertex attribute buffer format");
    if (slot >= g->attribs.size()) fail(RTC_ERROR_INVALID_OPERATION, "invalid vertex attribute buffer slot");
    g->attribs[slot].set(buf, off, stride, num, format);
  } else if (type == RTC_BUFFER_TYPE_INDEX) {
    if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot");
    if (format != (curve ? RTC_FORMAT_UINT : g->type == RTC_GEOMETRY_TYPE_QUAD ? RTC_FORMAT_UINT4 : RTC_FORMAT_UINT3)) fail(RTC_ERROR_INVALID_OPERATION, "invalid index buffer format");
    g->indices.set(buf, off, stride, num, format);
    ++g->indexVersion;
  } else
    fail(RTC_ERROR_INVALID_ARGUMENT, "unknown buffer type");
  g->update();
}
static size_t format_bytes(RTCFormat f) {
  if (f == RTC_FORMAT_UCHAR) return 1;
  if (f >= RTC_FORMAT_UINT && f <= RTC_FORMAT_UINT4) return 4 * (size_t)(f - RTC_FORMAT_UINT + 1);
  if (f >= RTC_FORMAT_FLOAT && f <= RTC_FORMAT_FLOAT4 + 12) return 4 * (size_t)(f - RTC_FORMAT_FLOAT + 1);
  fail(RTC_ERROR_INVALID_ARGUMENT, "invalid format");
}
void rtcSetGeometryBuffer(RTCGeometry g, enum RTCBufferType type, unsigned int slot, enum RTCFormat format, RTCBuffer buffer, size_t off, size_t stride, size_t num) {
  GEOM_BEGIN(g)
  VERIFY_HANDLE(buffer);
  if (G(g)->dev != B(buffer)->dev) fail(RTC_ERROR_INVALID_ARGUMENT, "inputs are from different devices");
  if (num > 0 && off + (num - 1) * stride + format_bytes(format) > B(buffer)->bytes) fail(RTC_ERROR_INVALID_ARGUMENT, "buffer range out of bounds");  // rtcore.cpp rtcSetGeometryBuffer
  set_buffer(G(g), type, slot, format, B(buffer), off, stride, num);
  GEOM_END
}
void rtcSetSharedGeometryBuffer(RTCGeometry g, enum RTCBufferType type, unsigned int slot, enum RTCFormat format, const void* ptr, size_t off, size_t stride, size_t num) {
  GEOM_BEGIN(g)
  if (num > 0) VERIFY_HANDLE(ptr);
  BufferImpl* b = new BufferImpl(G(g)->dev, off + (num ? (num - 1) * stride + format_bytes(format) : 0), const_cast<void*>(ptr ? ptr : (const void*)g));
  try { set_buffer(G(g), type, slot, format, b, off, stride, num); } catch (...) { b->release(); throw; }
  b->release();
  GEOM_END
}
// The same view of memory on the library's GPU: the buffer is marked as device memory and set_buffer checks it as any other; the
// commit and the interpolation tables copy it device-to-device (BufferView::copy_kind).
void rtcb200SetSharedGeometryBufferDevice(RTCGeometry g, enum RTCBufferType type, unsigned int slot, enum RTCFormat format, const void* d_ptr, size_t off,
                                          size_t stride, size_t num) {
  GEOM_BEGIN(g)
  if (num > 0 && !d_ptr) fail(RTC_ERROR_INVALID_ARGUMENT, "device pointer is NULL");
  if (d_ptr) {
    cudaPointerAttributes at{};
    const cudaError_t e = cudaPointerGetAttributes(&at, d_ptr);
    if (e != cudaSuccess) cudaGetLastError();   // not a pointer CUDA knows: host memory
    const bool ok = e == cudaSuccess && (at.type == cudaMemoryTypeManaged || (at.type == cudaMemoryTypeDevice && at.device == G(g)->dev->gpu));
    if (!ok) fail(RTC_ERROR_INVALID_ARGUMENT, "pointer is not device or managed memory on the device's GPU");
  }
  BufferImpl* b = new BufferImpl(G(g)->dev, off + (num ? (num - 1) * stride + format_bytes(format) : 0), const_cast<void*>(d_ptr ? d_ptr : (const void*)g));
  b->device = true;
  if (!d_ptr) b->ptr = nullptr;   // an empty view: no address, so the getters return NULL and nothing is copied from it
  try { set_buffer(G(g), type, slot, format, b, off, stride, num); } catch (...) { b->release(); throw; }
  b->release();
  GEOM_END
}
void* rtcSetNewGeometryBuffer(RTCGeometry g, enum RTCBufferType type, unsigned int slot, enum RTCFormat format, size_t stride, size_t num) {
  GEOM_BEGIN(g)
  size_t bytes = num * stride;
  if (type == RTC_BUFFER_TYPE_VERTEX || type == RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE) bytes += (16 - (stride % 16)) % 16;  // rtcore.cpp: vertex buffers get padding
  BufferImpl* b = new BufferImpl(G(g)->dev, bytes, nullptr);
  try { set_buffer(G(g), type, slot, format, b, 0, stride, num); } catch (...) { b->release(); throw; }
  void* p = b->ptr;
  b->release();
  return p;
  GEOM_END
  return nullptr;
}
// the view rtcGetGeometryBufferData[Device] reads
static const BufferView& geometry_buffer(GeometryImpl* g, RTCBufferType type, unsigned slot) {
  const BufferView* v = nullptr;
  if (type == RTC_BUFFER_TYPE_INDEX) { if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot"); v = &g->indices; }
  else if (type == RTC_BUFFER_TYPE_VERTEX) { if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot"); v = &g->vertices; }
  else if (type == RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE) { if (slot >= g->attribs.size()) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot"); v = &g->attribs[slot]; }
  else if (type == RTC_BUFFER_TYPE_FLAGS && is_linear_curve(g->type)) { if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot"); v = &g->flags; }
  else if ((type == RTC_BUFFER_TYPE_TANGENT && is_hermite(g->type)) || (type == RTC_BUFFER_TYPE_NORMAL && g->type == RTC_GEOMETRY_TYPE_ORIENTED_DISC_POINT)) { if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot"); v = &g->tangents; }
  else fail(RTC_ERROR_INVALID_ARGUMENT, "unknown buffer type");
  return *v;
}
void* rtcGetGeometryBufferData(RTCGeometry g, enum RTCBufferType type, unsigned int slot) {
  GEOM_BEGIN(g)
  const BufferView& v = geometry_buffer(G(g), type, slot);
  if (v.on_device()) fail(RTC_ERROR_INVALID_OPERATION, "buffer is in device memory: it has no host address (rtcGetGeometryBufferDataDevice)");
  return const_cast<char*>(v.data());
  GEOM_END
  return nullptr;
}
// a host buffer's host address (its host copy is the source, as for the *HostDevice buffers); a device buffer's device address
void* rtcGetGeometryBufferDataDevice(RTCGeometry g, enum RTCBufferType type, unsigned int slot) {
  GEOM_BEGIN(g)
  return const_cast<char*>(geometry_buffer(G(g), type, slot).data());
  GEOM_END
  return nullptr;
}
void rtcUpdateGeometryBuffer(RTCGeometry g, enum RTCBufferType type, unsigned int slot) {
  GEOM_BEGIN(g)
  if (type == RTC_BUFFER_TYPE_INDEX || type == RTC_BUFFER_TYPE_VERTEX || type == RTC_BUFFER_TYPE_FLAGS || type == RTC_BUFFER_TYPE_TANGENT || type == RTC_BUFFER_TYPE_NORMAL) { if (slot != 0) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot"); }
  else if (type == RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE) { if (slot >= G(g)->attribs.size()) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid buffer slot"); }
  else fail(RTC_ERROR_INVALID_ARGUMENT, "unknown buffer type");
  if (type == RTC_BUFFER_TYPE_INDEX) ++G(g)->indexVersion;
  G(g)->update();
  GEOM_END
}
void rtcSetGeometryUserData(RTCGeometry g, void* p) { GEOM_BEGIN(g) G(g)->userPtr = p; GEOM_END }
void* rtcGetGeometryUserData(RTCGeometry g) { GEOM_BEGIN(g) return G(g)->userPtr; GEOM_END return nullptr; }
// filter callbacks (rtcore.cpp:2188-2216; geometry.cpp:142-156): stored on the geometry, no commit needed; instances take none
static void check_filter_geometry(GeometryImpl* g) { if (g->type == RTC_GEOMETRY_TYPE_INSTANCE) fail(RTC_ERROR_INVALID_OPERATION, "filter functions not supported for this geometry"); }
void rtcSetGeometryEnableFilterFunctionFromArguments(RTCGeometry g, bool e) { GEOM_BEGIN(g) G(g)->set_filter([&] { G(g)->argFilterEnabled = e; }); GEOM_END }
void rtcSetGeometryIntersectFilterFunction(RTCGeometry g, RTCFilterFunctionN f) { GEOM_BEGIN(g) check_filter_geometry(G(g)); G(g)->set_filter([&] { G(g)->intersectFilter = f; }); GEOM_END }
void rtcSetGeometryOccludedFilterFunction(RTCGeometry g, RTCFilterFunctionN f) { GEOM_BEGIN(g) check_filter_geometry(G(g)); G(g)->set_filter([&] { G(g)->occludedFilter = f; }); GEOM_END }

// ---- scene --------------------------------------------------------------------------------------------------------
#define SCENE_BEGIN(s) DeviceImpl* dev_ = (s) ? S(s)->dev : nullptr; API_BEGIN VERIFY_HANDLE(s);
#define SCENE_END API_END(dev_)
RTCScene rtcNewScene(RTCDevice h) { API_BEGIN VERIFY_HANDLE(h); return reinterpret_cast<RTCScene>(new SceneImpl(D(h))); API_END(D(h)) return nullptr; }
RTCDevice rtcGetSceneDevice(RTCScene s) { SCENE_BEGIN(s) S(s)->dev->retain(); return reinterpret_cast<RTCDevice>(S(s)->dev); SCENE_END return nullptr; }
void rtcRetainScene(RTCScene s) { SCENE_BEGIN(s) S(s)->retain(); SCENE_END }
void rtcReleaseScene(RTCScene s) { SCENE_BEGIN(s) S(s)->release(); SCENE_END }
RTCTraversable rtcGetSceneTraversable(RTCScene s) {
  SCENE_BEGIN(s)
  if (!S(s)->everCommitted) fail(RTC_ERROR_INVALID_OPERATION, "Traversable is NULL. The scene has to be committed first.");
  return reinterpret_cast<RTCTraversable>(s);
  SCENE_END
  return nullptr;
}
static void attach_at(SceneImpl* s, GeometryImpl* g, unsigned id) {
  if (s->dev != g->dev) fail(RTC_ERROR_INVALID_ARGUMENT, "inputs are from different devices");
  if (id >= s->geoms.size()) s->geoms.resize((size_t)id + 1, nullptr);
  if (s->geoms[id]) fail(RTC_ERROR_INVALID_ARGUMENT, "geometry ID already in use");  // scene.cpp bind()
  g->retain();
  s->geoms[id] = g;
  s->flagsModified = true;
}
unsigned int rtcAttachGeometry(RTCScene s, RTCGeometry g) {
  SCENE_BEGIN(s)
  VERIFY_HANDLE(g);
  std::lock_guard<std::mutex> lk(S(s)->geomMutex);
  unsigned id = 0;
  while (id < S(s)->geoms.size() && S(s)->geoms[id]) ++id;  // lowest free ID, as the reference's IDPool
  attach_at(S(s), G(g), id);
  return id;
  SCENE_END
  return RTC_INVALID_GEOMETRY_ID;
}
void rtcAttachGeometryByID(RTCScene s, RTCGeometry g, unsigned int id) {
  SCENE_BEGIN(s)
  VERIFY_HANDLE(g);
  if (id == RTC_INVALID_GEOMETRY_ID) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid argument");
  std::lock_guard<std::mutex> lk(S(s)->geomMutex);
  attach_at(S(s), G(g), id);
  SCENE_END
}
void rtcDetachGeometry(RTCScene s, unsigned int id) {
  SCENE_BEGIN(s)
  if (id == RTC_INVALID_GEOMETRY_ID) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid argument");
  std::lock_guard<std::mutex> lk(S(s)->geomMutex);
  if (id >= S(s)->geoms.size() || !S(s)->geoms[id]) fail(RTC_ERROR_INVALID_OPERATION, "invalid geometry");
  S(s)->geoms[id]->release();
  S(s)->geoms[id] = nullptr;
  S(s)->flagsModified = true;
  SCENE_END
}
RTCGeometry rtcGetGeometry(RTCScene s, unsigned int id) {
  SCENE_BEGIN(s)
  if (id >= S(s)->geoms.size() || !S(s)->geoms[id]) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid geometry ID");
  return reinterpret_cast<RTCGeometry>(S(s)->geoms[id]);
  SCENE_END
  return nullptr;
}
RTCGeometry rtcGetGeometryThreadSafe(RTCScene s, unsigned int id) {
  SCENE_BEGIN(s)
  std::lock_guard<std::mutex> lk(S(s)->geomMutex);
  if (id >= S(s)->geoms.size() || !S(s)->geoms[id]) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid geometry ID");
  return reinterpret_cast<RTCGeometry>(S(s)->geoms[id]);
  SCENE_END
  return nullptr;
}
void* rtcGetGeometryUserDataFromScene(RTCScene s, unsigned int id) {
  SCENE_BEGIN(s)
  if (id >= S(s)->geoms.size() || !S(s)->geoms[id]) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid geometry ID");
  return S(s)->geoms[id]->userPtr;
  SCENE_END
  return nullptr;
}
// one commit path: on the legacy default stream, waiting for its work; settle() takes a stream commit still pending (one that this
// call found nothing to redo after)
void rtcCommitScene(RTCScene s) { SCENE_BEGIN(s) commit_scene(S(s), 0, true); S(s)->settle(); SCENE_END }
void rtcJoinCommitScene(RTCScene s) { rtcCommitScene(s); }
void rtcb200CommitSceneWithStream(RTCScene s, void* cuda_stream) {
  SCENE_BEGIN(s)
  const cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  // the commit's host bookkeeping would not replay with a captured graph: refused before anything is enqueued
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  S(s)->dev->use();
  cuda_check(cudaStreamIsCapturing(st, &capture), "cudaStreamIsCapturing");
  if (capture != cudaStreamCaptureStatusNone) fail(RTC_ERROR_INVALID_OPERATION, "the stream is capturing a CUDA graph: commits cannot be captured");
  commit_scene(S(s), st, false);
  SCENE_END
}
void rtcSetSceneProgressMonitorFunction(RTCScene s, RTCProgressMonitorFunction fn, void* p) { SCENE_BEGIN(s) S(s)->progFn = fn; S(s)->progPtr = p; SCENE_END }
void rtcSetSceneBuildQuality(RTCScene s, enum RTCBuildQuality q) {
  SCENE_BEGIN(s)
  if (q != RTC_BUILD_QUALITY_LOW && q != RTC_BUILD_QUALITY_MEDIUM && q != RTC_BUILD_QUALITY_HIGH) throw std::runtime_error("invalid build quality");
  if (S(s)->quality != q) { S(s)->quality = q; S(s)->flagsModified = true; }
  SCENE_END
}
void rtcSetSceneFlags(RTCScene s, enum RTCSceneFlags f) { SCENE_BEGIN(s) if (S(s)->flags != f) { S(s)->flags = f; S(s)->flagsModified = true; } SCENE_END }
enum RTCSceneFlags rtcGetSceneFlags(RTCScene s) { SCENE_BEGIN(s) return S(s)->flags; SCENE_END return RTC_SCENE_FLAG_NONE; }
void rtcGetSceneBounds(RTCScene s, struct RTCBounds* b) {
  SCENE_BEGIN(s)
  VERIFY_HANDLE(b);
  { std::lock_guard<std::mutex> lk(S(s)->geomMutex); if (S(s)->isModified()) fail(RTC_ERROR_INVALID_OPERATION, "scene not committed"); }
  S(s)->settle();
  const float* g = S(s)->apiBounds;
  b->lower_x = g[0]; b->lower_y = g[1]; b->lower_z = g[2]; b->align0 = 0;
  b->upper_x = g[3]; b->upper_y = g[4]; b->upper_z = g[5]; b->align1 = 0;
  SCENE_END
}
void rtcGetSceneLinearBounds(RTCScene s, struct RTCLinearBounds* b) {
  SCENE_BEGIN(s)
  VERIFY_HANDLE(b);
  rtcGetSceneBounds(s, &b->bounds0);
  b->bounds1 = b->bounds0;
  SCENE_END
}

// ---- queries.  No argument checks, like the reference's release build (rtcore.cpp:604-608); failures inside
// (uncommitted scene, CUDA errors) are reported through the device error slot. -----------------------------------
#define QUERY(scene, body) \
  SceneImpl* s_ = S(scene); \
  DeviceImpl* dev_ = s_ ? s_->dev : nullptr; \
  API_BEGIN body API_END(dev_)

void rtcIntersect1(RTCScene sc, struct RTCRayHit* rh, struct RTCIntersectArguments* a) { QUERY(sc, query_one(s_, rh, 96, nullptr, 1, 0, a);) }
void rtcIntersect4(const int* v, RTCScene sc, struct RTCRayHit4* rh, struct RTCIntersectArguments* a) { QUERY(sc, query_one(s_, rh, sizeof(RTCRayHit4), v, 4, 0, a);) }
void rtcIntersect8(const int* v, RTCScene sc, struct RTCRayHit8* rh, struct RTCIntersectArguments* a) { QUERY(sc, query_one(s_, rh, sizeof(RTCRayHit8), v, 8, 0, a);) }
void rtcIntersect16(const int* v, RTCScene sc, struct RTCRayHit16* rh, struct RTCIntersectArguments* a) { QUERY(sc, query_one(s_, rh, sizeof(RTCRayHit16), v, 16, 0, a);) }
void rtcOccluded1(RTCScene sc, struct RTCRay* r, struct RTCOccludedArguments* a) { QUERY(sc, query_one(s_, r, 48, nullptr, 1, 1, a);) }
void rtcOccluded4(const int* v, RTCScene sc, struct RTCRay4* r, struct RTCOccludedArguments* a) { QUERY(sc, query_one(s_, r, sizeof(RTCRay4), v, 4, 1, a);) }
void rtcOccluded8(const int* v, RTCScene sc, struct RTCRay8* r, struct RTCOccludedArguments* a) { QUERY(sc, query_one(s_, r, sizeof(RTCRay8), v, 8, 1, a);) }
void rtcOccluded16(const int* v, RTCScene sc, struct RTCRay16* r, struct RTCOccludedArguments* a) { QUERY(sc, query_one(s_, r, sizeof(RTCRay16), v, 16, 1, a);) }

void rtcTraversableIntersect1(RTCTraversable t, struct RTCRayHit* rh, struct RTCIntersectArguments* a) { rtcIntersect1(reinterpret_cast<RTCScene>(t), rh, a); }
void rtcTraversableIntersect4(const int* v, RTCTraversable t, struct RTCRayHit4* rh, struct RTCIntersectArguments* a) { rtcIntersect4(v, reinterpret_cast<RTCScene>(t), rh, a); }
void rtcTraversableIntersect8(const int* v, RTCTraversable t, struct RTCRayHit8* rh, struct RTCIntersectArguments* a) { rtcIntersect8(v, reinterpret_cast<RTCScene>(t), rh, a); }
void rtcTraversableIntersect16(const int* v, RTCTraversable t, struct RTCRayHit16* rh, struct RTCIntersectArguments* a) { rtcIntersect16(v, reinterpret_cast<RTCScene>(t), rh, a); }
void rtcTraversableOccluded1(RTCTraversable t, struct RTCRay* r, struct RTCOccludedArguments* a) { rtcOccluded1(reinterpret_cast<RTCScene>(t), r, a); }
void rtcTraversableOccluded4(const int* v, RTCTraversable t, struct RTCRay4* r, struct RTCOccludedArguments* a) { rtcOccluded4(v, reinterpret_cast<RTCScene>(t), r, a); }
void rtcTraversableOccluded8(const int* v, RTCTraversable t, struct RTCRay8* r, struct RTCOccludedArguments* a) { rtcOccluded8(v, reinterpret_cast<RTCScene>(t), r, a); }
void rtcTraversableOccluded16(const int* v, RTCTraversable t, struct RTCRay16* r, struct RTCOccludedArguments* a) { rtcOccluded16(v, reinterpret_cast<RTCScene>(t), r, a); }

// ---- batched extension ---------------------------------------------------------------------------------------------
static void check_K(unsigned K) { if (K != 4 && K != 8 && K != 16) fail(RTC_ERROR_INVALID_ARGUMENT, "packet width must be 4, 8 or 16"); }
void rtcb200Intersect1M(RTCScene sc, struct RTCRayHit* rh, size_t M, struct RTCIntersectArguments* a) { QUERY(sc, query_host(s_, rh, nullptr, 1, M, 96, 0, a);) }
void rtcb200Occluded1M(RTCScene sc, struct RTCRay* r, size_t M, struct RTCOccludedArguments* a) { QUERY(sc, query_host(s_, r, nullptr, 1, M, 48, 1, a);) }
void rtcb200IntersectNM(const int* v, RTCScene sc, void* rh, unsigned int K, size_t M, struct RTCIntersectArguments* a) { QUERY(sc, check_K(K); query_host(s_, rh, v, (int)K, M, (size_t)84 * K, 0, a);) }
void rtcb200OccludedNM(const int* v, RTCScene sc, void* r, unsigned int K, size_t M, struct RTCOccludedArguments* a) { QUERY(sc, check_K(K); query_host(s_, r, v, (int)K, M, (size_t)48 * K, 1, a);) }
void rtcb200Intersect1MDevice(RTCScene sc, struct RTCRayHit* rh, size_t M, struct RTCIntersectArguments* a, void* st) { QUERY(sc, const QueryArgs q = device_args(s_, a, 0); trace_device(s_, rh, nullptr, 1, M, 0, q.instID, q.instPrimID, (cudaStream_t)st, true);) }
void rtcb200Intersect1MGatherDevice(RTCScene sc, struct RTCRayHit* rh, size_t M, struct RTCIntersectArguments* a, void* st, void* compact_out) { QUERY(sc, const QueryArgs q = device_args(s_, a, 0); VERIFY_HANDLE(compact_out); trace_gather(s_, rh, M, q.instID, q.instPrimID, (cudaStream_t)st, compact_out);) }
void rtcb200Occluded1MDevice(RTCScene sc, struct RTCRay* r, size_t M, struct RTCOccludedArguments* a, void* st) { QUERY(sc, const QueryArgs q = device_args(s_, a, 1); trace_device(s_, r, nullptr, 1, M, 1, q.instID, q.instPrimID, (cudaStream_t)st, true);) }
void rtcb200IntersectNMDevice(const int* v, RTCScene sc, void* rh, unsigned int K, size_t M, struct RTCIntersectArguments* a, void* st) { QUERY(sc, check_K(K); const QueryArgs q = device_args(s_, a, 0); trace_device(s_, rh, v, (int)K, M, 0, q.instID, q.instPrimID, (cudaStream_t)st, true);) }
void rtcb200OccludedNMDevice(const int* v, RTCScene sc, void* r, unsigned int K, size_t M, struct RTCOccludedArguments* a, void* st) { QUERY(sc, check_K(K); const QueryArgs q = device_args(s_, a, 1); trace_device(s_, r, v, (int)K, M, 1, q.instID, q.instPrimID, (cudaStream_t)st, true);) }

void rtcb200InterpolateHitsDevice(RTCScene sc, const struct RTCB200InterpolateHitsArguments* a, void* st) {
  SceneImpl* s_ = S(sc);
  DeviceImpl* dev_ = s_ ? s_->dev : nullptr;
  API_BEGIN
    VERIFY_HANDLE(s_);
    std::lock_guard<std::mutex> lk(s_->commitMutex);
    if (check_interpolate_hits(s_, a)) {
      s_->dev->use();
      float* const out[6] = {a->P, a->dPdu, a->dPdv, a->ddPdudu, a->ddPdvdv, a->ddPdudv};
      interpolate_hits(s_, a, a->hits, out, (cudaStream_t)st);
    }
  API_END(dev_)
}
void rtcb200InterpolateHits(RTCScene sc, const struct RTCB200InterpolateHitsArguments* a) {
  SceneImpl* s_ = S(sc);
  DeviceImpl* dev_ = s_ ? s_->dev : nullptr;
  API_BEGIN
    VERIFY_HANDLE(s_);
    std::lock_guard<std::mutex> lk(s_->commitMutex);
    if (check_interpolate_hits(s_, a)) {
      t_ctx.ensure(s_->dev->gpu);
      cudaStream_t st = t_ctx.stream;
      // one device block: the hits, then every requested output (which starts as the caller's, so misses keep their values)
      float* const host[6] = {a->P, a->dPdu, a->dPdv, a->ddPdudu, a->ddPdvdv, a->ddPdudv};
      const size_t outBytes = a->M * a->valueCount * sizeof(float), hitBytes = a->M * sizeof(RTCRayHit);
      size_t bytes = hitBytes;
      for (float* h : host) if (h) bytes += outBytes;
      char* d = nullptr;
      cuda_check(cudaMallocAsync(reinterpret_cast<void**>(&d), bytes, st), "cudaMallocAsync(interpolation I/O)");
      try {
        cuda_check(cudaMemcpyAsync(d, a->hits, hitBytes, cudaMemcpyHostToDevice, st), "H2D hits");
        float* dev[6] = {};
        size_t off = hitBytes;
        for (int c = 0; c < 6; ++c)
          if (host[c]) {
            dev[c] = reinterpret_cast<float*>(d + off); off += outBytes;
            cuda_check(cudaMemcpyAsync(dev[c], host[c], outBytes, cudaMemcpyHostToDevice, st), "H2D outputs");
          }
        interpolate_hits(s_, a, reinterpret_cast<const RTCRayHit*>(d), dev, st);
        for (int c = 0; c < 6; ++c)
          if (host[c]) cuda_check(cudaMemcpyAsync(host[c], dev[c], outBytes, cudaMemcpyDeviceToHost, st), "D2H outputs");
        cuda_check(cudaStreamSynchronize(st), "interpolate");
      } catch (...) { cudaFreeAsync(d, st); throw; }
      cudaFreeAsync(d, st);
    }
  API_END(dev_)
}

void rtcb200GetSceneStats(RTCScene sc, struct RTCB200SceneStats* o) {
  SCENE_BEGIN(sc)
  VERIFY_HANDLE(o);
  SceneImpl* s = S(sc);
  s->settle();
  memset(o, 0, sizeof *o);
  o->num_triangles = s->gpu.num_tris; o->num_nodes = s->gpu.num_nodes;
  o->node_bytes = (unsigned long long)s->gpu.num_nodes * sizeof(rtk::Node8);
  o->tri_bytes = (unsigned long long)s->gpu.num_tris * sizeof(rtk::TriRec);
  o->build_ms = s->gpu.build_ms; o->sah_cost = s->gpu.sah_cost; o->builder = s->gpu.builder; o->max_depth = s->gpu.max_depth;
  if (s->gpu.d_stat) {
    s->dev->use();
    unsigned long long c[3];
    cuda_check(cudaMemcpy(c, s->gpu.d_stat, sizeof c, cudaMemcpyDeviceToHost), "read stat counters");
    o->trav_rays = c[0]; o->trav_nodes = c[1]; o->trav_tris = c[2];
  }
  SCENE_END
}
// What device code reads about a scene's geometries, in one allocation (embree4_b200.h RTCB200DeviceGeometryHeader):
//  - the header: where the geomID block is and how many ids it covers;
//  - what the argument filters read about the geometry of a record (RTCB200DeviceGeometry), one entry per value of a record's b.w:
//    the geomID in a triangle-only scene, the descriptor index otherwise, an instanced descriptor taking its child geometry's
//    values -- the geometry hit_geometry() finds for the host-pointer path.  The returned pointer is its first entry;
//  - the geomID block the shading getters read (RTCB200DeviceGeometryInfo): user data, and an instance's local-to-world transform.
// User data, the filter switch and transforms change without a commit, so every call takes them anew; unchanged contents are not
// uploaded twice.  Called with commitMutex held.
static const RTCB200DeviceGeometry* geometry_snapshot(SceneImpl* s) {
  std::vector<RTCB200DeviceGeometry> tab;
  std::vector<RTCB200DeviceGeometryInfo> ids;
  auto entry = [](const GeometryImpl* g) {
    RTCB200DeviceGeometry e;
    memset(&e, 0, sizeof e);
    if (g) { e.userPtr = g->userPtr; e.argFilterEnabled = g->argFilterEnabled ? 1u : 0u; }
    return e;
  };
  {
    std::lock_guard<std::mutex> lg(s->geomMutex);
    for (const GeometryImpl* g : s->geoms) {
      RTCB200DeviceGeometryInfo e;
      memset(&e, 0, sizeof e);
      if (g) {
        e.userPtr = g->userPtr;
        e.isInstance = g->type == RTC_GEOMETRY_TYPE_INSTANCE ? 1u : 0u;
        if (e.isInstance) memcpy(e.xfm, g->xfm, sizeof e.xfm);
      }
      ids.push_back(e);
    }
    if (!s->gpu.general) {
      for (const GeometryImpl* g : s->geoms) tab.push_back(entry(g));
    } else {
      for (const auto& id : s->descIds) {
        const GeometryImpl* g = nullptr;
        if (id.second == RTC_INVALID_GEOMETRY_ID) g = id.first < s->geoms.size() ? s->geoms[id.first] : nullptr;
        else if (id.second < s->geoms.size() && s->geoms[id.second] && s->geoms[id.second]->instScene) {
          SceneImpl* c = s->geoms[id.second]->instScene;
          std::lock_guard<std::mutex> lc(c->geomMutex);
          g = id.first < c->geoms.size() ? c->geoms[id.first] : nullptr;
        }
        tab.push_back(entry(g));
      }
    }
  }
  if (tab.empty()) tab.push_back(entry(nullptr));
  static_assert(sizeof(RTCB200DeviceGeometryHeader) == sizeof(RTCB200DeviceGeometry), "the header takes the place of one entry");
  const size_t head = sizeof(RTCB200DeviceGeometryHeader), tabBytes = tab.size() * sizeof(RTCB200DeviceGeometry);
  std::vector<unsigned char> blob(head + tabBytes + ids.size() * sizeof(RTCB200DeviceGeometryInfo));
  memcpy(blob.data() + head, tab.data(), tabBytes);
  if (!ids.empty()) memcpy(blob.data() + head + tabBytes, ids.data(), ids.size() * sizeof(RTCB200DeviceGeometryInfo));
  // the header holds the allocation's own address: the contents after it decide whether the last snapshot still holds
  if (!s->geomTables.empty() && blob.size() == s->lastGeomTable.size() &&
      memcmp(blob.data() + head, s->lastGeomTable.data() + head, blob.size() - head) == 0)
    return reinterpret_cast<const RTCB200DeviceGeometry*>(static_cast<const char*>(s->geomTables.back()) + head);
  // on the calling thread's own non-blocking stream: the upload waits for no other work, and is complete when the getter returns
  // (the caller's kernels run on streams of their own)
  s->dev->use();
  t_ctx.ensure(s->dev->gpu);
  void* p = nullptr;
  cuda_check(cudaMallocAsync(&p, blob.size(), t_ctx.stream), "cudaMallocAsync(geometry table)");
  s->geomTables.push_back(p);
  RTCB200DeviceGeometryHeader h;
  memset(&h, 0, sizeof h);
  h.byGeomID = ids.empty() ? nullptr : reinterpret_cast<const RTCB200DeviceGeometryInfo*>(static_cast<const char*>(p) + head + tabBytes);
  h.count = (unsigned)ids.size();
  memcpy(blob.data(), &h, head);
  cuda_check(cudaMemcpyAsync(p, blob.data(), blob.size(), cudaMemcpyHostToDevice, t_ctx.stream), "upload geometry table");
  cuda_check(cudaStreamSynchronize(t_ctx.stream), "upload geometry table");
  s->lastGeomTable.swap(blob);
  return reinterpret_cast<const RTCB200DeviceGeometry*>(static_cast<const char*>(p) + head);
}

// the arrays trace_device hands the kernel (make_params), for device-side queries; refused where trace_device would refuse
void rtcb200GetSceneDeviceTraversable(RTCScene sc, struct RTCB200DeviceTraversable* o) {
  SCENE_BEGIN(sc)
  VERIFY_HANDLE(o);
  memset(o, 0, sizeof *o);
  SceneImpl* s = S(sc);
  std::lock_guard<std::mutex> lk(s->commitMutex);
  if (!s->everCommitted) fail(RTC_ERROR_INVALID_OPERATION, "Traversable is NULL. The scene has to be committed first.");
  const QueryArgs none;   // no arguments' filter: only the geometries' own callbacks count
  if (filters_apply(s, none, 0) || filters_apply(s, none, 1))
    fail(RTC_ERROR_INVALID_OPERATION, "filter callbacks are host functions: device-side queries cannot call them");
  const rtk::SceneGPU& g = s->gpu;
  if (g.d_insts)
    fail(RTC_ERROR_INVALID_OPERATION, "device-side queries do not support scenes committed with instance traversal (see rtcb200SetTuning \"instance_flatten_max\")");
  bool any;   // a scene without primitives still answers its geometries' user data
  { std::lock_guard<std::mutex> lg(s->geomMutex); any = !s->geoms.empty(); }
  const RTCB200DeviceGeometry* geoms = any ? geometry_snapshot(s) : nullptr;
  o->nodes = g.nodes; o->records = g.tris;
  o->descs = g.general ? g.d_descs : nullptr;
  o->root_valid = g.root_valid; o->robust = (unsigned)g.robust; o->general = (unsigned short)g.general; o->curves = (unsigned)g.curves;
  o->device = (short)s->dev->gpu;
  o->geometries = geoms;
  SCENE_END
}
// the interpolation table the batched calls use for (type, slot), for rtcb200Interpolate1 in the caller's kernels; refused where the
// batched calls refuse the scene or the buffer
void rtcb200GetSceneDeviceInterpolator(RTCScene sc, enum RTCBufferType type, unsigned int slot, struct RTCB200DeviceInterpolator* o) {
  SCENE_BEGIN(sc)
  VERIFY_HANDLE(o);
  memset(o, 0, sizeof *o);
  SceneImpl* s = S(sc);
  std::lock_guard<std::mutex> lk(s->commitMutex);
  { std::lock_guard<std::mutex> lg(s->geomMutex); if (!s->everCommitted || s->isModified()) fail(RTC_ERROR_INVALID_OPERATION, "scene not committed"); }
  if (type == RTC_BUFFER_TYPE_VERTEX ? slot != 0 : type != RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE) fail(RTC_ERROR_INVALID_OPERATION, "invalid buffer");
  // built on the calling thread's own stream, like the geometry snapshot: the caller's kernels run on streams of their own
  s->dev->use();
  t_ctx.ensure(s->dev->gpu);
  const SceneImpl::InterpTable* t = interp_table(s, type, slot, t_ctx.stream);
  o->table = t->d_table; o->nentries = t->nentries;
  SCENE_END
}
static void scene_layout(const rtk::SceneGPU& g, RTCB200SceneLayout* o) {
  memset(o, 0, sizeof *o);
  if (g.root_valid) {
    o->num_nodes = g.num_nodes; o->num_records = g.num_tris;
    o->num_descs = g.d_descs ? g.num_descs : 0u;
    o->num_levels = (unsigned)g.levels.size();
    o->num_subs = g.builder == rtk::BUILDER_TWO_LEVEL ? (unsigned)g.subs.size() : 0u;
    o->top_nodes = g.builder == rtk::BUILDER_TWO_LEVEL ? g.top_cap : 0u;
  }
  o->max_depth = g.max_depth; o->general = (unsigned)g.general; o->robust = (unsigned)g.robust; o->builder = g.builder;
}
void rtcb200GetSceneLayout(RTCScene sc, struct RTCB200SceneLayout* o) { SCENE_BEGIN(sc) VERIFY_HANDLE(o); S(sc)->settle(); scene_layout(S(sc)->gpu, o); SCENE_END }
void rtcb200CopySceneArrays(RTCScene sc, void* nodes, void* records, struct RTCB200DescInfo* descs, unsigned int* levels, unsigned int* subs) {
  SCENE_BEGIN(sc)
  SceneImpl* s = S(sc);
  s->settle();
  const rtk::SceneGPU& g = s->gpu;
  RTCB200SceneLayout lay;
  scene_layout(g, &lay);
  s->dev->use();
  if (nodes && lay.num_nodes) cuda_check(cudaMemcpy(nodes, g.nodes, (size_t)lay.num_nodes * sizeof(rtk::Node8), cudaMemcpyDeviceToHost), "copy nodes");
  if (records && lay.num_records) cuda_check(cudaMemcpy(records, g.tris, (size_t)lay.num_records * sizeof(rtk::TriRec), cudaMemcpyDeviceToHost), "copy records");
  if (descs && lay.num_descs) {
    std::vector<rtk::GeomDesc> d(lay.num_descs);
    cuda_check(cudaMemcpy(d.data(), g.d_descs, d.size() * sizeof(rtk::GeomDesc), cudaMemcpyDeviceToHost), "copy descriptors");
    unsigned first = 0;
    for (size_t i = 0; i < d.size(); ++i) {
      RTCB200DescInfo& o = descs[i];
      o.geomID = d[i].geomID; o.instID = d[i].instID; o.kind = d[i].kind; o.first = first; o.count = d[i].ntris;
      o.is_quad = d[i].is_quad; o.tess = d[i].tess; o.basis = d[i].basis; o.hermite = d[i].hermite;
      memcpy(o.xfm, d[i].xfm, sizeof o.xfm);
      first += d[i].ntris;
    }
  }
  if (levels) for (unsigned l = 0; l < lay.num_levels; ++l) levels[l] = g.levels[l];
  if (subs)
    for (unsigned i = 0; i < lay.num_subs; ++i) {
      subs[4 * i] = g.subs[i].node_off; subs[4 * i + 1] = g.subs[i].tri_off;
      subs[4 * i + 2] = g.subs[i].nodes; subs[4 * i + 3] = g.subs[i].tris;
    }
  SCENE_END
}
void rtcb200SetSceneStatCounters(RTCScene sc, int enable) { SCENE_BEGIN(sc) S(sc)->statCounters = enable != 0; SCENE_END }
void rtcb200ResetSceneStatCounters(RTCScene sc) { SCENE_BEGIN(sc) if (S(sc)->gpu.d_stat) { S(sc)->dev->use(); cuda_check(cudaMemset(S(sc)->gpu.d_stat, 0, 24), "reset stat counters"); } SCENE_END }
unsigned long long rtcb200GetLaunchCount(void) { return rtk::launch_count(); }

// ---- peer-visible device buffers for the fused multi-GPU hit gather (one process per GPU: CUDA IPC over NVLink) ----
void* rtcb200PeerAlloc(RTCDevice h, size_t bytes) {
  API_BEGIN
  VERIFY_HANDLE(h);
  D(h)->use();
  void* p = nullptr;
  cuda_check(cudaMalloc(&p, bytes ? bytes : 16), "cudaMalloc(peer buffer)");
  return p;
  API_END(D(h))
  return nullptr;
}
void rtcb200PeerFree(RTCDevice h, void* p) { API_BEGIN VERIFY_HANDLE(h); D(h)->use(); if (p) cuda_check(cudaFree(p), "cudaFree(peer buffer)"); API_END(D(h)) }
int rtcb200PeerExport(RTCDevice h, void* p, unsigned char handle[64]) {
  API_BEGIN
  VERIFY_HANDLE(h); VERIFY_HANDLE(p); VERIFY_HANDLE(handle);
  D(h)->use();
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t ih;
  cuda_check(cudaIpcGetMemHandle(&ih, p), "cudaIpcGetMemHandle");
  memcpy(handle, &ih, 64);
  return 0;
  API_END(D(h))
  return -1;
}
void* rtcb200PeerImport(RTCDevice h, const unsigned char handle[64]) {
  API_BEGIN
  VERIFY_HANDLE(h); VERIFY_HANDLE(handle);
  D(h)->use();
  cudaIpcMemHandle_t ih;
  memcpy(&ih, handle, 64);
  void* p = nullptr;
  cuda_check(cudaIpcOpenMemHandle(&p, ih, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
  return p;
  API_END(D(h))
  return nullptr;
}
void rtcb200PeerCopy(RTCDevice h, void* dst, const void* src, size_t bytes) {
  API_BEGIN VERIFY_HANDLE(h); D(h)->use(); cuda_check(cudaMemcpy(dst, src, bytes, cudaMemcpyDefault), "cudaMemcpy(peer buffer)"); API_END(D(h))
}
void rtcb200PeerClose(RTCDevice h, void* p) { API_BEGIN VERIFY_HANDLE(h); D(h)->use(); if (p) cuda_check(cudaIpcCloseMemHandle(p), "cudaIpcCloseMemHandle"); API_END(D(h)) }
int rtcb200SetTuning(const char* key, int value) {
  if (!key) return -1;
  rtk::Tuning& t = rtk::tuning();
  if (!strcmp(key, "collapse_policy")) t.collapse_policy = value;
  else if (!strcmp(key, "refill_min")) t.refill_min = value;
  else if (!strcmp(key, "sah_small")) t.sah_small = value;
  else if (!strcmp(key, "instance_flatten_max") && value >= 0) t.instance_flatten_max = value;
  else if (!strcmp(key, "c_node")) t.c_node = value;
  else if (!strcmp(key, "c_tri")) t.c_tri = value;
  else if (!strcmp(key, "tri_batch_min")) t.tri_batch_min = value;
  else if (!strcmp(key, "tri_wait_max")) t.tri_wait_max = value;
  else if (!strcmp(key, "curve_batch_min")) t.curve_batch_min = value;
  else if (!strcmp(key, "curve_wait_max")) t.curve_wait_max = value;
  else if (!strcmp(key, "blocks_per_sm")) t.blocks_per_sm = value;
  else if (!strcmp(key, "curve_blocks_per_sm")) t.curve_blocks_per_sm = value;
  else if (!strcmp(key, "point_batch_min")) t.point_batch_min = value;
  else if (!strcmp(key, "point_wait_max")) t.point_wait_max = value;
  else if (!strcmp(key, "use_tma")) t.use_tma = value;
  else if (!strcmp(key, "tri_spread")) t.tri_spread = value != 0;
  else if (!strcmp(key, "tri_spread_occluded")) t.tri_spread_occluded = value != 0;
  else if (!strcmp(key, "gather_mode") && value >= 0 && value <= 1) t.gather_mode = value;
  else if (!strcmp(key, "host_d2h_partial")) g_host_d2h_partial = value != 0;
  else if (!strcmp(key, "host_chunk_log2") && value >= 10 && value <= 26) g_host_chunk_log2 = value;
  else if (!strcmp(key, "host_streams") && value >= 1 && value <= HostPipe::kStreams) g_host_streams = value;
  else return -1;
  return 0;
}
double rtcb200GetLastTraceMs(RTCScene sc) {
  SCENE_BEGIN(sc)
  SceneImpl* s = S(sc);
  if (!s->ev0) return -1.0;
  s->dev->use();
  cuda_check(cudaEventSynchronize(s->ev1), "event sync");
  float ms = 0;
  cuda_check(cudaEventElapsedTime(&ms, s->ev0, s->ev1), "event elapsed");
  return ms;
  SCENE_END
  return -1.0;
}

// ---- instancing (rtcore_geometry.h:231-250, kernels/common/rtcore.cpp:1408-1515) ----------------------------------
static void load_transform(RTCFormat format, const float* x, float out[12]) {   // loadTransform, rtcore.cpp:1408-1439
  switch ((int)format) {
    case 0x9134: { const float m[12] = {x[0], x[4], x[8], x[1], x[5], x[9], x[2], x[6], x[10], x[3], x[7], x[11]}; memcpy(out, m, sizeof m); break; }  // FLOAT3X4_ROW_MAJOR
    case 0x9234: memcpy(out, x, 12 * sizeof(float)); break;                                                                                          // FLOAT3X4_COLUMN_MAJOR
    case 0x9244: { const float m[12] = {x[0], x[1], x[2], x[4], x[5], x[6], x[8], x[9], x[10], x[12], x[13], x[14]}; memcpy(out, m, sizeof m); break; }  // FLOAT4X4_COLUMN_MAJOR
    default: fail(RTC_ERROR_INVALID_OPERATION, "invalid matrix format");
  }
}
static void store_transform(const float m[12], RTCFormat format, float* x) {    // storeTransform: transform_format.cuh, shared with the device
  if (!rtk::store_transform(m, (unsigned)format, x)) fail(RTC_ERROR_INVALID_OPERATION, "invalid matrix format");
}
void rtcSetGeometryInstancedScene(RTCGeometry g, RTCScene scene) {
  GEOM_BEGIN(g)
  VERIFY_HANDLE(scene);
  if (G(g)->type != RTC_GEOMETRY_TYPE_INSTANCE) fail(RTC_ERROR_INVALID_OPERATION, "operation not supported for this geometry");
  if (G(g)->dev != S(scene)->dev) fail(RTC_ERROR_INVALID_ARGUMENT, "inputs are from different devices");
  S(scene)->retain();
  if (G(g)->instScene) G(g)->instScene->release();
  G(g)->instScene = S(scene);
  G(g)->update();
  GEOM_END
}
void rtcSetGeometryTransform(RTCGeometry g, unsigned int timeStep, enum RTCFormat format, const void* xfm) {
  GEOM_BEGIN(g)
  VERIFY_HANDLE(xfm);
  if (G(g)->type != RTC_GEOMETRY_TYPE_INSTANCE) fail(RTC_ERROR_INVALID_OPERATION, "operation not supported for this geometry");
  if (timeStep != 0) fail(RTC_ERROR_INVALID_OPERATION, "invalid timestep");
  load_transform(format, static_cast<const float*>(xfm), G(g)->xfm);
  G(g)->update_world2local();
  G(g)->update();
  GEOM_END
}
void rtcGetGeometryTransform(RTCGeometry g, float, enum RTCFormat format, void* xfm) {
  GEOM_BEGIN(g)
  VERIFY_HANDLE(xfm);
  store_transform(G(g)->xfm, format, static_cast<float*>(xfm));
  GEOM_END
}
void rtcGetGeometryTransformEx(RTCGeometry g, unsigned int, float time, enum RTCFormat format, void* xfm) { rtcGetGeometryTransform(g, time, format, xfm); }
void rtcGetGeometryTransformFromScene(RTCScene s, unsigned int id, float time, enum RTCFormat format, void* xfm) {
  SCENE_BEGIN(s)
  if (id >= S(s)->geoms.size() || !S(s)->geoms[id]) fail(RTC_ERROR_INVALID_ARGUMENT, "invalid geometry ID");
  rtcGetGeometryTransform(reinterpret_cast<RTCGeometry>(S(s)->geoms[id]), time, format, xfm);
  SCENE_END
}
void rtcGetGeometryTransformFromTraversable(RTCTraversable t, unsigned int id, float time, enum RTCFormat format, void* xfm) {
  rtcGetGeometryTransformFromScene(reinterpret_cast<RTCScene>(t), id, time, format, xfm);
}

// ---- entry points of the reference that are thin variants of supported ones -----------------------------------------
void rtcSetSharedGeometryBufferHostDevice(RTCGeometry g, enum RTCBufferType type, unsigned int slot, enum RTCFormat format, const void* ptr,
                                          const void* /*dptr*/, size_t off, size_t stride, size_t num) {
  rtcSetSharedGeometryBuffer(g, type, slot, format, ptr, off, stride, num);   // buffers are uploaded at commit; the host copy is the source
}
void rtcSetNewGeometryBufferHostDevice(RTCGeometry g, enum RTCBufferType type, unsigned int slot, enum RTCFormat format, size_t stride,
                                       size_t num, void** ptr, void** dptr) {
  void* p = rtcSetNewGeometryBuffer(g, type, slot, format, stride, num);
  if (ptr) *ptr = p;
  if (dptr) *dptr = p;
}
void* rtcGetGeometryUserDataFromTraversable(RTCTraversable t, unsigned int id) { return rtcGetGeometryUserDataFromScene(reinterpret_cast<RTCScene>(t), id); }
void rtcSetGeometryTimeRange(RTCGeometry g, float, float) { GEOM_BEGIN(g) G(g)->update(); GEOM_END }          // one time step only
void rtcSetGeometryMaxRadiusScale(RTCGeometry g, float) { GEOM_BEGIN(g) G(g)->update(); GEOM_END }            // curves/points only

// ---- everything else the reference library exports (other geometry types, user callbacks, point queries, rtcBuildBVH,
// instancing, interpolation): exported so that ANY Embree 4 caller links against this library; each call records
// RTC_ERROR_INVALID_OPERATION (thread error slot, read with rtcGetDeviceError(NULL)) and returns 0 / NULL / false.
#define RTCB200_UNSUPPORTED(name)                                                                              \
  void* name(void) {                                                                                           \
    process_error(nullptr, RTC_ERROR_INVALID_OPERATION, #name " is not supported by the CUDA triangle back-end"); \
    return nullptr;                                                                                            \
  }
RTCB200_UNSUPPORTED(rtcBuildBVH)
RTCB200_UNSUPPORTED(rtcCollide)
RTCB200_UNSUPPORTED(rtcForwardIntersect1)
RTCB200_UNSUPPORTED(rtcForwardIntersect16)
RTCB200_UNSUPPORTED(rtcForwardIntersect16Ex)
RTCB200_UNSUPPORTED(rtcForwardIntersect1Ex)
RTCB200_UNSUPPORTED(rtcForwardIntersect4)
RTCB200_UNSUPPORTED(rtcForwardIntersect4Ex)
RTCB200_UNSUPPORTED(rtcForwardIntersect8)
RTCB200_UNSUPPORTED(rtcForwardIntersect8Ex)
RTCB200_UNSUPPORTED(rtcForwardOccluded1)
RTCB200_UNSUPPORTED(rtcForwardOccluded16)
RTCB200_UNSUPPORTED(rtcForwardOccluded16Ex)
RTCB200_UNSUPPORTED(rtcForwardOccluded1Ex)
RTCB200_UNSUPPORTED(rtcForwardOccluded4)
RTCB200_UNSUPPORTED(rtcForwardOccluded4Ex)
RTCB200_UNSUPPORTED(rtcForwardOccluded8)
RTCB200_UNSUPPORTED(rtcForwardOccluded8Ex)
RTCB200_UNSUPPORTED(rtcGetGeometryFace)
RTCB200_UNSUPPORTED(rtcGetGeometryFirstHalfEdge)
RTCB200_UNSUPPORTED(rtcGetGeometryNextHalfEdge)
RTCB200_UNSUPPORTED(rtcGetGeometryOppositeHalfEdge)
RTCB200_UNSUPPORTED(rtcGetGeometryPreviousHalfEdge)
RTCB200_UNSUPPORTED(rtcInvokeIntersectFilterFromGeometry)
RTCB200_UNSUPPORTED(rtcInvokeOccludedFilterFromGeometry)
RTCB200_UNSUPPORTED(rtcMakeStaticBVH)
RTCB200_UNSUPPORTED(rtcNewBVH)
RTCB200_UNSUPPORTED(rtcPointQuery)
RTCB200_UNSUPPORTED(rtcPointQuery16)
RTCB200_UNSUPPORTED(rtcPointQuery4)
RTCB200_UNSUPPORTED(rtcPointQuery8)
RTCB200_UNSUPPORTED(rtcReleaseBVH)
RTCB200_UNSUPPORTED(rtcRetainBVH)
RTCB200_UNSUPPORTED(rtcSetGeometryBoundsFunction)
RTCB200_UNSUPPORTED(rtcSetGeometryDisplacementFunction)
RTCB200_UNSUPPORTED(rtcSetGeometryInstancedScenes)
RTCB200_UNSUPPORTED(rtcSetGeometryIntersectFunction)
RTCB200_UNSUPPORTED(rtcSetGeometryOccludedFunction)
RTCB200_UNSUPPORTED(rtcSetGeometryPointQueryFunction)
RTCB200_UNSUPPORTED(rtcSetGeometrySubdivisionMode)
RTCB200_UNSUPPORTED(rtcSetGeometryTopologyCount)
RTCB200_UNSUPPORTED(rtcSetGeometryTransformQuaternion)
RTCB200_UNSUPPORTED(rtcSetGeometryUserPrimitiveCount)
RTCB200_UNSUPPORTED(rtcSetGeometryVertexAttributeTopology)
RTCB200_UNSUPPORTED(rtcThreadLocalAlloc)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect1)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect16)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect16Ex)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect1Ex)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect4)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect4Ex)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect8)
RTCB200_UNSUPPORTED(rtcTraversableForwardIntersect8Ex)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded1)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded16)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded16Ex)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded1Ex)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded4)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded4Ex)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded8)
RTCB200_UNSUPPORTED(rtcTraversableForwardOccluded8Ex)
RTCB200_UNSUPPORTED(rtcTraversablePointQuery)
RTCB200_UNSUPPORTED(rtcTraversablePointQuery16)
RTCB200_UNSUPPORTED(rtcTraversablePointQuery4)
RTCB200_UNSUPPORTED(rtcTraversablePointQuery8)

}  // extern "C"
