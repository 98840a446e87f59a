/* embree4_b200.h -- the C-ABI of the H100-native ray tracing kernel library.
 *
 * This is the drop-in boundary: a caller compiled against Embree 4.4.1's own
 * include/embree4/rtcore.h links against libembree4_b200.so unchanged for the
 * triangle-mesh hot path (device/scene/geometry/buffer objects, rtcCommitScene,
 * rtcIntersect1/4/8/16, rtcOccluded1/4/8/16).  Every declaration below is
 * binary compatible with -- and cites -- the reference interface it replaces
 * (paths relative to the reference tree; configuration of kernels/rtcore_config.h.in:
 * RTC_MAX_INSTANCE_LEVEL_COUNT=1, EMBREE_GEOMETRY_INSTANCE_ARRAY defined, EMBREE_MIN_WIDTH=0).
 *
 * Only plain C types cross this boundary: no C++ classes, no torch types.
 * Section B is the batched / device-pointer extension ("rtcb200*") that the
 * throughput configurations use; Embree 4 dropped its stream API
 * (CHANGELOG.md:101) so there is no reference symbol for it.
 */
#ifndef EMBREE4_B200_H
#define EMBREE4_B200_H

#include <stddef.h>
#include <stdbool.h>
#include <sys/types.h> /* ssize_t, as include/embree4/rtcore_common.h:8 */

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define RTCB200_ALIGN(n) __attribute__((aligned(n)))
#define RTCB200_API __attribute__((visibility("default")))
#else
#define RTCB200_ALIGN(n)
#define RTCB200_API
#endif

/* ---- version / constants (kernels/rtcore_config.h.in:10-16, rtcore_common.h:51-54) ---- */
#define RTC_VERSION_MAJOR 4
#define RTC_VERSION_MINOR 4
#define RTC_VERSION_PATCH 1
#define RTC_VERSION 40401
#define RTC_VERSION_STRING "4.4.1"
#define RTC_MAX_INSTANCE_LEVEL_COUNT 1
#define RTC_GEOMETRY_INSTANCE_ARRAY 1
#define RTC_INVALID_GEOMETRY_ID ((unsigned int)-1)

/* ---- opaque handles (rtcore_device.h:10-11, rtcore_scene.h:12-15, rtcore_buffer.h:36) ---- */
typedef struct RTCDeviceTy* RTCDevice;
typedef struct RTCSceneTy* RTCScene;
typedef struct RTCGeometryTy* RTCGeometry;
typedef struct RTCBufferTy* RTCBuffer;
typedef struct RTCTraversableTy* RTCTraversable; /* on this back-end == the scene, as scene.cpp:928-935 */

/* ---- enums: only the enumerators the triangle path can legally receive are named; values are the
 *      reference's (rtcore_common.h:57-197, rtcore_device.h:49-100, rtcore_geometry.h:18-51,
 *      rtcore_buffer.h:11-33, rtcore_scene.h:24-32) ---- */
enum RTCFormat {
  RTC_FORMAT_UNDEFINED = 0,
  RTC_FORMAT_UCHAR = 0x1001,       /* curve neighbour flags */
  RTC_FORMAT_UINT = 0x5001, RTC_FORMAT_UINT2, RTC_FORMAT_UINT3, RTC_FORMAT_UINT4,
  RTC_FORMAT_FLOAT = 0x9001, RTC_FORMAT_FLOAT2, RTC_FORMAT_FLOAT3, RTC_FORMAT_FLOAT4,
  RTC_FORMAT_FLOAT3X4_ROW_MAJOR = 0x9134, RTC_FORMAT_FLOAT3X4_COLUMN_MAJOR = 0x9234, RTC_FORMAT_FLOAT4X4_COLUMN_MAJOR = 0x9244
};
enum RTCBuildQuality {
  RTC_BUILD_QUALITY_LOW = 0,    /* -> device LBVH (Morton) build      */
  RTC_BUILD_QUALITY_MEDIUM = 1, /* -> device binned-SAH build         */
  RTC_BUILD_QUALITY_HIGH = 2,   /* accepted; built as MEDIUM          */
  RTC_BUILD_QUALITY_REFIT = 3   /* geometry quality: later commits with unchanged topology refit the kept BVH (bvh_refit.cpp) */
};
enum RTCSceneFlags {
  RTC_SCENE_FLAG_NONE = 0,
  RTC_SCENE_FLAG_DYNAMIC = 1 << 0,
  RTC_SCENE_FLAG_COMPACT = 1 << 1,
  RTC_SCENE_FLAG_ROBUST = 1 << 2,
  RTC_SCENE_FLAG_FILTER_FUNCTION_IN_ARGUMENTS = 1 << 3,
  RTC_SCENE_FLAG_PREFETCH_USM_SHARED_ON_GPU = 1 << 4
};
enum RTCRayQueryFlags {
  RTC_RAY_QUERY_FLAG_NONE = 0,
  RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER = 1 << 1,
  RTC_RAY_QUERY_FLAG_INCOHERENT = 0 << 16,
  RTC_RAY_QUERY_FLAG_COHERENT = 1 << 16
};
enum RTCFeatureFlags {
  RTC_FEATURE_FLAG_NONE = 0,
  RTC_FEATURE_FLAG_TRIANGLE = 1 << 1,
  RTC_FEATURE_FLAG_QUAD = 1 << 2,
  RTC_FEATURE_FLAG_ROUND_LINEAR_CURVE = 1 << 6,
  RTC_FEATURE_FLAG_FLAT_LINEAR_CURVE = 1 << 7,
  RTC_FEATURE_FLAG_ROUND_BEZIER_CURVE = 1 << 8, RTC_FEATURE_FLAG_ROUND_BSPLINE_CURVE = 1 << 11,
  RTC_FEATURE_FLAG_ROUND_HERMITE_CURVE = 1 << 14, RTC_FEATURE_FLAG_ROUND_CATMULL_ROM_CURVE = 1 << 17,
  RTC_FEATURE_FLAG_FLAT_BEZIER_CURVE = 1 << 9, RTC_FEATURE_FLAG_FLAT_BSPLINE_CURVE = 1 << 12,
  RTC_FEATURE_FLAG_FLAT_HERMITE_CURVE = 1 << 15, RTC_FEATURE_FLAG_FLAT_CATMULL_ROM_CURVE = 1 << 18,
  RTC_FEATURE_FLAG_SPHERE_POINT = 1 << 20, RTC_FEATURE_FLAG_DISC_POINT = 1 << 21, RTC_FEATURE_FLAG_ORIENTED_DISC_POINT = 1 << 22,
  RTC_FEATURE_FLAG_INSTANCE = 1 << 23,
  RTC_FEATURE_FLAG_ALL = 0xffffffff
};
enum RTCGeometryType {
  RTC_GEOMETRY_TYPE_TRIANGLE = 0,
  RTC_GEOMETRY_TYPE_QUAD = 1,      /* index buffer RTC_FORMAT_UINT4; intersected as the halves (v0,v1,v3), (v2,v1,v3) */
  RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE = 16, /* vertex buffer RTC_FORMAT_FLOAT4 (xyz, radius), index buffer RTC_FORMAT_UINT = first vertex
                                                of a segment, optional RTC_BUFFER_TYPE_FLAGS (rtcore_geometry.h:27; roundline_intersector.h) */
  RTC_GEOMETRY_TYPE_FLAT_LINEAR_CURVE = 17,  /* same buffers, ray-facing ribbons (line_intersector.h) */
  /* flat cubic curves (rtcore_geometry.h:31,35,39,47; curve_intersector_ribbon.h): vertex buffer RTC_FORMAT_FLOAT4 (xyz, radius),
   * index buffer RTC_FORMAT_UINT = first of the curve's four control vertices (Hermite: of its two vertex / tangent pairs,
   * tangents in RTC_BUFFER_TYPE_TANGENT, RTC_FORMAT_FLOAT4); ray-facing ribbons of rtcSetGeometryTessellationRate (default 4,
   * 1..16) segments; hits report u along the curve, v in [-1, 1] across the ribbon and Ng = dP/du */
  RTC_GEOMETRY_TYPE_FLAT_BEZIER_CURVE = 25,
  RTC_GEOMETRY_TYPE_FLAT_BSPLINE_CURVE = 33,
  RTC_GEOMETRY_TYPE_FLAT_HERMITE_CURVE = 41,
  RTC_GEOMETRY_TYPE_FLAT_CATMULL_ROM_CURVE = 59,
  /* round cubic curves (rtcore_geometry.h:30,34,38,46; curve_intersector_sweep.h): the same buffers; the curve is the sweep of a
   * sphere of radius r(u) along P(u), intersected by the reference's cylinder-bounded subdivision + Newton iteration; hits
   * report u along the curve, v = 0 and the surface normal */
  RTC_GEOMETRY_TYPE_ROUND_BEZIER_CURVE = 24,
  RTC_GEOMETRY_TYPE_ROUND_BSPLINE_CURVE = 32,
  RTC_GEOMETRY_TYPE_ROUND_HERMITE_CURVE = 40,
  RTC_GEOMETRY_TYPE_ROUND_CATMULL_ROM_CURVE = 58,
  /* point primitives (rtcore_geometry.h:42-44; sphere_intersector.h, disc_intersector.h): vertex buffer RTC_FORMAT_FLOAT4 (centre,
   * radius), one primitive per vertex, no index buffer; oriented discs add RTC_BUFFER_TYPE_NORMAL (RTC_FORMAT_FLOAT3), one
   * normal per vertex.  Hits report u = v = 0; Ng = the sphere normal, -ray direction (ray-facing disc) or the disc normal */
  RTC_GEOMETRY_TYPE_SPHERE_POINT = 50,
  RTC_GEOMETRY_TYPE_DISC_POINT = 51,
  RTC_GEOMETRY_TYPE_ORIENTED_DISC_POINT = 52,
  RTC_GEOMETRY_TYPE_INSTANCE = 121 /* single-level instances of triangle scenes (rtcore_geometry.h:51) */
};
enum RTCBufferType { RTC_BUFFER_TYPE_INDEX = 0, RTC_BUFFER_TYPE_VERTEX = 1, RTC_BUFFER_TYPE_VERTEX_ATTRIBUTE = 2, RTC_BUFFER_TYPE_NORMAL = 3, RTC_BUFFER_TYPE_TANGENT = 4, RTC_BUFFER_TYPE_FLAGS = 32 };
enum RTCCurveFlags { RTC_CURVE_FLAG_NEIGHBOR_LEFT = 1 << 0, RTC_CURVE_FLAG_NEIGHBOR_RIGHT = 1 << 1 };   /* rtcore_geometry.h:66-70 */
enum RTCError {
  RTC_ERROR_NONE = 0, RTC_ERROR_UNKNOWN = 1, RTC_ERROR_INVALID_ARGUMENT = 2, RTC_ERROR_INVALID_OPERATION = 3,
  RTC_ERROR_OUT_OF_MEMORY = 4, RTC_ERROR_UNSUPPORTED_CPU = 5, RTC_ERROR_CANCELLED = 6,
  RTC_ERROR_LEVEL_ZERO_RAYTRACING_SUPPORT_MISSING = 7
};
enum RTCDeviceProperty {
  RTC_DEVICE_PROPERTY_VERSION = 0, RTC_DEVICE_PROPERTY_VERSION_MAJOR = 1, RTC_DEVICE_PROPERTY_VERSION_MINOR = 2,
  RTC_DEVICE_PROPERTY_VERSION_PATCH = 3,
  RTC_DEVICE_PROPERTY_NATIVE_RAY4_SUPPORTED = 32, RTC_DEVICE_PROPERTY_NATIVE_RAY8_SUPPORTED = 33,
  RTC_DEVICE_PROPERTY_NATIVE_RAY16_SUPPORTED = 34,
  RTC_DEVICE_PROPERTY_BACKFACE_CULLING_SPHERES_ENABLED = 62, RTC_DEVICE_PROPERTY_BACKFACE_CULLING_CURVES_ENABLED = 63,
  RTC_DEVICE_PROPERTY_RAY_MASK_SUPPORTED = 64, RTC_DEVICE_PROPERTY_BACKFACE_CULLING_ENABLED = 65,
  RTC_DEVICE_PROPERTY_FILTER_FUNCTION_SUPPORTED = 66, RTC_DEVICE_PROPERTY_IGNORE_INVALID_RAYS_ENABLED = 67,
  RTC_DEVICE_PROPERTY_COMPACT_POLYS_ENABLED = 68,
  RTC_DEVICE_PROPERTY_TRIANGLE_GEOMETRY_SUPPORTED = 96, RTC_DEVICE_PROPERTY_QUAD_GEOMETRY_SUPPORTED = 97,
  RTC_DEVICE_PROPERTY_SUBDIVISION_GEOMETRY_SUPPORTED = 98, RTC_DEVICE_PROPERTY_CURVE_GEOMETRY_SUPPORTED = 99,
  RTC_DEVICE_PROPERTY_USER_GEOMETRY_SUPPORTED = 100, RTC_DEVICE_PROPERTY_POINT_GEOMETRY_SUPPORTED = 101,
  RTC_DEVICE_PROPERTY_TASKING_SYSTEM = 128, RTC_DEVICE_PROPERTY_JOIN_COMMIT_SUPPORTED = 129,
  RTC_DEVICE_PROPERTY_PARALLEL_COMMIT_SUPPORTED = 130,
  RTC_DEVICE_PROPERTY_CPU_DEVICE = 140, RTC_DEVICE_PROPERTY_SYCL_DEVICE = 141
};

/* ---- I/O records.  Layouts of rtcore_ray.h:11-52 (single) and :55-184 (packets):
 *      sizeof(RTCRay)=48, sizeof(RTCHit)=48, sizeof(RTCRayHit)=96, sizeof(RTCRayHit16)=1344. ---- */
struct RTCB200_ALIGN(16) RTCRay {
  float org_x, org_y, org_z, tnear;
  float dir_x, dir_y, dir_z, time;
  float tfar; unsigned int mask, id, flags;
};
struct RTCB200_ALIGN(16) RTCHit {
  float Ng_x, Ng_y, Ng_z, u, v;
  unsigned int primID, geomID, instID[RTC_MAX_INSTANCE_LEVEL_COUNT], instPrimID[RTC_MAX_INSTANCE_LEVEL_COUNT];
};
struct RTCRayHit { struct RTCRay ray; struct RTCHit hit; };

#define RTCB200_PACKET(K, A)                                                                             \
  struct RTCB200_ALIGN(A) RTCRay##K {                                                                    \
    float org_x[K], org_y[K], org_z[K], tnear[K], dir_x[K], dir_y[K], dir_z[K], time[K], tfar[K];       \
    unsigned int mask[K], id[K], flags[K];                                                               \
  };                                                                                                     \
  struct RTCB200_ALIGN(A) RTCHit##K {                                                                    \
    float Ng_x[K], Ng_y[K], Ng_z[K], u[K], v[K];                                                         \
    unsigned int primID[K], geomID[K], instID[RTC_MAX_INSTANCE_LEVEL_COUNT][K],                          \
        instPrimID[RTC_MAX_INSTANCE_LEVEL_COUNT][K];                                                     \
  };                                                                                                     \
  struct RTCRayHit##K { struct RTCRay##K ray; struct RTCHit##K hit; };
RTCB200_PACKET(4, 16)
RTCB200_PACKET(8, 32)
RTCB200_PACKET(16, 64)

struct RTCB200_ALIGN(16) RTCBounds { /* rtcore_common.h:163-167 */
  float lower_x, lower_y, lower_z, align0, upper_x, upper_y, upper_z, align1;
};
struct RTCB200_ALIGN(16) RTCLinearBounds { struct RTCBounds bounds0, bounds1; };

/* per-query context and arguments (rtcore_common.h:335-361, rtcore_scene.h:34-86).  `filter` is honoured by the
 * host-pointer entry points (see below); the Device entry points cannot call back into the host and record
 * RTC_ERROR_INVALID_OPERATION when a filter applies.  `intersect`/`occluded` (user geometries) must be NULL. */
struct RTCRayQueryContext {
  unsigned int instID[RTC_MAX_INSTANCE_LEVEL_COUNT];
  unsigned int instPrimID[RTC_MAX_INSTANCE_LEVEL_COUNT];
};
/* Filter callbacks (rtcore_common.h:311-324): called on the HOST for every candidate hit of a geometry that has a filter
 * (or, with RTC_RAY_QUERY_FLAG_INVOKE_ARGUMENT_FILTER / rtcSetGeometryEnableFilterFunctionFromArguments, for the
 * arguments' filter), always with N == 1: `ray` is an RTCRay whose tfar is the candidate distance, `hit` an RTCHit.
 * Setting valid[0] = 0 rejects the hit and the traversal goes on without it.  Host-pointer entry points only. */
struct RTCRayN;
struct RTCHitN;
struct RTCFilterFunctionNArguments {
  int* valid; void* geometryUserPtr; struct RTCRayQueryContext* context; struct RTCRayN* ray; struct RTCHitN* hit; unsigned int N;
};
typedef void (*RTCFilterFunctionN)(const struct RTCFilterFunctionNArguments* args);
typedef void (*RTCIntersectFunctionN)(const void* args);
typedef void (*RTCOccludedFunctionN)(const void* args);
struct RTCIntersectArguments {
  enum RTCRayQueryFlags flags; enum RTCFeatureFlags feature_mask; struct RTCRayQueryContext* context;
  RTCFilterFunctionN filter; RTCIntersectFunctionN intersect;
};
struct RTCOccludedArguments {
  enum RTCRayQueryFlags flags; enum RTCFeatureFlags feature_mask; struct RTCRayQueryContext* context;
  RTCFilterFunctionN filter; RTCOccludedFunctionN occluded;
};
static inline void rtcInitRayQueryContext(struct RTCRayQueryContext* c) {
  c->instID[0] = RTC_INVALID_GEOMETRY_ID; c->instPrimID[0] = RTC_INVALID_GEOMETRY_ID;
}
static inline void rtcInitIntersectArguments(struct RTCIntersectArguments* a) {
  a->flags = RTC_RAY_QUERY_FLAG_INCOHERENT; a->feature_mask = RTC_FEATURE_FLAG_ALL; a->context = NULL;
  a->filter = NULL; a->intersect = NULL;
}
static inline void rtcInitOccludedArguments(struct RTCOccludedArguments* a) {
  a->flags = RTC_RAY_QUERY_FLAG_INCOHERENT; a->feature_mask = RTC_FEATURE_FLAG_ALL; a->context = NULL;
  a->filter = NULL; a->occluded = NULL;
}

typedef void (*RTCErrorFunction)(void* userPtr, enum RTCError code, const char* str);
typedef bool (*RTCMemoryMonitorFunction)(void* ptr, ssize_t bytes, bool post);
typedef bool (*RTCProgressMonitorFunction)(void* ptr, double n);

/* =====================================================================================================
 * Section A -- Embree 4 entry points (same names, argument meaning and error behaviour).
 * Error convention (kernels/common/rtcore.h:23-49, device.cpp:263-330): no return codes; the FIRST failure is
 * latched per device (per thread when the device is NULL) until read by rtcGetDeviceError; the optional
 * error callback sees every failure.  Query functions do no argument checks (rtcore.cpp:604-608).
 * ===================================================================================================== */

/* device -- rtcore_device.h:15-125 / rtcore.cpp:19-140.  config keys: "verbose=N", "gpu=N" (CUDA ordinal, default:
 * current device); all other reference keys ("threads", "isa", "tri_accel", ...) are accepted and ignored. */
RTCB200_API RTCDevice rtcNewDevice(const char* config);
RTCB200_API void rtcRetainDevice(RTCDevice device);
RTCB200_API void rtcReleaseDevice(RTCDevice device);
RTCB200_API ssize_t rtcGetDeviceProperty(RTCDevice device, enum RTCDeviceProperty prop);
RTCB200_API void rtcSetDeviceProperty(RTCDevice device, enum RTCDeviceProperty prop, ssize_t value);
RTCB200_API const char* rtcGetErrorString(enum RTCError error);
RTCB200_API enum RTCError rtcGetDeviceError(RTCDevice device);
RTCB200_API const char* rtcGetDeviceLastErrorMessage(RTCDevice device);
RTCB200_API void rtcSetDeviceErrorFunction(RTCDevice device, RTCErrorFunction error, void* userPtr);
RTCB200_API void rtcSetDeviceMemoryMonitorFunction(RTCDevice device, RTCMemoryMonitorFunction fn, void* userPtr);

/* buffers -- rtcore_buffer.h:39-71 / kernels/common/buffer.h:16-97.  Host memory; uploaded at rtcCommitScene. */
RTCB200_API RTCBuffer rtcNewBuffer(RTCDevice device, size_t byteSize);
RTCB200_API RTCBuffer rtcNewSharedBuffer(RTCDevice device, void* ptr, size_t byteSize);
RTCB200_API RTCBuffer rtcNewBufferHostDevice(RTCDevice device, size_t byteSize);
RTCB200_API RTCBuffer rtcNewSharedBufferHostDevice(RTCDevice device, void* ptr, size_t byteSize);
RTCB200_API void* rtcGetBufferData(RTCBuffer buffer);
RTCB200_API void* rtcGetBufferDataDevice(RTCBuffer buffer);
RTCB200_API void rtcCommitBuffer(RTCBuffer buffer);
RTCB200_API void rtcRetainBuffer(RTCBuffer buffer);
RTCB200_API void rtcReleaseBuffer(RTCBuffer buffer);

/* geometry -- rtcore_geometry.h:130-207 / kernels/common/geometry.cpp:97-135, scene_triangle_mesh.cpp:35-147.
 * VERTEX slot 0 must be RTC_FORMAT_FLOAT3 (stride >= 12, 4-byte aligned), INDEX must be RTC_FORMAT_UINT3. */
RTCB200_API RTCGeometry rtcNewGeometry(RTCDevice device, enum RTCGeometryType type);
RTCB200_API void rtcRetainGeometry(RTCGeometry geometry);
RTCB200_API void rtcReleaseGeometry(RTCGeometry geometry);
RTCB200_API void rtcCommitGeometry(RTCGeometry geometry);
RTCB200_API void rtcEnableGeometry(RTCGeometry geometry);
RTCB200_API void rtcDisableGeometry(RTCGeometry geometry);
RTCB200_API void rtcSetGeometryTimeStepCount(RTCGeometry geometry, unsigned int timeStepCount); /* only 1 */
RTCB200_API void rtcSetGeometryTessellationRate(RTCGeometry geometry, float tessellationRate); /* flat cubic curves: segments per curve, clamped to 1..16 (scene_curves.cpp:247) */
RTCB200_API void rtcSetGeometryVertexAttributeCount(RTCGeometry geometry, unsigned int n);
RTCB200_API void rtcSetGeometryMask(RTCGeometry geometry, unsigned int mask);
RTCB200_API void rtcSetGeometryBuildQuality(RTCGeometry geometry, enum RTCBuildQuality quality);
RTCB200_API void rtcSetGeometryBuffer(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot,
                                      enum RTCFormat format, RTCBuffer buffer, size_t byteOffset, size_t byteStride,
                                      size_t itemCount);
RTCB200_API void rtcSetSharedGeometryBuffer(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot,
                                            enum RTCFormat format, const void* ptr, size_t byteOffset,
                                            size_t byteStride, size_t itemCount);
RTCB200_API void* rtcSetNewGeometryBuffer(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot,
                                          enum RTCFormat format, size_t byteStride, size_t itemCount);
RTCB200_API void* rtcGetGeometryBufferData(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot);
RTCB200_API void rtcUpdateGeometryBuffer(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot);
RTCB200_API void rtcSetGeometryUserData(RTCGeometry geometry, void* ptr);
RTCB200_API void* rtcGetGeometryUserData(RTCGeometry geometry);
RTCB200_API void rtcSetGeometryEnableFilterFunctionFromArguments(RTCGeometry geometry, bool enable);
/* instancing (rtcore_geometry.h:231-250 / kernels/geometry/instance_intersector.cpp:15-38): an INSTANCE geometry shows a
 * committed triangle scene through an affine transform; hits report instID[0] = the instance's geomID, the instanced
 * scene's geomID/primID and Ng in object space.  One instancing level (RTC_MAX_INSTANCE_LEVEL_COUNT == 1). */
RTCB200_API void rtcSetGeometryInstancedScene(RTCGeometry geometry, RTCScene scene);
RTCB200_API void rtcSetGeometryTransform(RTCGeometry geometry, unsigned int timeStep, enum RTCFormat format, const void* xfm);
RTCB200_API void rtcGetGeometryTransform(RTCGeometry geometry, float time, enum RTCFormat format, void* xfm);
RTCB200_API void rtcGetGeometryTransformEx(RTCGeometry geometry, unsigned int instPrimID, float time, enum RTCFormat format, void* xfm);
RTCB200_API void rtcGetGeometryTransformFromScene(RTCScene scene, unsigned int geomID, float time, enum RTCFormat format, void* xfm);
RTCB200_API void rtcGetGeometryTransformFromTraversable(RTCTraversable traversable, unsigned int geomID, float time, enum RTCFormat format, void* xfm);
/* host callbacks: a non-NULL function raises RTC_ERROR_INVALID_OPERATION (cannot run on the device) */
RTCB200_API void rtcSetGeometryIntersectFilterFunction(RTCGeometry geometry, RTCFilterFunctionN filter);
RTCB200_API void rtcSetGeometryOccludedFilterFunction(RTCGeometry geometry, RTCFilterFunctionN filter);

/* scene -- rtcore_scene.h:89-140 / kernels/common/scene.cpp:152-235,762-1040, rtcore.cpp:293-416 */
RTCB200_API RTCScene rtcNewScene(RTCDevice device);
RTCB200_API RTCDevice rtcGetSceneDevice(RTCScene scene); /* returns an extra reference (rtcore.cpp:305) */
RTCB200_API void rtcRetainScene(RTCScene scene);
RTCB200_API void rtcReleaseScene(RTCScene scene);
RTCB200_API RTCTraversable rtcGetSceneTraversable(RTCScene scene);
RTCB200_API unsigned int rtcAttachGeometry(RTCScene scene, RTCGeometry geometry);
RTCB200_API void rtcAttachGeometryByID(RTCScene scene, RTCGeometry geometry, unsigned int geomID);
RTCB200_API void rtcDetachGeometry(RTCScene scene, unsigned int geomID);
RTCB200_API RTCGeometry rtcGetGeometry(RTCScene scene, unsigned int geomID);
RTCB200_API RTCGeometry rtcGetGeometryThreadSafe(RTCScene scene, unsigned int geomID);
RTCB200_API void* rtcGetGeometryUserDataFromScene(RTCScene scene, unsigned int geomID);
RTCB200_API void rtcCommitScene(RTCScene scene);     /* upload + device BVH build; blocking like the reference */
RTCB200_API void rtcJoinCommitScene(RTCScene scene); /* == rtcCommitScene, serialised per scene */
RTCB200_API void rtcSetSceneProgressMonitorFunction(RTCScene scene, RTCProgressMonitorFunction fn, void* ptr);
RTCB200_API void rtcSetSceneBuildQuality(RTCScene scene, enum RTCBuildQuality quality);
RTCB200_API void rtcSetSceneFlags(RTCScene scene, enum RTCSceneFlags flags);
RTCB200_API enum RTCSceneFlags rtcGetSceneFlags(RTCScene scene);
RTCB200_API void rtcGetSceneBounds(RTCScene scene, struct RTCBounds* bounds_o);
RTCB200_API void rtcGetSceneLinearBounds(RTCScene scene, struct RTCLinearBounds* bounds_o);

/* ray queries -- rtcore_scene.h:152-215 / rtcore.cpp:599-630 (1), 670-713 (4), 797-841 (8), 858-901 (16),
 * 918-946 (occluded1), 987-1200 (occluded4/8/16).  Synchronous: the record is updated on return.
 * `valid[i] == -1` marks an active lane, 0 an inactive one; inactive lanes come back bit-identical.
 * Closest hit writes ray.tfar, hit.Ng/u/v/primID/geomID/instID[0]/instPrimID[0]; a miss writes nothing.
 * Occluded writes ray.tfar = -inf on any hit, nothing otherwise. */
RTCB200_API void rtcIntersect1(RTCScene scene, struct RTCRayHit* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcIntersect4(const int* valid, RTCScene scene, struct RTCRayHit4* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcIntersect8(const int* valid, RTCScene scene, struct RTCRayHit8* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcIntersect16(const int* valid, RTCScene scene, struct RTCRayHit16* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcOccluded1(RTCScene scene, struct RTCRay* ray, struct RTCOccludedArguments* args);
RTCB200_API void rtcOccluded4(const int* valid, RTCScene scene, struct RTCRay4* ray, struct RTCOccludedArguments* args);
RTCB200_API void rtcOccluded8(const int* valid, RTCScene scene, struct RTCRay8* ray, struct RTCOccludedArguments* args);
RTCB200_API void rtcOccluded16(const int* valid, RTCScene scene, struct RTCRay16* ray, struct RTCOccludedArguments* args);
RTCB200_API void rtcTraversableIntersect1(RTCTraversable t, struct RTCRayHit* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcTraversableIntersect4(const int* valid, RTCTraversable t, struct RTCRayHit4* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcTraversableIntersect8(const int* valid, RTCTraversable t, struct RTCRayHit8* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcTraversableIntersect16(const int* valid, RTCTraversable t, struct RTCRayHit16* rayhit, struct RTCIntersectArguments* args);
RTCB200_API void rtcTraversableOccluded1(RTCTraversable t, struct RTCRay* ray, struct RTCOccludedArguments* args);
RTCB200_API void rtcTraversableOccluded4(const int* valid, RTCTraversable t, struct RTCRay4* ray, struct RTCOccludedArguments* args);
RTCB200_API void rtcTraversableOccluded8(const int* valid, RTCTraversable t, struct RTCRay8* ray, struct RTCOccludedArguments* args);
RTCB200_API void rtcTraversableOccluded16(const int* valid, RTCTraversable t, struct RTCRay16* ray, struct RTCOccludedArguments* args);

/* =====================================================================================================
 * Section B -- batched extension.  One call traces M records; semantics per record are exactly those of the
 * single-record entry points above.  "Host" variants take host pointers (pageable or pinned) and pipeline
 * H2D copy / trace / D2H copy in chunks; "Device" variants take device pointers on the scene's GPU and enqueue
 * on `cuda_stream` (a cudaStream_t passed as void*; NULL = the legacy default stream) without synchronising.
 * ===================================================================================================== */
RTCB200_API void rtcb200Intersect1M(RTCScene scene, struct RTCRayHit* rayhits, size_t M, struct RTCIntersectArguments* args);
RTCB200_API void rtcb200Occluded1M(RTCScene scene, struct RTCRay* rays, size_t M, struct RTCOccludedArguments* args);
/* M packets of K = 4, 8 or 16 lanes; valid = M*K ints (or NULL = all active) */
RTCB200_API void rtcb200IntersectNM(const int* valid, RTCScene scene, void* rayhitK, unsigned int K, size_t M, struct RTCIntersectArguments* args);
RTCB200_API void rtcb200OccludedNM(const int* valid, RTCScene scene, void* rayK, unsigned int K, size_t M, struct RTCOccludedArguments* args);
RTCB200_API void rtcb200Intersect1MDevice(RTCScene scene, struct RTCRayHit* d_rayhits, size_t M, struct RTCIntersectArguments* args, void* cuda_stream);
/* as rtcb200Intersect1MDevice, and additionally writes one compact 32-byte record {tfar, Ng.xyz, u, v, primID, geomID} per
 * ray (primID = geomID = -1 on a miss) to compact_out[i] (32-byte aligned).  compact_out may be memory of ANOTHER GPU imported with
 * rtcb200PeerImport (the multi-GPU hit gather): the trace kernel stores the records itself, straight over NVLink when
 * the buffer is a peer's -- by default staged per 32-ray block in a local buffer and sent as 1 KB (eight full lines) when
 * the block is complete; rtcb200SetTuning("gather_mode", 0) selects one 32-byte store per record as its ray terminates.
 * Either way, work enqueued on cuda_stream after this call sees the complete buffer. */
RTCB200_API void rtcb200Intersect1MGatherDevice(RTCScene scene, struct RTCRayHit* d_rayhits, size_t M, struct RTCIntersectArguments* args, void* cuda_stream, void* compact_out);
RTCB200_API void rtcb200Occluded1MDevice(RTCScene scene, struct RTCRay* d_rays, size_t M, struct RTCOccludedArguments* args, void* cuda_stream);
RTCB200_API void rtcb200IntersectNMDevice(const int* d_valid, RTCScene scene, void* d_rayhitK, unsigned int K, size_t M, struct RTCIntersectArguments* args, void* cuda_stream);
RTCB200_API void rtcb200OccludedNMDevice(const int* d_valid, RTCScene scene, void* d_rayK, unsigned int K, size_t M, struct RTCOccludedArguments* args, void* cuda_stream);

/* Peer-visible device buffers (one process per GPU): allocate on the owner, export a 64-byte handle, import it in the
 * other processes (CUDA IPC, peer access over NVLink enabled on import). */
RTCB200_API void* rtcb200PeerAlloc(RTCDevice device, size_t bytes);
RTCB200_API void rtcb200PeerFree(RTCDevice device, void* ptr);
RTCB200_API int rtcb200PeerExport(RTCDevice device, void* ptr, unsigned char handle[64]);
RTCB200_API void* rtcb200PeerImport(RTCDevice device, const unsigned char handle[64]);
RTCB200_API void rtcb200PeerClose(RTCDevice device, void* ptr);
RTCB200_API void rtcb200PeerCopy(RTCDevice device, void* dst, const void* src, size_t bytes); /* blocking cudaMemcpyDefault */

/* Build / traversal statistics of the last commit and, when enabled, of traced rays
 * (device analogue of EMBREE_STAT_COUNTERS, kernels/common/stat.h:82-90). */
struct RTCB200SceneStats {
  unsigned long long num_triangles;      /* valid triangles in the BVH (after the validity filter) */
  unsigned long long num_nodes;          /* 80-byte BVH8 nodes */
  unsigned long long node_bytes, tri_bytes;
  double build_ms;                       /* device time of the last rtcCommitScene build */
  double sah_cost;                       /* SAH cost of the committed BVH8 (area-weighted, c_trav=1, c_tri=1) */
  unsigned long long trav_rays, trav_nodes, trav_tris; /* accumulated while counting is enabled */
  unsigned int builder;                  /* last commit: 0 = LBVH build, 1 = binned-SAH build, 2 = refit of the kept BVH */
  unsigned int max_depth;
};
RTCB200_API void rtcb200GetSceneStats(RTCScene scene, struct RTCB200SceneStats* out);
RTCB200_API void rtcb200SetSceneStatCounters(RTCScene scene, int enable); /* routes queries to the counting kernel */
RTCB200_API void rtcb200ResetSceneStatCounters(RTCScene scene);
/* Read-only inspection of a committed scene's acceleration structure, for tests and debugging tools (no query needs it).
 * rtcb200GetSceneLayout reports the sizes; rtcb200CopySceneArrays copies the scene's arrays into caller buffers of those sizes
 * (any pointer may be NULL): nodes = num_nodes 96-byte BVH8 nodes, records = num_records 48-byte leaf records (layouts:
 * embree_b200/csrc/rt_core.cuh Node8 / TriRec), descs = num_descs descriptors (general scenes -- instances, quads, curves or
 * points -- whose records hold a descriptor index instead of a geomID), levels = num_levels node ids where each BVH8 level starts
 * (the last entry is num_nodes; empty when the commit kept none), subs = 4 x num_subs words per mesh of a two-level scene (first
 * node, first record, node count, record count of its relocated BVH; the first top_nodes nodes are reserved for the top level). */
struct RTCB200SceneLayout {
  unsigned int num_nodes, num_records, num_descs, num_levels, num_subs, top_nodes;
  unsigned int max_depth;                /* BVH8 levels of a single-BVH build (0 for a two-level scene) */
  unsigned int general, robust;
  unsigned int builder;                  /* as RTCB200SceneStats.builder; 3 = two-level assembly */
};
struct RTCB200DescInfo {
  unsigned int geomID, instID;           /* instID: RTC_INVALID_GEOMETRY_ID unless seen through an instance */
  unsigned int kind;                     /* 0 triangle / quad, 1 round linear, 2 flat linear, 3 flat cubic, 4 round cubic, 5 sphere, 6 disc, 7 oriented disc point */
  unsigned int first, count;             /* global index of the first BVH primitive, number of BVH primitives (valid or not) */
  unsigned int is_quad, tess, basis, hermite;   /* basis: 0 Bezier, 1 B-spline, 2 Catmull-Rom (Hermite input is converted to Bezier) */
  float xfm[12];                         /* local-to-world columns vx | vy | vz | p of the instance (identity when not instanced) */
};
RTCB200_API void rtcb200GetSceneLayout(RTCScene scene, struct RTCB200SceneLayout* out);
RTCB200_API void rtcb200CopySceneArrays(RTCScene scene, void* nodes, void* records, struct RTCB200DescInfo* descs, unsigned int* levels,
                                        unsigned int* subs);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
RTCB200_API unsigned long long rtcb200GetLaunchCount(void);
/* experiment knobs (process-wide): kernels "collapse_policy", "c_node", "c_tri", "sah_small", "tri_batch_min",
 * "tri_wait_max" ("curve_batch_min", "curve_wait_max": the same two for scenes with curves, "point_batch_min",
 * "point_wait_max" for scenes of points only), "refill_min", "blocks_per_sm" ("curve_blocks_per_sm" for scenes with curves),
 * "use_tma"; host-pointer pipeline "host_chunk_log2", "host_streams"; hit gather "gather_mode" (0 one store per record,
 * 1 complete 32-ray blocks as 1 KB stores); "tri_spread" (warp-wide triangle redistribution, on by default).
 * The defaults are the shipped, measured configuration.
 * Returns 0, or -1 for an unknown key or an out-of-range value. */
RTCB200_API int rtcb200SetTuning(const char* key, int value);
/* device time (ms) of the most recent batched Device trace launch, measured with events on its stream; -1 if none */
RTCB200_API double rtcb200GetLastTraceMs(RTCScene scene);

/* =====================================================================================================
 * Section C -- the rest of the reference library's export list (kernels/export.linux.map: every rtc* symbol).
 * Thin variants of supported calls are implemented; the others (geometry types other than triangles, host
 * callbacks, point queries, rtcBuildBVH, instancing, interpolation) exist so that any Embree 4 caller LINKS
 * unchanged: calling one records RTC_ERROR_INVALID_OPERATION in the thread error slot and returns 0/NULL/false.
 * They are declared without prototypes on purpose -- compile callers against the reference's own headers.
 * ===================================================================================================== */
RTCB200_API void* rtcGetGeometryBufferDataDevice(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot);
RTCB200_API void rtcSetSharedGeometryBufferHostDevice(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot, enum RTCFormat format,
                                                      const void* ptr, const void* dptr, size_t byteOffset, size_t byteStride, size_t itemCount);
RTCB200_API void rtcSetNewGeometryBufferHostDevice(RTCGeometry geometry, enum RTCBufferType type, unsigned int slot, enum RTCFormat format,
                                                   size_t byteStride, size_t itemCount, void** ptr, void** dptr);
RTCB200_API void* rtcGetGeometryUserDataFromTraversable(RTCTraversable traversable, unsigned int geomID);
RTCB200_API void rtcSetGeometryTimeRange(RTCGeometry geometry, float startTime, float endTime);
RTCB200_API void rtcSetGeometryMaxRadiusScale(RTCGeometry geometry, float maxRadiusScale);
/* Vertex-data interpolation (rtcore_geometry.h:284-387; scene_triangle_mesh.h:49-105, scene_quad_mesh.h, geometry.cpp:163-235): host-side
 * arithmetic on the geometry's vertex / vertex-attribute buffers at (primID, u, v) for triangle and quad meshes -- what the tutorials'
 * shading code calls after a hit (rtcInterpolate0/1/2 are inline wrappers in the reference header).  Other geometry types:
 * RTC_ERROR_INVALID_OPERATION. */
struct RTCInterpolateArguments {
  RTCGeometry geometry; unsigned int primID; float u, v; enum RTCBufferType bufferType; unsigned int bufferSlot;
  float *P, *dPdu, *dPdv, *ddPdudu, *ddPdvdv, *ddPdudv; unsigned int valueCount;
};
struct RTCInterpolateNArguments {
  RTCGeometry geometry; const void* valid; const unsigned int* primIDs; const float *u, *v; unsigned int N;
  enum RTCBufferType bufferType; unsigned int bufferSlot; float *P, *dPdu, *dPdv, *ddPdudu, *ddPdvdv, *ddPdudv; unsigned int valueCount;
};
RTCB200_API void rtcInterpolate(const struct RTCInterpolateArguments* args);
RTCB200_API void rtcInterpolateN(const struct RTCInterpolateNArguments* args);
#define RTCB200_DECLARE_UNSUPPORTED(name) RTCB200_API void* name(void);
RTCB200_DECLARE_UNSUPPORTED(rtcBuildBVH)
RTCB200_DECLARE_UNSUPPORTED(rtcCollide)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect1)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect16)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect16Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect1Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect4)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect4Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect8)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardIntersect8Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded1)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded16)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded16Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded1Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded4)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded4Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded8)
RTCB200_DECLARE_UNSUPPORTED(rtcForwardOccluded8Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcGetGeometryFace)
RTCB200_DECLARE_UNSUPPORTED(rtcGetGeometryFirstHalfEdge)
RTCB200_DECLARE_UNSUPPORTED(rtcGetGeometryNextHalfEdge)
RTCB200_DECLARE_UNSUPPORTED(rtcGetGeometryOppositeHalfEdge)
RTCB200_DECLARE_UNSUPPORTED(rtcGetGeometryPreviousHalfEdge)
RTCB200_DECLARE_UNSUPPORTED(rtcInvokeIntersectFilterFromGeometry)
RTCB200_DECLARE_UNSUPPORTED(rtcInvokeOccludedFilterFromGeometry)
RTCB200_DECLARE_UNSUPPORTED(rtcMakeStaticBVH)
RTCB200_DECLARE_UNSUPPORTED(rtcNewBVH)
RTCB200_DECLARE_UNSUPPORTED(rtcPointQuery)
RTCB200_DECLARE_UNSUPPORTED(rtcPointQuery16)
RTCB200_DECLARE_UNSUPPORTED(rtcPointQuery4)
RTCB200_DECLARE_UNSUPPORTED(rtcPointQuery8)
RTCB200_DECLARE_UNSUPPORTED(rtcReleaseBVH)
RTCB200_DECLARE_UNSUPPORTED(rtcRetainBVH)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryBoundsFunction)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryDisplacementFunction)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryInstancedScenes)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryIntersectFunction)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryOccludedFunction)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryPointQueryFunction)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometrySubdivisionMode)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryTopologyCount)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryTransformQuaternion)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryUserPrimitiveCount)
RTCB200_DECLARE_UNSUPPORTED(rtcSetGeometryVertexAttributeTopology)
RTCB200_DECLARE_UNSUPPORTED(rtcThreadLocalAlloc)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect1)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect16)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect16Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect1Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect4)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect4Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect8)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardIntersect8Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded1)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded16)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded16Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded1Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded4)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded4Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded8)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversableForwardOccluded8Ex)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversablePointQuery)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversablePointQuery16)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversablePointQuery4)
RTCB200_DECLARE_UNSUPPORTED(rtcTraversablePointQuery8)

#ifdef __cplusplus
}
#endif
#endif /* EMBREE4_B200_H */
