// Host driver for the reference's OWN tutorial device code tutorials/hair_geometry/hair_geometry_device.cpp (BASELINE configs[3]a),
// which tests/link_compat/build.sh compiles untouched from $EMBREE_REFERENCE.  This file supplies what hair_geometry.cpp /
// tutorial.cpp / the scene loader would: g_device, g_stats, the lights and camera of models/furBall_A.ecs, and an ISPCScene
// filled by hand with a procedural fur ball (the shipped model cannot travel to the GPU box) -- one hair set whose curve type is
// chosen on the command line (round linear segments as in furBall_A.xml, flat or round cubic Bezier curves as the tutorials'
// hair generators make them) around one triangle sphere.  The tutorial code then does everything itself: rtcNewGeometry /
// rtcSetSharedGeometryBuffer / rtcSetGeometryTessellationRate / rtcSetGeometryEnableFilterFunctionFromArguments / rtcCommitScene,
// and per pixel a path of rtcTraversableIntersect1 + rtcTraversableOccluded1 with its transparency-accumulating occlusion filter.
// The frame is written to a file so the same code can be linked against the reference library (golden) and libembree4_b200.so.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <tutorials/common/tutorial/tutorial_device.h>
#include <tutorials/common/tutorial/scene_device.h>
#include <tutorials/common/tutorial/camera.h>
#include <common/tasking/taskscheduler.h>

namespace embree {
RTCDevice g_device = nullptr;
extern "C" RayStats* g_stats = nullptr;
extern "C" ISPCScene* g_ispc_scene = nullptr;
extern "C" bool g_changed = false;
extern "C" {
Vec3fa g_dirlight_direction = normalize(Vec3fa(1, -1, 1));   // furBall_A.ecs: -dirlight 1 -1 1 3 3 3, -ambientlight 1 1 1
Vec3fa g_dirlight_intensity = Vec3fa(3.0f);
Vec3fa g_ambient_intensity = Vec3fa(1.0f);
}
extern "C" void device_init(char* cfg);
extern "C" void device_render(int* pixels, const unsigned int width, const unsigned int height, const float time, const ISPCCamera& camera);
extern "C" void renderFrameStandard(int* pixels, const unsigned int width, const unsigned int height, const float time, const ISPCCamera& camera);
extern "C" void device_cleanup();
}  // namespace embree

using namespace embree;

static unsigned g_seed = 12345u;
static float frand() { g_seed = g_seed * 1664525u + 1013904223u; return (float)(g_seed >> 8) * (1.0f / 16777216.0f); }
static float grand() { float s = 0.0f; for (int i = 0; i < 6; ++i) s += frand(); return (s - 3.0f) * 1.4142135f; }   // ~N(0,1)

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: %s out.raw [width height threads curvetype strands device-config]\n  curvetype: 0 round linear, 1 flat Bezier, 2 round Bezier\n", argv[0]); return 2; }
  const unsigned width = argc > 2 ? atoi(argv[2]) : 96, height = argc > 3 ? atoi(argv[3]) : 72;
  const size_t threads = argc > 4 ? atoi(argv[4]) : 4;
  const int ctype = argc > 5 ? atoi(argv[5]) : 0;
  const unsigned strands = argc > 6 ? atoi(argv[6]) : 3000;
  TaskScheduler::create(threads, false, true);
  g_device = rtcNewDevice(argc > 7 ? argv[7] : nullptr);
  if (!g_device) { fprintf(stderr, "rtcNewDevice failed: %d\n", (int)rtcGetDeviceError(nullptr)); return 1; }
  g_stats = (RayStats*)alignedMalloc(TaskScheduler::threadCount() * sizeof(RayStats), 64);
  for (size_t i = 0; i < TaskScheduler::threadCount(); ++i) g_stats[i].numRays = 0;

  // ---- the scene the loader would have produced: geometries[0] = triangle sphere (radius 0.9), geometries[1] = hair set
  const int NP = 24;
  std::vector<Vec3fa> sv;
  std::vector<ISPCTriangle> st;
  for (int i = 0; i <= NP; ++i)
    for (int j = 0; j < 2 * NP; ++j) {
      const float th = float(M_PI) * i / NP, ph = float(M_PI) * j / NP;
      sv.push_back(Vec3fa(0.9f * sinf(th) * cosf(ph), 0.5f + 0.9f * cosf(th), 0.9f * sinf(th) * sinf(ph)));
    }
  for (int i = 0; i < NP; ++i)
    for (int j = 0; j < 2 * NP; ++j) {
      const unsigned a = i * 2 * NP + j, b = i * 2 * NP + (j + 1) % (2 * NP), c = a + 2 * NP, d = b + 2 * NP;
      ISPCTriangle t0, t1;
      memset(&t0, 0, sizeof t0); memset(&t1, 0, sizeof t1);
      t0.v0 = a; t0.v1 = c; t0.v2 = b; t1.v0 = b; t1.v1 = c; t1.v2 = d;
      st.push_back(t0); st.push_back(t1);
    }
  sv.push_back(Vec3fa(0.0f));   // 16-byte padding element
  ISPCTriangleMesh* mesh = (ISPCTriangleMesh*)alignedMalloc(sizeof(ISPCTriangleMesh), 16);
  memset((void*)mesh, 0, sizeof(ISPCTriangleMesh));
  mesh->geom.type = TRIANGLE_MESH;
  Vec3fa* mpos[1] = {sv.data()};
  mesh->positions = mpos; mesh->triangles = st.data();
  mesh->numTimeSteps = 1; mesh->numVertices = (unsigned)sv.size() - 1; mesh->numTriangles = (unsigned)st.size();
  mesh->startTime = 0.0f; mesh->endTime = 1.0f;

  const int K = ctype == 0 ? 7 : 10;                    // knots per strand
  std::vector<Vec3fa> hv;
  std::vector<ISPCHair> hh;
  for (unsigned s = 0; s < strands; ++s) {
    float n[3] = {grand(), grand(), grand()};
    float l = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]); if (l < 1e-6f) l = 1.0f;
    for (int a = 0; a < 3; ++a) n[a] /= l;
    float p[3] = {0.9f * n[0], 0.5f + 0.9f * n[1], 0.9f * n[2]}, d[3] = {n[0], n[1], n[2]};
    const unsigned first = (unsigned)hv.size();
    for (int k = 0; k < K; ++k) {
      Vec3ff v(p[0], p[1], p[2], 0.006f * (1.0f - 0.7f * k / K));   // xyz + radius
      hv.push_back(*(Vec3fa*)&v);
      for (int a = 0; a < 3; ++a) d[a] += 0.4f * grand();
      l = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      for (int a = 0; a < 3; ++a) { d[a] /= l; p[a] += d[a] * (ctype == 0 ? 0.07f : 0.05f); }
    }
    const int step = ctype == 0 ? 1 : 3, last = ctype == 0 ? K - 1 : K - 3;
    for (int k = 0; k < last; k += step) { ISPCHair h; h.vertex = first + k; h.id = s; hh.push_back(h); }
  }
  hv.push_back(Vec3fa(0.0f));
  ISPCHairSet* hair = (ISPCHairSet*)alignedMalloc(sizeof(ISPCHairSet), 16);
  memset((void*)hair, 0, sizeof(ISPCHairSet));
  hair->geom.type = CURVES;
  Vec3fa* hpos[1] = {hv.data()};
  hair->positions = hpos; hair->hairs = hh.data(); hair->flags = nullptr;
  hair->type = ctype == 0 ? RTC_GEOMETRY_TYPE_ROUND_LINEAR_CURVE : ctype == 1 ? RTC_GEOMETRY_TYPE_FLAT_BEZIER_CURVE : RTC_GEOMETRY_TYPE_ROUND_BEZIER_CURVE;
  hair->numTimeSteps = 1; hair->numVertices = (unsigned)hv.size() - 1; hair->numHairs = (unsigned)hh.size(); hair->numHairCurves = (unsigned)hh.size();
  hair->tessellation_rate = 4; hair->startTime = 0.0f; hair->endTime = 1.0f;

  ISPCScene* scene = (ISPCScene*)alignedMalloc(sizeof(ISPCScene), 16);
  memset((void*)scene, 0, sizeof(ISPCScene));
  ISPCGeometry* geoms[2] = {(ISPCGeometry*)mesh, (ISPCGeometry*)hair};
  scene->scene = rtcNewScene(g_device);
  scene->geometries = geoms; scene->numGeometries = 2;
  g_ispc_scene = scene;

  Camera camera;
  camera.from = Vec3fa(0.0f, 0.5f, 4.0f);    // furBall_A.ecs: -vp 0 .5 4 -vi 0 .5 0 -fov 50
  camera.to = Vec3fa(0.0f, 0.5f, 0.0f);
  camera.fov = 50.0f;
  std::vector<int> pixels((size_t)width * height, 0);
  device_init(nullptr);
  RTCError err = rtcGetDeviceError(g_device);
  const ISPCCamera ic = camera.getISPCCamera(width, height);
  device_render(pixels.data(), width, height, 0.0f, ic);            // allocates and clears the accumulation buffer
  renderFrameStandard(pixels.data(), width, height, 0.0f, ic);
  if (err == RTC_ERROR_NONE) err = rtcGetDeviceError(g_device);
  FILE* f = fopen(argv[1], "wb");
  fwrite(pixels.data(), sizeof(int), pixels.size(), f);
  fclose(f);
  size_t rays = 0;
  for (size_t i = 0; i < TaskScheduler::threadCount(); ++i) rays += g_stats[i].numRays;
  printf("rendered %ux%u, curve type %d, %zu hairs, %zu rays (primary + secondary + shadow), device error %d\n", width, height, ctype, hh.size(), rays, (int)err);
  return err == RTC_ERROR_NONE ? 0 : 1;
}
