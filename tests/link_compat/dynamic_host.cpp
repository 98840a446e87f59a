// Host driver for the reference's OWN tutorial device code tutorials/dynamic_scene/dynamic_scene_device.cpp (BASELINE configs[3]b), which
// tests/link_compat/build.sh compiles untouched from $EMBREE_REFERENCE: an RTC_SCENE_FLAG_DYNAMIC | RTC_SCENE_FLAG_ROBUST scene (build quality
// LOW) of a ground plane and 20 spheres with per-geometry build qualities, whose vertices the tutorial rewrites every frame through
// rtcGetGeometryBufferData / rtcUpdateGeometryBuffer / rtcCommitGeometry before rtcCommitScene.  This file supplies what tutorial.cpp would
// (g_device, g_stats, the camera of dynamic_scene.cpp:23-24) and renders a few frames of the animation to files, so the same tutorial code
// can be linked against the reference library (golden frames) and against libembree4_b200.so (every sphere moves every frame, so the
// library rebuilds one BVH over everything per commit rather than taking its two-level path).
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include <tutorials/common/tutorial/tutorial_device.h>
#include <tutorials/common/tutorial/camera.h>
#include <common/tasking/taskscheduler.h>

namespace embree {
RTCDevice g_device = nullptr;
extern "C" RayStats* g_stats = nullptr;
extern "C" void device_init(char* cfg);
extern "C" void device_render(int* pixels, const unsigned int width, const unsigned int height, const float time, const ISPCCamera& camera);
extern "C" void renderFrameStandard(int* pixels, const unsigned int width, const unsigned int height, const float time, const ISPCCamera& camera);
extern "C" void device_cleanup();
}  // namespace embree

int main(int argc, char** argv) {
  using namespace embree;
  if (argc < 2) { fprintf(stderr, "usage: %s out_prefix [width height threads frames]\n", argv[0]); return 2; }
  const unsigned width = argc > 2 ? atoi(argv[2]) : 160, height = argc > 3 ? atoi(argv[3]) : 120;
  const size_t threads = argc > 4 ? atoi(argv[4]) : 4;
  const int frames = argc > 5 ? atoi(argv[5]) : 3;
  TaskScheduler::create(threads, false, true);
  g_device = rtcNewDevice(nullptr);
  if (!g_device) { fprintf(stderr, "rtcNewDevice failed: %d\n", (int)rtcGetDeviceError(nullptr)); return 1; }
  g_stats = (RayStats*)alignedMalloc(TaskScheduler::threadCount() * sizeof(RayStats), 64);
  for (size_t i = 0; i < TaskScheduler::threadCount(); ++i) g_stats[i].numRays = 0;
  Camera camera;
  camera.from = Vec3fa(2.0f, 2.0f, 2.0f);    // dynamic_scene.cpp:23-24
  camera.to = Vec3fa(0.0f, 0.0f, 0.0f);
  std::vector<int> pixels((size_t)width * height, 0);
  device_init(nullptr);
  RTCError err = rtcGetDeviceError(g_device);
  const ISPCCamera ic = camera.getISPCCamera(width, height);
  for (int f = 0; f < frames && err == RTC_ERROR_NONE; ++f) {
    const float time = 0.7f * f;
    device_render(pixels.data(), width, height, time, ic);          // animate every sphere + rtcCommitScene
    renderFrameStandard(pixels.data(), width, height, time, ic);
    err = rtcGetDeviceError(g_device);
    const std::string name = std::string(argv[1]) + "_" + std::to_string(f) + ".raw";
    FILE* fp = fopen(name.c_str(), "wb");
    fwrite(pixels.data(), sizeof(int), pixels.size(), fp);
    fclose(fp);
  }
  device_cleanup();
  size_t rays = 0;
  for (size_t i = 0; i < TaskScheduler::threadCount(); ++i) rays += g_stats[i].numRays;
  printf("rendered %d frames of %ux%u, %zu rays, device error %d\n", frames, width, height, rays, (int)err);
  alignedFree(g_stats);
  rtcReleaseDevice(g_device);
  return err == RTC_ERROR_NONE ? 0 : 1;
}
