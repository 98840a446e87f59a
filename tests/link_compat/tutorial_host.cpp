// Host driver for the reference's OWN tutorial device code (tutorials/triangle_geometry/triangle_geometry_device.cpp =
// BASELINE configs[0]), which tests/link_compat/build.sh compiles untouched from $EMBREE_REFERENCE: this file only supplies
// what tutorials/common/tutorial/tutorial.cpp would (g_device, g_stats, the camera of triangle_geometry.cpp:23-24) and
// writes the rendered frame to a file, so the same tutorial code can be linked once against the reference library
// (golden image, generated in the container) and once against libembree4_b200.so (test on the GPU).
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <tutorials/common/tutorial/tutorial_device.h>
#include <tutorials/common/tutorial/camera.h>
#include <common/tasking/taskscheduler.h>

#ifndef CAMERA_FROM
#define CAMERA_FROM 1.5f, 1.5f, -1.5f
#endif

namespace embree {
RTCDevice g_device = nullptr;
extern "C" RayStats* g_stats = nullptr;
extern "C" void device_init(char* cfg);
extern "C" void renderFrameStandard(int* pixels, const unsigned int width, const unsigned int height, const float time, const ISPCCamera& camera);
extern "C" void device_cleanup();
}  // namespace embree

int main(int argc, char** argv) {
  using namespace embree;
  if (argc < 2) { fprintf(stderr, "usage: %s out.raw [width height threads]\n", argv[0]); return 2; }
  const unsigned width = argc > 2 ? atoi(argv[2]) : 160, height = argc > 3 ? atoi(argv[3]) : 120;
  const size_t threads = argc > 4 ? atoi(argv[4]) : 4;
  TaskScheduler::create(threads, false, true);
  g_device = rtcNewDevice(nullptr);
  if (!g_device) { fprintf(stderr, "rtcNewDevice failed: %d\n", (int)rtcGetDeviceError(nullptr)); return 1; }
  g_stats = (RayStats*)alignedMalloc(TaskScheduler::threadCount() * sizeof(RayStats), 64);
  for (size_t i = 0; i < TaskScheduler::threadCount(); ++i) g_stats[i].numRays = 0;
  Camera camera;
  camera.from = Vec3fa(CAMERA_FROM);         // triangle_geometry.cpp:23-24 (point_geometry.cpp:23-24 through -DCAMERA_FROM)
  camera.to = Vec3fa(0.0f, 0.0f, 0.0f);
  std::vector<int> pixels((size_t)width * height, 0);
  device_init(nullptr);
  renderFrameStandard(pixels.data(), width, height, 0.0f, camera.getISPCCamera(width, height));
  const RTCError err = rtcGetDeviceError(g_device);
  device_cleanup();
  FILE* f = fopen(argv[1], "wb");
  fwrite(pixels.data(), sizeof(int), pixels.size(), f);
  fclose(f);
  size_t rays = 0;
  for (size_t i = 0; i < TaskScheduler::threadCount(); ++i) rays += g_stats[i].numRays;
  printf("rendered %ux%u, %zu rays, device error %d\n", width, height, rays, (int)err);
  alignedFree(g_stats);
  rtcReleaseDevice(g_device);
  return err == RTC_ERROR_NONE ? 0 : 1;
}
