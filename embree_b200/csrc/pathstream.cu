// pathstream.cu -- wavefront form of the reference's path-tracer tile loop, the CALLER of the hot path for BASELINE
// configs[4] (tutorials/pathtracer/pathtracer_device.cpp:1489-1603): one stream of RTCRayHit records per GPU, and per
// bounce   rtcb200Intersect1MDevice -> pts200_bounce -> rtcb200Occluded1MDevice -> pts200_shade.
// The kernels here are hand-written sm_90a CUDA in their own small C-ABI library (libpathstream_b200.so): they are
// tutorial-side code, not part of the Embree API, and link nothing from libembree4_b200.so.
//
// What one reference loop iteration does after rtcIntersect1, restated per path (thread = path, records in place):
//   miss            -> the path ends (:1513-1527); the record becomes an inactive ray (tnear = +inf, tfar = -inf)
//   dg.P            = org + tfar * dir                                                  (:1539)
//   dg.eps          = 32 * 1.19209e-07 * max(|P.x|, |P.y|, |P.z|, tfar)                 (:1119-1120, postIntersect)
//   dg.Ng = dg.Ns   = face_forward(dir, normalize(Ng))                                  (:1543-1544)
//   wi1             = cosineSampleHemisphere(get2D, Ns)   -- matte material, c = albedo  (sampling.h:52-78, frame():
//                     linearspace3.h:117-124)
//   shadow ray      = (P, ls.dir, eps, ls.dist) towards a point light; get2D is consumed (:1565-1571)
//   next ray        = (P + sign(dot(wi1, Ng)) * eps * Ng, normalize(wi1), eps, inf)      (:1597-1600)
// and after rtcOccluded1:  L += Lw * ls.weight * brdf  when shadow.tfar >= 0            (:1586-1592)
// The sampler is the tutorials' RandomSampler (random_sampler.h:15-80): MurmurHash3 seed, LCG stream, one state per path.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#define PTS_API extern "C" __attribute__((visibility("default")))

namespace {

struct Sampler { uint32_t s; };
__device__ __forceinline__ uint32_t murmur_mix(uint32_t hash, uint32_t k) {
  k *= 0xcc9e2d51u; k = (k << 15) | (k >> 17); k *= 0x1b873593u;
  hash ^= k;
  return ((hash << 13) | (hash >> 19)) * 5u + 0xe6546b64u;
}
__device__ __forceinline__ uint32_t murmur_finalize(uint32_t h) {
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}
__device__ __forceinline__ void sampler_init(Sampler& s, int x, int y, int sampleId) {   // random_sampler.h:57-72
  uint32_t h = murmur_mix(0u, (uint32_t)(x | (y << 16)));
  h = murmur_mix(h, (uint32_t)sampleId);
  s.s = murmur_finalize(h);
}
__device__ __forceinline__ float sampler_get1d(Sampler& s) {                            // :74-90
  s.s = s.s * 1664525u + 1013904223u;
  return (float)(int)(s.s >> 1) * 4.656612873077392578125e-10f;
}

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3 operator*(float s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ V3 normalize(V3 a) { return rsqrtf(dot(a, a)) * a; }

struct Camera { float px, py, pz, ux, uy, uz, vx, vy, vz, wx, wy, wz; int width, height, spp; };
struct Light { float px, py, pz, intensity, albedo; };

// ---- primary rays: pixel = path / spp, sample = path % spp; jittered pinhole ray exactly as renderPixelFunction sets it
// up (pathtracer_device.cpp:1470-1484: RandomSampler_init(x, y, sample), fx = x + get1D, fy = y + get1D, time = get1D)
__global__ void __launch_bounds__(256) primary_kernel(float4* __restrict__ rays, uint32_t* __restrict__ rng, float* __restrict__ Lw,
                                                      unsigned long long first_path, uint32_t n, Camera cam) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long path = first_path + i;
  const uint32_t pixel = (uint32_t)(path / (unsigned)cam.spp), sample = (uint32_t)(path % (unsigned)cam.spp);
  const int x = (int)(pixel % (uint32_t)cam.width), y = (int)(pixel / (uint32_t)cam.width);
  Sampler s;
  sampler_init(s, x, y, (int)sample);
  const float fx = (float)x + sampler_get1d(s), fy = (float)y + sampler_get1d(s);
  (void)sampler_get1d(s);   // time
  const V3 d = normalize(V3{fx * cam.ux + fy * cam.vx + cam.wx, fx * cam.uy + fy * cam.vy + cam.wy, fx * cam.uz + fy * cam.vz + cam.wz});
  float4* r = rays + (size_t)i * 6;
  r[0] = make_float4(cam.px, cam.py, cam.pz, 0.0f);
  r[1] = make_float4(d.x, d.y, d.z, 0.0f);
  r[2] = make_float4(INFINITY, __uint_as_float(0xFFFFFFFFu), __uint_as_float(i), __uint_as_float(0u));   // tfar, mask, id = path slot, flags
  r[3] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  r[4] = make_float4(0.0f, __uint_as_float(0xFFFFFFFFu), __uint_as_float(0xFFFFFFFFu), __uint_as_float(0xFFFFFFFFu));   // v, primID, geomID, instID
  r[5] = make_float4(__uint_as_float(0xFFFFFFFFu), 0.0f, 0.0f, 0.0f);
  rng[i] = s.s;
  Lw[i] = 1.0f;
}

// ---- one bounce: consume the hit of record i, emit its shadow ray and overwrite the record with the next ray
__global__ void __launch_bounds__(256) bounce_kernel(float4* __restrict__ rays, float4* __restrict__ shadow, uint32_t* __restrict__ rng,
                                                     float* __restrict__ Lw, float* __restrict__ pending, uint32_t n, Light light) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4* r = rays + (size_t)i * 6;
  float4* sh = shadow + (size_t)i * 3;
  const float4 r0 = r[0], r1 = r[1], r2 = r[2], h0 = r[3], h1 = r[4];
  const bool alive = r2.x >= 0.0f && __float_as_uint(h1.z) != 0xFFFFFFFFu;   // inactive records carry tfar = -inf; a miss ends the path
  if (!alive) {
    r[0] = make_float4(r0.x, r0.y, r0.z, INFINITY);
    r[2] = make_float4(-INFINITY, r2.y, r2.z, r2.w);
    sh[0] = make_float4(0.0f, 0.0f, 0.0f, INFINITY);
    sh[1] = make_float4(0.0f, 0.0f, 1.0f, 0.0f);
    sh[2] = make_float4(-INFINITY, __uint_as_float(0xFFFFFFFFu), r2.z, 0.0f);   // already "occluded": rtcOccluded1 returns at once
    pending[i] = 0.0f;
    return;
  }
  const V3 org{r0.x, r0.y, r0.z}, dir{r1.x, r1.y, r1.z};
  const float t = r2.x;
  const V3 P = org + t * dir;
  const float eps = 32.0f * 1.19209e-07f * fmaxf(fmaxf(fabsf(P.x), fabsf(P.y)), fmaxf(fabsf(P.z), t));
  V3 Ng = normalize(V3{h0.x, h0.y, h0.z});
  if (dot(dir, Ng) >= 0.0f) Ng = -1.0f * Ng;                     // face_forward(dir, Ng)
  Sampler s{rng[i]};
  // Material__sample (matte): cosine-weighted direction in frame(Ns)
  const float u1 = sampler_get1d(s), u2 = sampler_get1d(s);
  const float phi = 2.0f * 3.14159265358979323846f * u1, ct = sqrtf(u2), st = sqrtf(1.0f - u2);
  float sphi, cphi;
  sincosf(phi, &sphi, &cphi);
  const V3 dx0 = cross(V3{1, 0, 0}, Ng), dx1 = cross(V3{0, 1, 0}, Ng);
  const V3 dx = normalize(dot(dx0, dx0) > dot(dx1, dx1) ? dx0 : dx1);
  const V3 dy = normalize(cross(Ng, dx));
  const V3 wi = (cphi * st) * dx + (sphi * st) * dy + ct * Ng;
  // Lights_sample (point light); the 2D sample is drawn as the reference does although a point light ignores it
  (void)sampler_get1d(s); (void)sampler_get1d(s);
  const V3 toL = V3{light.px, light.py, light.pz} - P;
  const float dist2 = dot(toL, toL), dist = sqrtf(dist2);
  const V3 ld = (1.0f / dist) * toL;
  const float cosl = fmaxf(dot(ld, Ng), 0.0f);
  const float lw = Lw[i];
  pending[i] = lw * (light.intensity / dist2) * (light.albedo * 0.318309886f) * cosl;   // added by shade_kernel when unoccluded
  sh[0] = make_float4(P.x, P.y, P.z, eps);
  sh[1] = make_float4(ld.x, ld.y, ld.z, 0.0f);
  sh[2] = make_float4(dist, __uint_as_float(0xFFFFFFFFu), r2.z, __uint_as_float(0u));
  // secondary ray
  Lw[i] = lw * light.albedo;                                      // Lw * c / pdf with c = albedo * cos / pi, pdf = cos / pi
  const float sign = dot(wi, Ng) < 0.0f ? -1.0f : 1.0f;
  const V3 P2 = P + (sign * eps) * Ng;
  const V3 d2 = normalize(wi);
  r[0] = make_float4(P2.x, P2.y, P2.z, eps);
  r[1] = make_float4(d2.x, d2.y, d2.z, 0.0f);
  r[2] = make_float4(INFINITY, r2.y, r2.z, r2.w);
  r[4] = make_float4(h1.x, __uint_as_float(0xFFFFFFFFu), __uint_as_float(0xFFFFFFFFu), __uint_as_float(0xFFFFFFFFu));
  rng[i] = s.s;
}

// ---- after rtcOccluded1 on the shadow stream: unoccluded light samples contribute (shadow.tfar stays >= 0)
__global__ void __launch_bounds__(256) shade_kernel(const float4* __restrict__ shadow, const float* __restrict__ pending,
                                                    float* __restrict__ L, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float tfar = shadow[(size_t)i * 3 + 2].x;
  if (tfar >= 0.0f) L[i] += pending[i];
}

}  // namespace

// C-ABI ----------------------------------------------------------------------------------------------------------------
// camera: p, then the pinhole basis (u, v per pixel step, w = direction of pixel (0,0)); all pointers are device memory.
PTS_API int pts200_primary(void* d_rayhits, void* d_rng, void* d_Lw, unsigned long long first_path, unsigned n, const float* cam12,
                           int width, int height, int spp, void* stream) {
  Camera c{cam12[0], cam12[1], cam12[2], cam12[3], cam12[4], cam12[5], cam12[6], cam12[7], cam12[8], cam12[9], cam12[10], cam12[11], width, height, spp};
  if (n == 0) return 0;
  primary_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>((float4*)d_rayhits, (uint32_t*)d_rng, (float*)d_Lw, first_path, n, c);
  return (int)cudaGetLastError();
}
PTS_API int pts200_bounce(void* d_rayhits, void* d_shadow, void* d_rng, void* d_Lw, void* d_pending, unsigned n, const float* light5, void* stream) {
  Light l{light5[0], light5[1], light5[2], light5[3], light5[4]};
  if (n == 0) return 0;
  bounce_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>((float4*)d_rayhits, (float4*)d_shadow, (uint32_t*)d_rng, (float*)d_Lw,
                                                                  (float*)d_pending, n, l);
  return (int)cudaGetLastError();
}
PTS_API int pts200_shade(const void* d_shadow, const void* d_pending, void* d_L, unsigned n, void* stream) {
  if (n == 0) return 0;
  shade_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>((const float4*)d_shadow, (const float*)d_pending, (float*)d_L, n);
  return (int)cudaGetLastError();
}
