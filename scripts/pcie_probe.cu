// PCIe probe: linear vs strided (2D) copies of RTCRayHit streams, and zero-copy kernel gather/scatter.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a scripts/pcie_probe.cu -o scripts/_build/pcie_probe
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

__global__ void gather48(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n) {   // ray half of each record
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n * 3; i += stride) { size_t r = i / 3, k = i % 3; dst[r * 6 + k] = src[r * 6 + k]; }
}
__global__ void scatter64(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n) {  // bytes 32..96 of each record
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n * 4; i += stride) { size_t r = i / 4, k = 2 + i % 4; dst[r * 6 + k] = src[r * 6 + k]; }
}
int main() {
  const size_t n = size_t(1) << 24;   // 16 Mi records, 1.6 GB
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  char *h, *d;
  CK(cudaHostAlloc(&h, n * 96, cudaHostAllocMapped));
  CK(cudaMalloc(&d, n * 96));
  memset(h, 1, n * 96);
  char* hd; CK(cudaHostGetDevicePointer(&hd, h, 0));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaStream_t s1, s2; cudaStreamCreate(&s1); cudaStreamCreate(&s2);
  auto time = [&](const char* name, double bytes, auto fn) {
    fn(); cudaDeviceSynchronize();
    cudaEventRecord(e0); for (int i = 0; i < 3; ++i) fn(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 3;
    printf("%-44s %8.2f ms  %7.1f GB/s useful  (%.0f Mrec/s)\n", name, ms, bytes / ms * 1e-6, n / ms * 1e-3);
  };
  time("H2D linear 96B", n * 96.0, [&] { cudaMemcpyAsync(d, h, n * 96, cudaMemcpyHostToDevice, 0); });
  time("D2H linear 96B", n * 96.0, [&] { cudaMemcpyAsync(h, d, n * 96, cudaMemcpyDeviceToHost, 0); });
  time("H2D 2D 48 of 96", n * 48.0, [&] { cudaMemcpy2DAsync(d, 96, h, 96, 48, n, cudaMemcpyHostToDevice, 0); });
  time("D2H 2D 64 of 96", n * 64.0, [&] { cudaMemcpy2DAsync(h + 32, 96, d + 32, 96, 64, n, cudaMemcpyDeviceToHost, 0); });
  time("H2D kernel gather 48 of 96 (zero-copy)", n * 48.0, [&] { gather48<<<sms * 8, 256>>>((const uint4*)hd, (uint4*)d, n); });
  time("D2H kernel scatter 64 of 96 (zero-copy)", n * 64.0, [&] { scatter64<<<sms * 8, 256>>>((const uint4*)d, (uint4*)hd, n); });
  time("duplex linear 96B both ways", n * 192.0, [&] {
    cudaMemcpyAsync(d, h, n * 48, cudaMemcpyHostToDevice, s1); cudaMemcpyAsync(h + n * 48, d + n * 48, n * 48, cudaMemcpyDeviceToHost, s2);
    cudaMemcpyAsync(d, h, n * 48, cudaMemcpyHostToDevice, s1); cudaMemcpyAsync(h + n * 48, d + n * 48, n * 48, cudaMemcpyDeviceToHost, s2);
    cudaStreamSynchronize(s1); cudaStreamSynchronize(s2); });
  time("duplex kernel gather48 || scatter64", n * 112.0, [&] {
    gather48<<<sms * 4, 256, 0, s1>>>((const uint4*)hd, (uint4*)d, n / 2);
    scatter64<<<sms * 4, 256, 0, s2>>>((const uint4*)(d + n * 48), (uint4*)(hd + n * 48), n / 2);
    gather48<<<sms * 4, 256, 0, s1>>>((const uint4*)hd, (uint4*)d, n / 2);
    scatter64<<<sms * 4, 256, 0, s2>>>((const uint4*)(d + n * 48), (uint4*)(hd + n * 48), n / 2);
    cudaStreamSynchronize(s1); cudaStreamSynchronize(s2); });
  return 0;
}
