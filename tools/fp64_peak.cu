// FP64 peak micro-benchmarks on the bench GPU: vector DFMA and tensor DMMA (mma.sync.m8n8k4.f64).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peak fp64_peak.cu ; prints JSON.
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_dfma(double* out, int iters) {
  double a[16];
  const double x = 1.0000001 + threadIdx.x * 1e-9, y = 0.9999999;
#pragma unroll
  for (int i = 0; i < 16; ++i) a[i] = i * 0.1;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = fma(a[i], x, y);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_dmma(double* out, int iters) {
  double c0[4] = {0, 0, 0, 0}, c1[4] = {0, 0, 0, 0};
  const double a = 1.0 + threadIdx.x * 1e-6, b = 0.5;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0[2 * u]), "+d"(c0[2 * u + 1]) : "d"(a), "d"(b));
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c1[2 * u]), "+d"(c1[2 * u + 1]) : "d"(a), "d"(b));
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = c0[0] + c0[1] + c0[2] + c0[3] + c1[0] + c1[1] + c1[2] + c1[3];
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  const int blocks = p.multiProcessorCount * 4, threads = 512;
  double* out;
  cudaMalloc(&out, sizeof(double) * blocks * threads);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms;
  const int iters = 20000;
  k_dfma<<<blocks, threads>>>(out, 100);
  cudaDeviceSynchronize();
  double best_fma = 0, best_mma = 0;
  for (int rep = 0; rep < 5; ++rep) {
    cudaEventRecord(e0);
    k_dfma<<<blocks, threads>>>(out, iters);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    const double tf = 2.0 * 16 * (double)iters * blocks * threads / (ms * 1e-3) / 1e12;
    if (tf > best_fma) best_fma = tf;
  }
  k_dmma<<<blocks, threads>>>(out, 100);
  cudaDeviceSynchronize();
  for (int rep = 0; rep < 5; ++rep) {
    cudaEventRecord(e0);
    k_dmma<<<blocks, threads>>>(out, iters);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    // per warp per mma: 8*8*4*2 flops; 4 mma per iteration
    const double tf = 4.0 * 512.0 * (double)iters * blocks * (threads / 32) / (ms * 1e-3) / 1e12;
    if (tf > best_mma) best_mma = tf;
  }
  printf("{\"gpu\": \"%s\", \"sms\": %d, \"fp64_fma_tflops\": %.3f, \"fp64_dmma_tflops\": %.3f}\n", p.name, p.multiProcessorCount, best_fma, best_mma);
  return 0;
}
