// fp64 peak microbenchmark for the roofline denominators (SURVEY.md section 8d): DFMA (SIMT) and
// DMMA m8n8k4 (tensor) throughput on all SMs.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peak fp64_peak.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k_dfma(double* out, int iters) {
  double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  const double b = 1.0000001, c = 1e-9;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, b, c); a1 = fma(a1, b, c); a2 = fma(a2, b, c); a3 = fma(a3, b, c);
    a4 = fma(a4, b, c); a5 = fma(a5, b, c); a6 = fma(a6, b, c); a7 = fma(a7, b, c);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}
__global__ void k_dmma(double* out, int iters) {
  double c[8][2]; for (int i = 0; i < 8; ++i) { c[i][0] = 0; c[i][1] = 0; }
  double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
  }
  double s = 0; for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  double* out; cudaMalloc(&out, (size_t)sms * 8 * 1024 * sizeof(double));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int iters = 20000;
  for (int threads : {256, 512, 1024}) {
    const int blocks = sms * (2048 / threads);
    for (int rep = 0; rep < 2; ++rep) {
      cudaEventRecord(e0); k_dfma<<<blocks, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      if (rep) printf("DFMA threads/CTA=%d: %.2f TFLOP/s\n", threads, 2.0 * 8 * iters * (double)blocks * threads / (ms * 1e-3) / 1e12);
      cudaEventRecord(e0); k_dmma<<<blocks, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
      cudaEventElapsedTime(&ms, e0, e1);
      if (rep) printf("DMMA threads/CTA=%d: %.2f TFLOP/s\n", threads, 2.0 * 256 * 8 * iters * (double)blocks * (threads / 32) / (ms * 1e-3) / 1e12);
    }
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
