// DMMA (mma.sync m8n8k4 f64) issue behaviour of a single warp / few warps per SM sub-core on sm_90a:
// cycles per DMMA for W warps per CTA (one CTA per SM) with ACC independent accumulators each, and DFMA for comparison.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/dmma_latency.bin tools/dmma_latency.cu
#include <cstdio>
#include <cuda_runtime.h>
template <int ACC> __global__ void k(double* out, long long* cyc, int iters) {
  double c[ACC][2];
#pragma unroll
  for (int i = 0; i < ACC; ++i) { c[i][0] = 0; c[i][1] = 0; }
  const double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < ACC; ++i)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
  }
  const long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < ACC; ++i) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int ACC> __global__ void kf(double* out, long long* cyc, int iters) {
  double c[ACC];
#pragma unroll
  for (int i = 0; i < ACC; ++i) c[i] = threadIdx.x * 1e-9 + i;
  const double b = 1.0000001, d = 1e-9;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < ACC; ++i) c[i] = fma(c[i], b, d);
  }
  const long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < ACC; ++i) s += c[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int ACC> void run(int sms, int warps, double* out, long long* dc) {
  const int iters = 2000; long long c = 0;
  k<ACC><<<sms, warps * 32>>>(out, dc, iters); cudaDeviceSynchronize(); cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
  printf("DMMA  warps/CTA=%2d acc=%2d: %.1f cycles per DMMA per warp\n", warps, ACC, (double)c / (iters * ACC));
  kf<ACC><<<sms, warps * 32>>>(out, dc, iters); cudaDeviceSynchronize(); cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
  printf("DFMA  warps/CTA=%2d acc=%2d: %.1f cycles per DFMA per warp\n", warps, ACC, (double)c / (iters * ACC));
}
int main() {
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  double* out; long long* dc; cudaMalloc(&out, (size_t)sms * 1024 * 8); cudaMalloc(&dc, 8);
  for (int w : {1, 4, 8, 16, 32}) { run<1>(sms, w, out, dc); run<4>(sms, w, out, dc); run<16>(sms, w, out, dc); }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
