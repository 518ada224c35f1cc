// fp64 tensor-core (DMMA m8n8k4) throughput on register / shared-memory operand patterns that a real GEMM inner loop has.
// The round-1 peak probe (rcvd_debug_fp64_tensor_peak) multiplies the SAME a, b registers into 8 accumulators; a GEMM warp tile of
// NI x NJ units feeds NI + NJ distinct fragments into NI * NJ accumulators and reloads them from shared memory every 4 k.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/dmma_patterns.bin tools/dmma_patterns.cu && tools/dmma_patterns.bin
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
template <int NI, int NJ, int MODE>   // MODE 0: fragments constant in registers; 1: reloaded from shared memory every step (conflict-free LDS.64)
__global__ void __launch_bounds__(128) k(double* out, int iters) {
  extern __shared__ double sm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 4 * 2 * 80 * 4; i += blockDim.x) sm[i] = 1.0 + 1e-9 * i;
  __syncthreads();
  double acc[NI][NJ][2];
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) { acc[i][j][0] = 0; acc[i][j][1] = 0; }
  double a[NI], b[NJ];
#pragma unroll
  for (int i = 0; i < NI; ++i) a[i] = 1e-3 * (lane + i);
#pragma unroll
  for (int j = 0; j < NJ; ++j) b[j] = 1.0 + 1e-6 * (lane + j);
  const double* base = sm + (warp & 1) * 320 + lane;     // 8 rows x 4 doubles of 32 B = 256 contiguous bytes per fragment: conflict-free
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      if (MODE == 1) {
#pragma unroll
        for (int i = 0; i < NI; ++i) a[i] = base[k4 * 640 + i * 32];
#pragma unroll
        for (int j = 0; j < NJ; ++j) b[j] = base[k4 * 640 + 160 + j * 32];
      }
#pragma unroll
      for (int i = 0; i < NI; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) dmma(acc[i][j][0], acc[i][j][1], a[i], b[j]);
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) s += acc[i][j][0] + acc[i][j][1];
  out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int NI, int NJ, int MODE> void run(const char* name, int ctas_per_sm) {
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  const int blocks = prop.multiProcessorCount * ctas_per_sm, iters = 4000;
  double* out; cudaMalloc(&out, (size_t)blocks * 128 * 8);
  cudaFuncSetAttribute(k<NI, NJ, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
  const size_t smem = ctas_per_sm <= 2 ? 100 * 1024 : 40 * 1024;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  double best = 0;
  for (int rep = 0; rep < 4; ++rep) {
    cudaEventRecord(e0); k<NI, NJ, MODE><<<blocks, 128, smem>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double tf = 512.0 * NI * NJ * 4 * iters * (double)blocks * 4 / (ms * 1e-3) / 1e12;
    if (rep && tf > best) best = tf;
  }
  printf("%-58s %d CTAs/SM (%2d warps/SM): %6.2f TFLOP/s  [%s]\n", name, ctas_per_sm, ctas_per_sm * 4, best, cudaGetErrorString(cudaGetLastError()));
  cudaFree(out);
}
int main() {
  run<2, 4, 0>("2x4 units, fragments constant in registers", 2); run<2, 4, 0>("2x4 units, fragments constant in registers", 4);
  run<4, 4, 0>("4x4 units, registers", 2); run<4, 4, 0>("4x4 units, registers", 4);
  run<5, 5, 0>("5x5 units, registers", 2);
  run<4, 4, 1>("4x4 units, fragments reloaded from smem every 4 k", 2); run<4, 4, 1>("4x4 units, fragments reloaded from smem every 4 k", 4);
  run<5, 5, 1>("5x5 units, fragments reloaded from smem every 4 k", 2);
  run<5, 4, 1>("5x4 units, smem", 2); run<4, 5, 1>("4x5 units, smem", 2);
  return 0;
}
