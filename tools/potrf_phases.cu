// Cycle breakdown of k_potrf_smem (one CTA, npad = 208) from thread 0's point of view.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -DRCVD_POTRF_PHASES -I include -I robust_cvd_b200/csrc -o tools/potrf_phases.bin tools/potrf_phases.cu
#include <cstdio>
#include <vector>
#include <cmath>
#include "rcvd_linalg.cuh"
using namespace rcvd;
int main() {
  const int n = 208;
  std::vector<double> A((size_t)n * n);
  for (int i = 0; i < n; ++i) for (int j = 0; j <= i; ++j) { double v = std::sin(0.37 * i + 1.3 * j) * 0.5; if (i == j) v = n; A[(size_t)i * n + j] = v; A[(size_t)j * n + i] = v; }
  double *dA, *dT; int *dF, *dfail, *dprog; cudaMalloc(&dA, A.size() * 8); cudaMalloc(&dT, n * 16 * 8); cudaMalloc(&dF, 4); cudaMalloc(&dfail, 4); cudaMalloc(&dprog, 4);
  int zero = 0; cudaMemcpy(dF, &zero, 4, cudaMemcpyHostToDevice); cudaMemset(dfail, 0, 4);
  cudaFuncSetAttribute(k_potrf_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)potrf_smem_bytes(n));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int rep = 0; rep < 4; ++rep) {   // rep 0 warms up
    cudaMemcpy(dA, A.data(), A.size() * 8, cudaMemcpyHostToDevice);
    long long z[16] = {0}; cudaMemcpyToSymbol(g_potrf_phase, z, sizeof(z));
    cudaEventRecord(e0); k_potrf_smem<<<1, kPotrfSmemThreads, potrf_smem_bytes(n)>>>(dA, dT, dF, n, dfail, dprog); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    long long ph[16]; cudaMemcpyFromSymbol(ph, g_potrf_phase, sizeof(ph));
    printf("rep %d: %.1f us; cycles: load %lld, first chol %lld, panel(thread0) %lld, wait-panel %lld, update-to-lookahead %lld, lookahead chol %lld, rest of update %lld, wait-update %lld  (%s)\n",
           rep, ms * 1e3, ph[0], ph[1], ph[2], ph[3], ph[4], ph[5], ph[6], ph[7], cudaGetErrorString(cudaGetLastError()));
    printf("        blocked chol16 (14 tiles x 4 block steps): store+sync+block loads %lld, pivot chain %lld, row solves+sync %lld, diag rows+DMMA %lld\n", ph[8], ph[9], ph[10], ph[11]);
  }
  // correctness: compare with a plain host Cholesky
  std::vector<double> Lh = A, Ld((size_t)n * n);
  for (int j = 0; j < n; ++j) {
    double d = Lh[(size_t)j * n + j]; for (int k = 0; k < j; ++k) d -= Lh[(size_t)j * n + k] * Lh[(size_t)j * n + k];
    d = std::sqrt(d); Lh[(size_t)j * n + j] = d;
    for (int i = j + 1; i < n; ++i) { double v = Lh[(size_t)i * n + j]; for (int k = 0; k < j; ++k) v -= Lh[(size_t)i * n + k] * Lh[(size_t)j * n + k]; Lh[(size_t)i * n + j] = v / d; }
  }
  cudaMemcpy(Ld.data(), dA, Ld.size() * 8, cudaMemcpyDeviceToHost);
  double err = 0; for (int i = 0; i < n; ++i) for (int j = 0; j <= i; ++j) err = std::max(err, std::fabs(Ld[(size_t)i * n + j] - Lh[(size_t)i * n + j]));
  printf("max |L_gpu - L_host| = %.3e\n", err);
  return 0;
}
