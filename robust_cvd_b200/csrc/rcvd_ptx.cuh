// rcvd_ptx.cuh -- the inline PTX of the device code (and the packed-triangle index it shares), each form defined once.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rcvd {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void dmma_8x8x4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// m16n8k4: two m8n8k4 units stacked in M that share the B fragment -- rows g (a0 -> c0, c1) and g + 8 (a1 -> c2, c3).
// On the H100 it issues at twice the fp64 rate of m8n8k4 (rcvd_debug_fp64_tensor_peak measures every shape live).
__device__ __forceinline__ void dmma_16x8x4(double& c0, double& c1, double& c2, double& c3, double a0, double a1, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3) : "d"(a0), "d"(a1), "d"(b));
}

// cp.async of 16 bytes through L2 only; the zero-fill form reads nothing and stores zeros when !valid
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async4_ca(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// cp.async.wait_group with a run-time count of groups that may stay in flight (0..3)
__device__ __forceinline__ void cp_async_wait_upto3(int n) {
  if (n >= 3) cp_async_wait<3>(); else if (n == 2) cp_async_wait<2>(); else if (n == 1) cp_async_wait<1>(); else cp_async_wait<0>();
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void prefetch_l2_bulk(const void* gmem, int bytes) { asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem), "r"(bytes) : "memory"); }

// GPU-scope flags between kernels that run at the same time (k_potrf_smem -> streamed k_trsm_ll, k_substitution).  The writer's CTA
// barrier orders every thread's stores before one thread's release (cumulativity), like cutlass::Semaphore::release.
__device__ __forceinline__ int ld_acquire_gpu(const int* p) { int v; asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_release_gpu(int* p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_release_add(int* p, int v) { asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// named barriers: the id and the thread count are immediates
template <int ID, int N> __device__ __forceinline__ void named_bar_sync() { asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory"); }
template <int ID, int N> __device__ __forceinline__ void named_bar_arrive() { asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(N) : "memory"); }

// Row and column (i, j) of entry t of a packed lower triangle stored row by row: t = i (i + 1) / 2 + j, 0 <= j <= i.  The float
// square root may round across a row boundary; the two loops correct it.  Index: int, or unsigned (blockIdx.x, converted as such).
template <class Index> __device__ __forceinline__ int2 tri_index(Index t) {
  int i = (int)((sqrtf(8.f * t + 1.f) - 1.f) * 0.5f);
  while ((i + 1) * (i + 2) / 2 <= (int)t) ++i;
  while (i * (i + 1) / 2 > (int)t) --i;
  return make_int2(i, (int)t - i * (i + 1) / 2);
}

}  // namespace rcvd
