// rcvd_cg.cuh -- block-Jacobi preconditioned conjugate gradients on the damped normal equations (S H S + D2) y = S g.
//
// The linear solver of a single-GPU handle whose block-Cholesky storage (H, the factor with its fill, the off-diagonal factor blocks
// and the diagonal inverses) exceeds cholesky_budget: it needs H, the N damped diagonal blocks, their inverses and a few vectors.
// The diagonal blocks are factored and inverted by the block Cholesky's own per-frame kernels (k_load_factor, k_potrf_*, k_trinv,
// rcvd_linalg.cuh) and applied with its substitution GEMVs (k_fwd_diag, k_bwd_diag): z = L^-T L^-1 r frame by frame.
//
// Restated Ceres semantics: ConjugateGradientsSolver (ceres/conjugate_gradients_solver.h) as LevenbergMarquardtStrategy drives it
// (q_tolerance = eta = 0.1, r_tolerance disabled, min / max_num_iterations 0 / 500, residual_reset_period 10, x0 = 0).  Iteration i
// stops when i (Q_i - Q_i-1) / Q_i < eta, Q(x) = x'Ax - 2 b'x (Nash's truncated-Newton test), or at the cap, whose iterate is a
// usable step (Ceres' NO_CONVERGENCE).  b = 0 gives y = 0.  Where Ceres reports FAILURE (rho = r'z zero or infinite, beta zero or
// infinite, alpha infinite) or an indefinite matrix (p'q <= 0), and on any NaN in those scalars, the solve sets *fail: the LM loop
// treats the step as invalid.  tests/cg_ref.py is the numpy restatement.
//
// Every reduction is two-stage in a fixed order (per-CTA partials, then k_cg_scalar), and the SpMV writes per-block slots that one
// kernel sums per frame in a fixed order: no atomics, two runs give identical iterates and iteration counts.  The host enqueues the
// iterations in chunks of kCgChunk and reads CgState::stop once per chunk; every kernel of an iteration after the stop returns at
// once, so the result is the one a check after every iteration would give.
#pragma once
#include <cstdint>
#include "rcvd_plan.h"

namespace rcvd {

constexpr int kCgThreads = 256;
constexpr int kCgDotBlocks = 264;          // fixed grid of the vector kernels (2 per SM on an H100): their partials are summed in order
constexpr int kCgChunk = 10;               // iterations enqueued between two reads of CgState::stop
constexpr int kCgResetPeriod = 10;         // Ceres' residual_reset_period: r = b - A x instead of r - alpha q every 10th iteration
constexpr int kCgMaxIterations = 500;      // Solver::Options::max_linear_solver_iterations
constexpr double kCgEta = 0.1;             // Solver::Options::eta (the q_tolerance LevenbergMarquardtStrategy passes)

struct CgState {
  int stop;             // the solve has ended (converged, capped or broken down): later kernels of it return at once
  int iterations;       // iterations run
  int capped;           // it ended at max_iterations
  int max_iterations;
  double eta, rho, alpha, beta, q0;
};

enum { CG_INIT = 0, CG_RHO, CG_CURVATURE, CG_MODEL };

// The block Cholesky is chosen while its storage fits in 4/5 of the device's total memory; the rest holds the constraint records and
// the vectors.  Total, not free, memory: on a shared device the free memory changes from run to run, and so would the choice.
inline int64_t cholesky_budget(uint64_t device_total_bytes) { return (int64_t)(device_total_bytes / 5 * 4); }

inline int cg_partials(int N) { return N > kCgDotBlocks ? N : kCgDotBlocks; }   // k_cg_gather writes one per frame

// Device bytes of each linear solver for a plan (allocate_storage allocates exactly these).  Cholesky: H, the factor (diagonal, fill
// and off-diagonal blocks), the TRSM operand blocks T, the diagonal inverses and their 16 x 16 tile inverses.  CG: H, the N diagonal
// factors, their inverses and tile inverses, the SpMV slots (a row and a column slot per H block), r z p q, the partials, the per-frame
// slot lists, the state.
struct LinearStorage { int64_t cholesky, cg; };
inline LinearStorage linear_storage(const FactorPlan& pl, int N, int npad) {
  const int64_t bs = (int64_t)npad * npad * 8, nH = (int64_t)pl.hblocks.size(), Upad = (int64_t)N * npad, tiles = (int64_t)N * npad * 16 * 8;
  LinearStorage s;
  s.cholesky = bs * (nH + (N + pl.nLoff) + std::max(pl.nLoff, 1) + N) + tiles;
  s.cg = bs * (nH + 2 * (int64_t)N) + tiles + 8 * (2 * nH * npad + 4 * Upad + cg_partials(N)) + 4 * ((int64_t)N + 1 + 2 * nH + N) +
         (int64_t)sizeof(CgState);
  return s;
}

// Per frame, the SpMV slots that hold its part of A p: slot b (block b's rows, M v_c) when the frame is block b's row frame, slot
// nH + b (its columns, M^T v_r) when it is the column frame -- a diagonal block contributes both.  CSR over frames, ascending slots.
inline void cg_slot_lists(const FactorPlan& pl, int N, std::vector<int>& off, std::vector<int>& slots) {
  const int nH = (int)pl.hblocks.size();
  off.assign(N + 1, 0);
  for (const HBlock& b : pl.hblocks) { off[b.r + 1]++; off[b.c + 1]++; }
  for (int f = 0; f < N; ++f) off[f + 1] += off[f];
  slots.assign(2 * (size_t)nH, 0);
  std::vector<int> fill(off.begin(), off.end() - 1);
  for (int s = 0; s < 2 * nH; ++s) { const HBlock& b = pl.hblocks[s % nH]; slots[fill[s < nH ? b.r : b.c]++] = s; }
}

__device__ __forceinline__ double block_sum(double v, double* red /* [kCgThreads / 32] */) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kCgThreads / 32; ++w) t += red[w];
  return t;   // thread 0
}

// The SpMV H (S v) over the stored blocks, each read once: block b = (r, c) writes slot b = M (S v)_c over its rows and slot nH + b =
// M^T (S v)_r over its columns; a diagonal block holds its lower triangle, so it uses j <= i for the first and j < i for the second.
// One CTA per block, 8 warps over the rows, 256-column passes (8 columns per lane), the column partials summed over the warps in order.
// grid: H blocks; dynamic smem (3 npad + 8 x 256) doubles.  k_cg_spmv and k_cg_gather run unconditionally with st null (the timing hook).
__global__ void __launch_bounds__(kCgThreads) k_cg_spmv(const double* __restrict__ H, const HBlock* __restrict__ hb, const double* __restrict__ S,
                                                        const double* __restrict__ v, double* __restrict__ slots, int nH, int npad, int nf,
                                                        const CgState* __restrict__ st) {
  if (st && st->stop) return;
  extern __shared__ double sm[];
  double *vr = sm, *vc = sm + npad, *racc = vc + npad, *cred = racc + npad;
  const int b = blockIdx.x;
  const HBlock blk = hb[b];
  const bool diag = blk.r == blk.c;
  for (int i = threadIdx.x; i < npad; i += kCgThreads) {
    const size_t r = (size_t)blk.r * npad + i, c = (size_t)blk.c * npad + i;
    vr[i] = i < nf ? S[r] * v[r] : 0.0;
    vc[i] = i < nf ? S[c] * v[c] : 0.0;
    racc[i] = 0.0;
  }
  __syncthreads();
  const double* M = H + (size_t)b * npad * npad;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j0 = 0; j0 < nf; j0 += 256) {
    double cacc[8], vj[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { const int j = j0 + 32 * k + lane; cacc[k] = 0.0; vj[k] = j < nf ? vc[j] : 0.0; }
#pragma unroll 2
    for (int i = warp; i < nf; i += 8) {
      const double* Mi = M + (size_t)i * npad;
      double m[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) { const int j = j0 + 32 * k + lane; m[k] = j < nf ? __ldcs(Mi + j) : 0.0; }
      const double xi = vr[i];
      double s = 0.0;
      if (diag) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { const int j = j0 + 32 * k + lane; s += j <= i ? m[k] * vj[k] : 0.0; cacc[k] += j < i ? m[k] * xi : 0.0; }
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) { s += m[k] * vj[k]; cacc[k] += m[k] * xi; }
      }
      s = warp_sum(s);
      if (lane == 0) racc[i] += s;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) cred[warp * 256 + 32 * k + lane] = cacc[k];
    __syncthreads();
    const int j = j0 + threadIdx.x;
    if (j < nf) {
      double c = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) c += cred[w * 256 + threadIdx.x];
      slots[((size_t)nH + b) * npad + j] = c;
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < nf; i += kCgThreads) slots[(size_t)b * npad + i] = racc[i];
}

// out = S (sum of the frame's slots) + D2 v = (S H S + D2) v, zero in the padding; part[f] = v_f . out_f.  grid: N frames.
__global__ void __launch_bounds__(kCgThreads) k_cg_gather(const double* __restrict__ slots, const int* __restrict__ off, const int* __restrict__ ids,
                                                          const double* __restrict__ S, const double* __restrict__ D2, const double* __restrict__ v,
                                                          double* __restrict__ out, double* __restrict__ part, int npad, int nf,
                                                          const CgState* __restrict__ st) {
  __shared__ double red[kCgThreads / 32];
  if (st && st->stop) return;
  const int f = blockIdx.x, s0 = off[f], s1 = off[f + 1];
  double dot = 0.0;
  for (int i = threadIdx.x; i < npad; i += kCgThreads) {
    const size_t e = (size_t)f * npad + i;
    double o = 0.0;
    if (i < nf) {
      double s = 0.0;
      for (int q = s0; q < s1; ++q) s += slots[(size_t)ids[q] * npad + i];
      o = S[e] * s + D2[e] * v[e];
    }
    out[e] = o;
    dot += v[e] * o;
  }
  dot = block_sum(dot, red);
  if (threadIdx.x == 0) part[f] = dot;
}

// x = 0, r = b; part = partials of b.b
__global__ void __launch_bounds__(kCgThreads) k_cg_init(const double* __restrict__ b, double* __restrict__ x, double* __restrict__ r,
                                                        double* __restrict__ part, int n) {
  __shared__ double red[kCgThreads / 32];
  double dot = 0.0;
  for (int i = blockIdx.x * kCgThreads + threadIdx.x; i < n; i += gridDim.x * kCgThreads) { x[i] = 0.0; r[i] = b[i]; dot += b[i] * b[i]; }
  dot = block_sum(dot, red);
  if (threadIdx.x == 0) part[blockIdx.x] = dot;
}

// part = partials of a.b
__global__ void __launch_bounds__(kCgThreads) k_cg_dot(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ part, int n,
                                                       const CgState* __restrict__ st) {
  __shared__ double red[kCgThreads / 32];
  if (st->stop) return;
  double dot = 0.0;
  for (int i = blockIdx.x * kCgThreads + threadIdx.x; i < n; i += gridDim.x * kCgThreads) dot += a[i] * b[i];
  dot = block_sum(dot, red);
  if (threadIdx.x == 0) part[blockIdx.x] = dot;
}

// p = z (first iteration), p = z + beta p after
__global__ void __launch_bounds__(kCgThreads) k_cg_direction(const double* __restrict__ z, double* __restrict__ p, int n, const CgState* __restrict__ st) {
  if (st->stop) return;
  const bool first = st->iterations == 1;
  const double beta = st->beta;
  for (int i = blockIdx.x * kCgThreads + threadIdx.x; i < n; i += gridDim.x * kCgThreads) p[i] = first ? z[i] : z[i] + beta * p[i];
}

// The update of iteration i.  mode 0: x += alpha p, r -= alpha q.  The residual reset (every kCgResetPeriod-th iteration) is mode 1,
// x += alpha p, then q = A x (k_cg_spmv + k_cg_gather), then mode 2, r = b - q.  Modes 0 and 2: part = partials of x.(b + r), -Q(x).
__global__ void __launch_bounds__(kCgThreads) k_cg_step(double* __restrict__ x, const double* __restrict__ p, double* __restrict__ r,
                                                        const double* __restrict__ q, const double* __restrict__ b, double* __restrict__ part, int n,
                                                        int mode, const CgState* __restrict__ st) {
  __shared__ double red[kCgThreads / 32];
  if (st->stop) return;
  const double alpha = st->alpha;
  double dot = 0.0;
  for (int i = blockIdx.x * kCgThreads + threadIdx.x; i < n; i += gridDim.x * kCgThreads) {
    double xi = x[i];
    if (mode <= 1) { xi += alpha * p[i]; x[i] = xi; }
    if (mode == 1) continue;
    const double ri = mode == 0 ? r[i] - alpha * q[i] : b[i] - q[i];
    r[i] = ri;
    dot += xi * (b[i] + ri);
  }
  if (mode == 1) return;
  dot = block_sum(dot, red);
  if (threadIdx.x == 0) part[blockIdx.x] = dot;
}

// The scalar decisions of the iteration, one CTA: v = sum of part[0, n) in a fixed order, then
//   CG_INIT       v = b.b: the state of a new solve; b = 0 ends it at once (y = 0)
//   CG_RHO        v = r.z: iteration i = iterations + 1 starts; rho, beta = rho / rho_prev
//   CG_CURVATURE  v = p.q: alpha = rho / p.q
//   CG_MODEL      v = x.(b + r) = -Q(x_i): the quadratic-model test, then the iteration cap
__global__ void __launch_bounds__(kCgThreads) k_cg_scalar(const double* __restrict__ part, int n, CgState* __restrict__ st, int* __restrict__ fail,
                                                          int phase, double eta, int max_iterations) {
  __shared__ double red[kCgThreads / 32];
  if (phase != CG_INIT && st->stop) return;
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += kCgThreads) v += part[i];
  v = block_sum(v, red);
  if (threadIdx.x != 0) return;
  bool broke = false;
  switch (phase) {
    case CG_INIT:
      st->stop = v == 0.0; st->iterations = 0; st->capped = 0; st->max_iterations = max_iterations;
      st->eta = eta; st->rho = 1.0; st->alpha = 0.0; st->beta = 0.0; st->q0 = 0.0;   // x0 = 0: Q(x0) = 0
      break;
    case CG_RHO: {
      const int i = ++st->iterations;
      const double last = st->rho;
      st->rho = v;
      broke = v == 0.0 || !isfinite(v);
      if (!broke && i > 1) { st->beta = v / last; broke = st->beta == 0.0 || !isfinite(st->beta); }
      break;
    }
    case CG_CURVATURE:
      broke = !(v > 0.0) || isinf(v);
      if (!broke) { st->alpha = st->rho / v; broke = !isfinite(st->alpha); }
      break;
    default: {
      const double q1 = -v, zeta = st->iterations * (q1 - st->q0) / q1;
      if (zeta < st->eta) { st->stop = 1; break; }
      st->q0 = q1;
      if (st->iterations >= st->max_iterations) { st->stop = 1; st->capped = 1; }
    }
  }
  if (broke) { st->stop = 1; *fail = 1; }
}

}  // namespace rcvd
