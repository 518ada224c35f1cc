// rcvd_linalg.cuh -- exact block-sparse Cholesky of the damped normal equations on device.
//
// The reference solves (J_s^T J_s + D^2) y = J_s^T r with Ceres' SPARSE_NORMAL_CHOLESKY
// (lib/PoseOptimizer.cpp:956).  Here the matrix is block-sparse over frames (one dense
// npad x npad block per coupled frame pair, npad = per-frame unknowns rounded to 16);
// a fill-reducing elimination order and level schedule are computed once on the host and
// the numeric work runs as batched per-level kernels:
//   k_potrf   (one CTA per diagonal block)      L_kk, plus 16x16 diagonal-tile inverses
//   k_trinv   (one CTA per 16-column panel)     inv(L_kk)
//   k_gemm_nt (fp64 tensor-core DMMA, 64x64)    X_rk = A_rk inv(L_kk)^T  (large blocks; k_trsm_ll below otherwise)
//   k_update_tma (rcvd_update.cuh)              A_rc -= X_rk X_ck^T
// and the triangular solves become GEMVs with inv(L_kk).
#pragma once
#include "rcvd_device.cuh"
#include "rcvd_ptx.cuh"

namespace rcvd {

// ---------------------------------------------------------------------------
// Large diagonal blocks (npad > 224: the lower triangle no longer fits in one CTA's shared memory), right-looking with
// 16-wide panels, TWO launches per panel so that the O(n^3) trailing update runs on the whole machine:
//   k_potrf_panel (one CTA per frame)            pivot-tile Cholesky + tile inverse (-> invT) + panel X = A Di^T
//   k_potrf_trail (64x64 tiles x frames, DMMA)   A[i][j] -= X_i X_j^T on the trailing lower triangle
// (a single-CTA version of this loop spent 6.5 ms per level at npad = 784; `bench.py --workload config4... --frames 160`).
// ---------------------------------------------------------------------------
constexpr int kPotrfThreads = 256;

__global__ void __launch_bounds__(kPotrfThreads) k_potrf_panel(double* __restrict__ Lb, double* __restrict__ invT,
                                                                const int* __restrict__ frames, int npad, int jb, int* __restrict__ fail) {
  __shared__ double D[16][17];
  __shared__ double Di[16][17];
  const int frame = frames[blockIdx.x];
  double* A = Lb + (size_t)frame * npad * npad;
  double* iT = invT + (size_t)frame * npad * 16;   // nt tiles of 16x16
  const int tid = threadIdx.x;
  const int j0 = jb * 16;
  {
    const int r = tid >> 4, cc = tid & 15;
    D[r][cc] = (cc <= r) ? A[(size_t)(j0 + r) * npad + j0 + cc] : 0.0;
  }
  __syncthreads();
  if (tid < 32) {
    // unblocked Cholesky of the 16x16 tile, lane i owns row i
    const int i = tid;
    for (int j = 0; j < 16; ++j) {
      if (i == j) {
        double d = D[j][j];
        for (int q = 0; q < j; ++q) d -= D[j][q] * D[j][q];
        if (!(d > 0.0) || !isfinite(d)) { *fail = 1; d = 1.0; }
        D[j][j] = sqrt(d);
      }
      __syncwarp();
      if (i > j && i < 16) {
        double s = D[i][j];
        for (int q = 0; q < j; ++q) s -= D[i][q] * D[j][q];
        D[i][j] = s / D[j][j];
      }
      __syncwarp();
    }
    // inverse of the lower-triangular tile: lane c computes column c
    if (i < 16) {
      const int cidx = i;
      double xcol[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        double s = (r == cidx) ? 1.0 : 0.0;
#pragma unroll
        for (int q = 0; q < 16; ++q) if (q < r) s -= D[r][q] * xcol[q];
        xcol[r] = (r < cidx) ? 0.0 : s / D[r][r];
      }
#pragma unroll
      for (int r = 0; r < 16; ++r) Di[r][cidx] = xcol[r];
    }
  }
  __syncthreads();
  {
    const int r = tid >> 4, cc = tid & 15;
    A[(size_t)(j0 + r) * npad + j0 + cc] = D[r][cc];
    iT[(size_t)jb * 256 + r * 16 + cc] = Di[r][cc];
  }
  // panel solve: X[i][:] = A[i][j0..j0+15] * Di^T for rows below the tile
  const int below = npad - (j0 + 16);
  for (int rr = tid; rr < below; rr += kPotrfThreads) {
    double a[16], xo[16];
    double* row = A + (size_t)(j0 + 16 + rr) * npad + j0;
#pragma unroll
    for (int q = 0; q < 16; ++q) a[q] = row[q];
#pragma unroll
    for (int cc = 0; cc < 16; ++cc) {
      double s = 0.0;
#pragma unroll
      for (int q = 0; q < 16; ++q) if (q <= cc) s += a[q] * Di[cc][q];
      xo[cc] = s;
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) row[q] = xo[q];
  }
}

// ---------------------------------------------------------------------------
// k_potrf_smem: same factorisation with the whole lower triangle resident in shared memory
// (npad <= 224: 105 tiles x 2 KB = 210 KB of the 227 KB a CTA may use).  Tiles are 16x16
// doubles, XOR-swizzled (element (r,k) at r*16 + (k ^ 4*(r&3))) so that the fp64 tensor-core
// fragment loads of the panel / trailing updates are bank-conflict free without padding.
// ---------------------------------------------------------------------------
constexpr int kPotrfSmemThreads = 512;
constexpr int kTileSz = 256;
constexpr size_t kMaxDynSmem = 220 * 1024;   // dynamic shared memory a factorisation kernel may use (factor_kernels picks the variants by it)
__host__ __device__ inline size_t potrf_smem_bytes(int npad) { const int nt = npad / 16; return (size_t)(nt * (nt + 1) / 2 + 1) * kTileSz * sizeof(double); }
__device__ __forceinline__ int swz(int r, int k) { return r * 16 + (k ^ ((r & 3) << 2)); }

// C(16x16) = A(16x16) * B(16x16)^T into acc[i8][j8][2] with DMMA; A, B swizzled tiles in smem.
__device__ __forceinline__ void tile_mma_nt(const double* __restrict__ At, const double* __restrict__ Bt, double acc[2][2][2], int g, int t) {
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4) {
    double af[2], bf[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) { af[i] = At[swz(i * 8 + g, k4 * 4 + t)]; bf[i] = Bt[swz(i * 8 + g, k4 * 4 + t)]; }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) dmma_8x8x4(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
  }
}

#ifdef RCVD_POTRF_PHASES   // tools/potrf_phases.cu: cycle counts per phase of CTA 0 (thread 0's view)
__device__ long long g_potrf_phase[16];
#define POTRF_PHASE(n) do { if (threadIdx.x == 0 && blockIdx.x == 0) { const long long now_ = clock64(); g_potrf_phase[n] += now_ - last_; last_ = now_; } } while (0)
#define CHOL_PHASE(n) do { if (threadIdx.x == 0 && blockIdx.x == 0) { const long long now_ = clock64(); g_potrf_phase[n] += now_ - cl_; cl_ = now_; } } while (0)
#else
#define CHOL_PHASE(n) do { } while (0)
#define POTRF_PHASE(n) do { } while (0)
#endif

// 4x4-blocked Cholesky of one 16x16 tile by a single warp.  Column by column with one row per lane, the pivot chain is 16 x (shuffle,
// rsqrt, mul, 15 shuffle+FMA column updates) ~ 5.6 k cycles, most of it the shuffle traffic of the rank-1 updates.  Here the tile lives in
// the DMMA accumulator fragments (three 8x8 units of the lower triangle); per block of four columns every lane factors the 4x4 diagonal
// block redundantly from ten broadcast shared-memory loads (no communication inside the four-pivot chain), the lanes of the rows below
// solve their 4-wide panel row, and the rank-4 trailing update is three DMMA.8x8x4 with K = 4.  Writes L back to the swizzled tile
// (lower triangle) and the reciprocal pivots 1/l_jj to pinv[0..15].
__device__ __forceinline__ void warp_chol16_blocked(double* __restrict__ D, double* __restrict__ pinv, int lane, int* __restrict__ fail) {
  const int g = lane >> 2, t = lane & 3;
  double c[3][2];                                  // units (0,0), (1,0), (1,1): rows 8*ui + g, columns 8*uj + 2t, + 1
  const int ui[3] = {0, 1, 1}, uj[3] = {0, 0, 1};
#pragma unroll
  for (int u = 0; u < 3; ++u) { const double2 v = *reinterpret_cast<const double2*>(&D[swz(8 * ui[u] + g, 8 * uj[u] + 2 * t)]); c[u][0] = v.x; c[u][1] = v.y; }
  bool bad = false;
#ifdef RCVD_POTRF_PHASES
  long long cl_ = clock64();
#endif
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const int k0 = 4 * b;
    if (b > 0) {
      // the trailing part of the fragments (columns >= k0) goes back to shared memory; columns < k0 there already hold L
#pragma unroll
      for (int u = 0; u < 3; ++u) if (8 * uj[u] + 2 * t >= k0) *reinterpret_cast<double2*>(&D[swz(8 * ui[u] + g, 8 * uj[u] + 2 * t)]) = make_double2(c[u][0], c[u][1]);
    }
    __syncwarp();
    // 1. the 4x4 diagonal block, on every lane (broadcast loads)
    double a00 = D[swz(k0, k0)], a10 = D[swz(k0 + 1, k0)], a11 = D[swz(k0 + 1, k0 + 1)], a20 = D[swz(k0 + 2, k0)], a21 = D[swz(k0 + 2, k0 + 1)],
           a22 = D[swz(k0 + 2, k0 + 2)], a30 = D[swz(k0 + 3, k0)], a31 = D[swz(k0 + 3, k0 + 1)], a32 = D[swz(k0 + 3, k0 + 2)], a33 = D[swz(k0 + 3, k0 + 3)];
    CHOL_PHASE(8);
    // Pivots in PAIRS: for the 2x2 leading block [[a, b], [b, c]] the second reciprocal pivot is 1/sqrt(c - b^2/a) = rsqrt(a c - b^2) sqrt(a),
    // so rsqrt(a) and rsqrt(a c - b^2) issue side by side (the determinant carries the same cancellation error, relative to the pivot,
    // as c - (b/sqrt a)^2 does) -- two rsqrt latencies per 4x4 block on the dependent chain instead of four.
    double t01 = a10 * a10;
    double det01 = fma(a00, a11, -t01);
    if (!(a00 > 0.0) || !isfinite(a00)) { bad = true; a00 = 1.0; det01 = 1.0; }
    if (!(det01 > 0.0) || !isfinite(det01)) { bad = true; det01 = a00; }
    const double p0 = rsqrt(a00), r01 = rsqrt(det01);
    const double sq0 = a00 * p0;                    // sqrt(a00) = L[0][0]
    const double p1 = r01 * sq0;
    const double l11 = det01 * r01 * p0;            // sqrt(det01 / a00) = L[1][1]
    const double l10 = a10 * p0, l20 = a20 * p0, l30 = a30 * p0;
    const double l21 = (a21 - l20 * l10) * p1, l31 = (a31 - l30 * l10) * p1;
    double b22 = fma(-l21, l21, fma(-l20, l20, a22)), b33 = fma(-l31, l31, fma(-l30, l30, a33));
    const double b32 = fma(-l31, l21, fma(-l30, l20, a32));
    double det23 = fma(b22, b33, -(b32 * b32));
    if (!(b22 > 0.0) || !isfinite(b22)) { bad = true; b22 = 1.0; det23 = 1.0; }
    if (!(det23 > 0.0) || !isfinite(det23)) { bad = true; det23 = b22; }
    const double p2 = rsqrt(b22), r23 = rsqrt(det23);
    const double sq2 = b22 * p2;
    const double p3 = r23 * sq2;
    const double l33 = det23 * r23 * p2;
    const double l32 = b32 * p2;
    CHOL_PHASE(9);
    // 2. block column k0 .. k0+3 of L: lane r (< 16) owns row r.  Rows below the block are solved here (their values are read by no
    //    other lane in step 1); the rows of the diagonal block itself are written after the warp barrier below, when every lane has
    //    read the block.  Branch-free so that the four solves interleave with the pivot chain above.
    const int r = lane & 15;
    const bool below = lane < 16 && r >= k0 + 4;
    double x0 = D[swz(r, k0)] * p0;
    double x1 = (D[swz(r, k0 + 1)] - x0 * l10) * p1;
    double x2 = (D[swz(r, k0 + 2)] - x0 * l20 - x1 * l21) * p2;
    double x3 = (D[swz(r, k0 + 3)] - x0 * l30 - x1 * l31 - x2 * l32) * p3;
    if (below) { D[swz(r, k0)] = x0; D[swz(r, k0 + 1)] = x1; D[swz(r, k0 + 2)] = x2; D[swz(r, k0 + 3)] = x3; }
    __syncwarp();
    CHOL_PHASE(10);
    if (lane == 0) {                                // the diagonal block itself (zeros above the diagonal) and the reciprocal pivots:
      // every lane holds them, one lane stores them (per-row selects on four lanes compiled to a three-way divergent branch)
      *reinterpret_cast<double2*>(&D[swz(k0, k0)]) = make_double2(sq0, 0.0);         *reinterpret_cast<double2*>(&D[swz(k0, k0 + 2)]) = make_double2(0.0, 0.0);
      *reinterpret_cast<double2*>(&D[swz(k0 + 1, k0)]) = make_double2(l10, l11);     *reinterpret_cast<double2*>(&D[swz(k0 + 1, k0 + 2)]) = make_double2(0.0, 0.0);
      *reinterpret_cast<double2*>(&D[swz(k0 + 2, k0)]) = make_double2(l20, l21);          *reinterpret_cast<double2*>(&D[swz(k0 + 2, k0 + 2)]) = make_double2(sq2, 0.0);
      *reinterpret_cast<double2*>(&D[swz(k0 + 3, k0)]) = make_double2(l30, l31);          *reinterpret_cast<double2*>(&D[swz(k0 + 3, k0 + 2)]) = make_double2(l32, l33);
      *reinterpret_cast<double2*>(&pinv[k0]) = make_double2(p0, p1);                      *reinterpret_cast<double2*>(&pinv[k0 + 2]) = make_double2(p2, p3);
    }
    // 3. rank-4 trailing update of rows / columns >= k0 + 4 on the tensor cores (operands of eliminated rows masked to zero)
    if (b < 3) {
      double pa[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) { const int r = 8 * i + g; pa[i] = r >= k0 + 4 ? D[swz(r, k0 + t)] : 0.0; }
#pragma unroll
      for (int u = 0; u < 3; ++u) dmma_8x8x4(c[u][0], c[u][1], -pa[ui[u]], pa[uj[u]]);
    }
    CHOL_PHASE(11);
  }
  if (bad && lane == 0) *fail = 1;
}


// Tile column jb of L is final at the end of tile step jb.  The worker warps store it to Lb at the start of step jb + 1, while the
// chain warp works alone before barrier 2, and then publish progress[frame] = jb + 1 (the last column after the loop): the streamed
// k_trsm_ll reads row panel jt of L and the tile inverse Di_jt as soon as progress reaches jt + 1.  Every step runs even after a
// non-positive pivot (*fail is set, the pivot replaced), so the counter always reaches nt.
__global__ void __launch_bounds__(kPotrfSmemThreads) k_potrf_smem(double* __restrict__ Lb, double* __restrict__ invT,
                                                                   const int* __restrict__ frames, int npad, int* __restrict__ fail,
                                                                   int* __restrict__ progress) {
  // Launched as a programmatic dependent of the previous level's U1 on the narrow levels: wait for it (and its memory) before reading
  // anything; a no-op after an ordinary launch dependency.  Then this CTA's inputs are complete, and a programmatic dependent launch
  // (the streamed k_trsm_ll, which reads blocks U1 updated) may start beside it.
  griddep_wait();
  griddep_launch_dependents();
  extern __shared__ __align__(16) double tiles[];
  const int frame = frames[blockIdx.x];
  double* A = Lb + (size_t)frame * npad * npad;
  double* iT = invT + (size_t)frame * npad * 16;
  const int nt = npad / 16, ntl = nt * (nt + 1) / 2;
  double* pinv = tiles + (size_t)ntl * kTileSz;     // [npad] reciprocal pivots (fits the spare 2 KB tile for npad <= 256)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = kPotrfSmemThreads / 32;
  const int g = lane >> 2, t = lane & 3;
  // worker warps only: store tile column jc to Lb (16-byte chunks, 128 contiguous bytes per row; the diagonal tile's upper triangle
  // zeroed), meet on barrier 3, then one thread publishes jc + 1
  auto publish = [&](int jc) {
    for (int idx = tid - 32; idx < (nt - jc) * 128; idx += kPotrfSmemThreads - 32) {
      const int ti = jc + (idx >> 7), e = idx & 127, r = e >> 3, c = (e & 7) * 2;
      double2 v = *reinterpret_cast<const double2*>(&tiles[(size_t)(ti * (ti + 1) / 2 + jc) * kTileSz + swz(r, c)]);
      if (ti == jc) { if (c > r) v.x = 0.0; if (c + 1 > r) v.y = 0.0; }
      *reinterpret_cast<double2*>(&A[(size_t)(ti * 16 + r) * npad + jc * 16 + c]) = v;
    }
    named_bar_sync<3, kPotrfSmemThreads - 32>();
    if (tid == 32) st_release_gpu(progress + frame, jc + 1);
  };
#ifdef RCVD_POTRF_PHASES
  long long last_ = clock64();
#endif
  // asynchronous tile load: 16-byte chunks (the swizzle keeps aligned pairs together), all in flight at once
  for (int idx = tid; idx < ntl * 128; idx += kPotrfSmemThreads) {
    const int tl = idx >> 7, e = idx & 127, r = e >> 3, c = (e & 7) * 2;
    const int2 tij = tri_index(tl);
    cp_async16(&tiles[(size_t)tl * kTileSz + swz(r, c)], &A[(size_t)(tij.x * 16 + r) * npad + tij.y * 16 + c]);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  POTRF_PHASE(0);
  if (warp == 0) warp_chol16_blocked(tiles, pinv, lane, fail);
  __syncthreads();
  POTRF_PHASE(1);
  for (int jb = 0; jb < nt; ++jb) {
    const double* D = tiles + (size_t)(jb * (jb + 1) / 2 + jb) * kTileSz;
    const double* pv = pinv + jb * 16;
    // ---- panel by forward substitution (one thread per row below the tile); warp nw-1 computes the tile inverse ----
    // Warp 0, the chain warp, solves only the rows of tile (jb+1, jb) -- all its lookahead needs -- updates tile (jb+1, jb+1),
    // ARRIVES on named barrier 2 and factors the tile; the other warps SYNC on barrier 2 before they start their panel rows, so the
    // chain warp has the shared-memory pipe and the fp64 pipe to itself for its short serial part, and the others' panel + trailing
    // tiles run beside the next pivot tile's Cholesky.  (tools/potrf_phases.cu, thread 0's view of one step when every warp entered
    // the panel and the DMMA section together and the pivot tile was a shuffle chain: panel 1.45 k -- 152 broadcast LDS per row
    // thread, LSU-bound -- + barrier 0.2 k + own tile update 1.4 k cycles, next to 5.3 k of Cholesky.)
    const int rows = (nt - jb - 1) * 16;
    int prow = -1;                                   // this thread's panel row (index below the pivot tile), -1: none
    // (keeping the warps that share the chain warp's scheduler idle made the pivot tile faster, 4.3 k -> 3.9 k cycles, and the other
    // warps' trailing update slower by more: 2.77 against 2.68 ms per factorisation)
    const int nwork = nw - 1, widx = warp - 1;       // worker warps beside the chain warp
    if (warp == 0) { if (lane < 16 && rows > 0) prow = lane; } else if (widx * 32 + lane < rows - 16) prow = 16 + widx * 32 + lane;
    if (warp != 0) {
      if (jb > 0) publish(jb - 1);                   // in the time the chain warp needs before it arrives on barrier 2
      named_bar_sync<2, kPotrfSmemThreads>();
    }
    if (prow >= 0) {
      const int ti = jb + 1 + (prow >> 4), r = prow & 15;
      double* Tt = tiles + (size_t)(ti * (ti + 1) / 2 + jb) * kTileSz;
      double a[16];
#pragma unroll
      for (int q = 0; q < 16; q += 2) { const double2 v = *reinterpret_cast<const double2*>(&Tt[swz(r, q)]); a[q] = v.x; a[q + 1] = v.y; }
      // right-looking substitution: once x_q is final every later column takes its term at once (independent FMAs) -- the dependent
      // chain is one multiply + one FMA per column instead of the 120 chained FMAs of the dot-product form.  Two columns per pass so
      // that L comes in as 16-byte pairs (64 + 16 shared-memory loads per row instead of 120 + 32: the panel is LSU-bound).
#pragma unroll
      for (int q = 0; q < 16; q += 2) {
        const double2 pq = *reinterpret_cast<const double2*>(&pv[q]);
        const double2 dq = *reinterpret_cast<const double2*>(&D[swz(q + 1, q)]);     // L[q+1][q], (L[q+1][q+1] unused)
        a[q] *= pq.x;
        a[q + 1] = (a[q + 1] - a[q] * dq.x) * pq.y;
#pragma unroll
        for (int c = 0; c < 16; ++c) if (c > q + 1) { const double2 l = *reinterpret_cast<const double2*>(&D[swz(c, q)]); a[c] -= a[q] * l.x; a[c] -= a[q + 1] * l.y; }
      }
#pragma unroll
      for (int q = 0; q < 16; q += 2) *reinterpret_cast<double2*>(&Tt[swz(r, q)]) = make_double2(a[q], a[q + 1]);
    } else if (warp == nw - 1 && lane < 16) {
      // inverse of the triangular tile (only needed by k_trinv): column `lane`, forward substitution
      const int cidx = lane;
      double xcol[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) xcol[r] = (r == cidx) ? 1.0 : 0.0;
#pragma unroll
      for (int q = 0; q < 16; q += 2) {            // right-looking, two columns per pass, like the panel rows
        const double2 pq = *reinterpret_cast<const double2*>(&pv[q]);
        const double2 dq = *reinterpret_cast<const double2*>(&D[swz(q + 1, q)]);
        xcol[q] *= pq.x;
        xcol[q + 1] = (xcol[q + 1] - xcol[q] * dq.x) * pq.y;
#pragma unroll
        for (int r = 0; r < 16; ++r) if (r > q + 1) { const double2 l = *reinterpret_cast<const double2*>(&D[swz(r, q)]); xcol[r] -= l.x * xcol[q]; xcol[r] -= l.y * xcol[q + 1]; }
      }
#pragma unroll
      for (int r = 0; r < 16; ++r) iT[(size_t)jb * 256 + r * 16 + cidx] = xcol[r];
    }
    POTRF_PHASE(2);
    if (warp != 0) named_bar_sync<3, kPotrfSmemThreads - 32>();
    POTRF_PHASE(3);
    // ---- trailing update (DMMA) with lookahead: warp 0 updates tile (jb+1, jb+1) first and factors it at once ----
    const int m = nt - jb - 1, ntr = m * (m + 1) / 2;
    auto upd_tile = [&](int gi, int gj) -> double* {
      const double* Xi = tiles + (size_t)(gi * (gi + 1) / 2 + jb) * kTileSz;
      const double* Xj = tiles + (size_t)(gj * (gj + 1) / 2 + jb) * kTileSz;
      double* Ct = tiles + (size_t)(gi * (gi + 1) / 2 + gj) * kTileSz;
      double acc[2][2][2] = {{{0.0, 0.0}, {0.0, 0.0}}, {{0.0, 0.0}, {0.0, 0.0}}};
      tile_mma_nt(Xi, Xj, acc, g, t);
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          double2* ptr = reinterpret_cast<double2*>(&Ct[swz(i * 8 + g, j * 8 + 2 * t)]);
          double2 v = *ptr; v.x -= acc[i][j][0]; v.y -= acc[i][j][1]; *ptr = v;
        }
      return Ct;
    };
    // warp 0 owns the chain (measured: 88.7 -> 83.0 us per 208x208 block in tools/potrf_phases.cu, against every warp taking
    // trailing tiles): its panel rows, tile (jb+1, jb+1) and the next pivot tile, with the SM to itself until it arrives on barrier 2
    if (warp == 0) {
      double* Ct = nullptr;
      if (ntr > 0) { __syncwarp(); Ct = upd_tile(jb + 1, jb + 1); }
      __threadfence_block();
      named_bar_arrive<2, kPotrfSmemThreads>();
      POTRF_PHASE(4);
      if (ntr > 0) { __syncwarp(); warp_chol16_blocked(Ct, pinv + (jb + 1) * 16, lane, fail); }
      POTRF_PHASE(5);
    } else {
      for (int tl = 1 + widx; tl < ntr; tl += nwork) { const int2 tij = tri_index(tl); upd_tile(jb + 1 + tij.x, jb + 1 + tij.y); }   // tl = 0 is (jb+1, jb+1)
    }
    POTRF_PHASE(6);
    __syncthreads();
    POTRF_PHASE(7);
  }
  if (warp != 0) publish(nt - 1);
}

// ---------------------------------------------------------------------------
// k_trinv: inv(L_kk), one CTA per 16-column panel j; forward substitution by tiles using the
// diagonal-tile inverses from k_potrf.  Writes the full npad x npad block (zeros above).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_trinv(const double* __restrict__ Lb, const double* __restrict__ invT, double* __restrict__ invL,
                                                const int* __restrict__ frames, int npad) {
  extern __shared__ double Z[];   // [nt][16][16] tile column j of the inverse (tiles >= j), then the staged L row panel [16][npad+1]
  __shared__ double W[16][17];
  const int frame = frames[blockIdx.y];
  const int j = blockIdx.x;
  const int nt = npad / 16;
  double* Lrow_s = Z + (size_t)nt * 256;
  const int ldp = npad + 1;
  const double* A = Lb + (size_t)frame * npad * npad;
  const double* iT = invT + (size_t)frame * npad * 16;
  double* out = invL + (size_t)frame * npad * npad;
  const int tid = threadIdx.x, r = tid >> 4, c = tid & 15;
  for (int i = 0; i < j; ++i) out[(size_t)(i * 16 + r) * npad + j * 16 + c] = 0.0;
  Z[(size_t)j * 256 + tid] = iT[(size_t)j * 256 + tid];
  out[(size_t)(j * 16 + r) * npad + j * 16 + c] = Z[(size_t)j * 256 + tid];
  __syncthreads();
  for (int i = j + 1; i < nt; ++i) {
    // stage L[i*16 .. i*16+15][j*16 .. i*16-1] (coalesced 128 B row segments)
    const int kw = (i - j) * 16;
    for (int e = tid; e < 16 * kw; e += 256) { const int rr = e / kw, kk = e % kw; Lrow_s[rr * ldp + kk] = A[(size_t)(i * 16 + rr) * npad + j * 16 + kk]; }
    __syncthreads();
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    const double* lr = Lrow_s + r * ldp;
    const double* zp = Z + (size_t)j * 256 + c;
    for (int kk = 0; kk < kw; kk += 4) {     // kw is a multiple of 16
      s0 += lr[kk] * zp[(size_t)kk * 16]; s1 += lr[kk + 1] * zp[(size_t)(kk + 1) * 16];
      s2 += lr[kk + 2] * zp[(size_t)(kk + 2) * 16]; s3 += lr[kk + 3] * zp[(size_t)(kk + 3) * 16];
    }
    W[r][c] = (s0 + s1) + (s2 + s3);
    __syncthreads();
    double zv = 0.0;
    const double* ti = iT + (size_t)i * 256;
#pragma unroll
    for (int q = 0; q < 16; ++q) zv -= ti[r * 16 + q] * W[q][c];
    Z[(size_t)i * 256 + tid] = zv;
    out[(size_t)(i * 16 + r) * npad + j * 16 + c] = zv;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// k_gemm_nt: the TRSM of the large-block path (npad > 416, where a k_trsm_ll strip no longer fits in shared memory),
// T[t.dst] = Lb[t.src] * invL[t.kframe]^T for the task t of blockIdx.z, with inv(L_kk) lower triangular.
// fp64 tensor cores (mma.sync m8n8k4 -> DMMA), CTA tile 64x64, 4 warps of 32x32,
// K staged 16 at a time through a cp.async double buffer.  The short last tile row is cheap because out-of-range mma tiles
// are never issued.
// ---------------------------------------------------------------------------
struct TrsmTask { int dst; int src; int kframe; };   // T index, L block id, column frame (the task of k_gemm_nt and of k_trsm_ll)

constexpr int kGemmLd = 20;   // padded leading dimension of the 64x16 smem tiles (conflict-free DMMA fragment loads)

// One 16-deep K stage of a warp's (NI*8) x (NJ*8) sub-tile: NI/NJ are compile-time so that no tensor instruction is predicated
// (a predicated mma.sync costs a WARPSYNC + branch pair each).
template <int NI, int NJ>
__device__ __forceinline__ void gemm_stage(const double* __restrict__ as, const double* __restrict__ bsm, double (&acc)[4][4][2], int wm, int wn, int g, int t) {
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4) {
    double af[NI > 0 ? NI : 1], bf[NJ > 0 ? NJ : 1];
#pragma unroll
    for (int i = 0; i < NI; ++i) af[i] = as[(wm + i * 8 + g) * kGemmLd + k4 * 4 + t];
#pragma unroll
    for (int j = 0; j < NJ; ++j) bf[j] = bsm[(wn + j * 8 + g) * kGemmLd + k4 * 4 + t];
#pragma unroll
    for (int i = 0; i < NI; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) dmma_8x8x4(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
  }
}

__global__ void __launch_bounds__(128, 4) k_gemm_nt(double* __restrict__ T, const double* __restrict__ Lb, const double* __restrict__ invL,
                                                  const TrsmTask* __restrict__ tasks, int npad) {
  __shared__ __align__(16) double As[2][64 * kGemmLd];
  __shared__ __align__(16) double Bs[2][64 * kGemmLd];
  const TrsmTask task = tasks[blockIdx.z];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const size_t bs = (size_t)npad * npad;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const int g = lane >> 2, t = lane & 3;
  // B lower triangular (inv(L_kk)): B[n][k] = 0 for k > n, so only K chunks up to this tile's last column matter
  const int kchunks = min(npad, n0 + 64) / 16;
  // 8-row / 8-column mma tiles of this warp that lie inside the matrix (npad is a multiple of 16, tiles are 64 -> ni, nj in {0, 2, 4})
  const int ni = min(4, max(0, (npad - (m0 + wm)) / 8)), nj = min(4, max(0, (npad - (n0 + wn)) / 8));
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }

  auto load_stage = [&](int st, int kk) {
    const double* Ag = Lb + (size_t)task.src * bs + kk * 16;
    const double* Bg = invL + (size_t)task.kframe * bs + kk * 16;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int cidx = tid + q * 128;
      const int row = cidx >> 3, kc = (cidx & 7) * 2;
      const bool va = (m0 + row) < npad, vb = (n0 + row) < npad;
      cp_async16(&As[st][row * kGemmLd + kc], Ag + (size_t)(va ? m0 + row : 0) * npad + kc, va);
      cp_async16(&Bs[st][row * kGemmLd + kc], Bg + (size_t)(vb ? n0 + row : 0) * npad + kc, vb);
    }
    cp_async_commit();
  };

  load_stage(0, 0);
  for (int kk = 0; kk < kchunks; ++kk) {
    const int st = kk & 1;
    if (kk + 1 < kchunks) { load_stage(st ^ 1, kk + 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    const double* as = As[st]; const double* bsm = Bs[st];
    // warp-uniform dispatch on the number of in-range 8-wide mma tiles; interior tiles, the hot path, are tested first
    if (ni == 4 && nj == 4) gemm_stage<4, 4>(as, bsm, acc, wm, wn, g, t);
    else if (ni == 4 && nj == 2) gemm_stage<4, 2>(as, bsm, acc, wm, wn, g, t);
    else if (ni == 2 && nj == 4) gemm_stage<2, 4>(as, bsm, acc, wm, wn, g, t);
    else if (ni == 2 && nj == 2) gemm_stage<2, 2>(as, bsm, acc, wm, wn, g, t);
    __syncthreads();
  }
  double* C = T + (size_t)task.dst * bs;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = m0 + wm + i * 8 + g;
    if (row >= npad) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = n0 + wn + j * 8 + 2 * t;
      if (col >= npad) continue;
      *reinterpret_cast<double2*>(C + (size_t)row * npad + col) = make_double2(acc[i][j][0], acc[i][j][1]);
    }
  }
}

// k_potrf_trail: rank-16 trailing update of the large-block Cholesky (see k_potrf_panel).  grid = (lower 64x64 tile pairs of
// the trailing matrix, frames); 4 warps of 32x32, one 16-deep DMMA stage; entries above the diagonal are not touched.
__global__ void __launch_bounds__(128, 4) k_potrf_trail(double* __restrict__ Lb, const int* __restrict__ frames, int npad, int jb) {
  __shared__ __align__(16) double Ps[2][64 * kGemmLd];
  const int frame = frames[blockIdx.y];
  double* A = Lb + (size_t)frame * npad * npad;
  const int j0 = jb * 16, j1 = j0 + 16;
  const int2 tij = tri_index(blockIdx.x);
  const int m0 = j1 + tij.x * 64, n0 = j1 + tij.y * 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  for (int e = tid; e < 64 * 8; e += 128) {     // 64 rows x 8 double2
    const int row = e >> 3, kc = (e & 7) * 2;
    const bool va = (m0 + row) < npad, vb = (n0 + row) < npad;
    cp_async16(&Ps[0][row * kGemmLd + kc], A + (size_t)(va ? m0 + row : 0) * npad + j0 + kc, va);
    cp_async16(&Ps[1][row * kGemmLd + kc], A + (size_t)(vb ? n0 + row : 0) * npad + j0 + kc, vb);
  }
  cp_async_commit(); cp_async_wait<0>();
  __syncthreads();
  const int ni = min(4, max(0, (npad - (m0 + wm)) / 8)), nj = min(4, max(0, (npad - (n0 + wn)) / 8));
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }
  if (ni == 4 && nj == 4) gemm_stage<4, 4>(Ps[0], Ps[1], acc, wm, wn, g, t);
  else if (ni == 4 && nj == 2) gemm_stage<4, 2>(Ps[0], Ps[1], acc, wm, wn, g, t);
  else if (ni == 2 && nj == 4) gemm_stage<2, 4>(Ps[0], Ps[1], acc, wm, wn, g, t);
  else if (ni == 2 && nj == 2) gemm_stage<2, 2>(Ps[0], Ps[1], acc, wm, wn, g, t);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = m0 + wm + i * 8 + g;
    if (i >= ni) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = n0 + wn + j * 8 + 2 * t;
      if (j >= nj || col > row) continue;             // strictly-upper entries are never read
      double* ptr = A + (size_t)row * npad + col;
      if (col + 1 <= row) { double2 o = *reinterpret_cast<double2*>(ptr); o.x -= acc[i][j][0]; o.y -= acc[i][j][1]; *reinterpret_cast<double2*>(ptr) = o; }
      else ptr[0] -= acc[i][j][0];
    }
  }
}

// ---------------------------------------------------------------------------
// k_trsm_ll: X_rk = A_rk * L_kk^{-T} by a left-looking tile recurrence on the fp64 tensor cores, needing only the 16x16
// diagonal-tile inverses of k_potrf (no explicit inverse of L_kk):
//     X[:, jt] = (A[:, jt] - sum_{pt<jt} X[:, pt] L[jt, pt]^T) * Di_jt^T          jt = 0 .. npad/16 - 1
// One CTA = one kTrsmStrip-row strip of one block: 4 warps x kTrsmRW rows; the strip of X lives in shared memory
// (kTrsmStrip x (npad+4) doubles), the L row panel of step jt is staged with cp.async one step ahead.
// ---------------------------------------------------------------------------
// strip = 4 warps x RW rows.  RW = 8 (32-row strips, 108 KB -> two CTAs per SM, twice the CTAs): every warp issues one DMMA per
// 16 clk at best, so its 13-step chain costs (rows/8) x 728 DMMA x 16 clk -- halving the rows per warp halves the latency of a
// launch that does not fill the machine (the dense tail), and two co-resident CTAs hide each other's staging waits elsewhere.
constexpr int kTrsmRW = 8;
constexpr int kTrsmStrip = 4 * kTrsmRW;
// The L row panels are prefetched AHEAD steps ahead through a ring.  AHEAD = 2 (108 KB at npad 208, two CTAs per SM) for launches that
// fill the machine; AHEAD = 4 (169 KB, one CTA per SM) for the narrow levels, where a launch is a single wave and every step of the
// chain otherwise waits for its panel to come back from L2 (measured: all launches at AHEAD = 4 made the wide levels slower,
// trsm 2.03 -> 2.72 ms per factorisation, because occupancy halves where throughput counts).
__host__ __device__ inline size_t trsm_ll_smem_bytes(int npad, int ahead) { return ((size_t)kTrsmStrip * (npad + 4) + ahead * 16 * (size_t)(npad + 4) + ahead * 16 * 20) * sizeof(double); }

// kStreamed: launched as a programmatic dependent of the k_potrf_smem of the same level, so it runs while the Cholesky of its column
// frame is still going on.  Step jt reads only row panel jt of L_kk and Di_jt, which k_potrf_smem publishes in progress[kframe] >= jt + 1;
// a panel is staged once it is published, up to kTrsmAhead steps ahead.  The arithmetic and its order are those of the unstreamed kernel.
template <int kTrsmAhead, bool kStreamed = false>
__global__ void __launch_bounds__(128) k_trsm_ll(double* __restrict__ T, const double* __restrict__ Lb, const double* __restrict__ invT,
                                                  const TrsmTask* __restrict__ tasks, int npad, const int* progress) {
  static_assert(!kStreamed || kTrsmAhead <= 4, "cp_async_wait_upto3 leaves at most three groups in flight");
  extern __shared__ __align__(16) double smx[];
  __shared__ int s_ready;                        // (kStreamed) the progress thread 0 read last
  const int ld = npad + 4;                       // ld = 4 (mod 16): conflict-free DMMA fragment loads
  double* Xs = smx;                              // [kTrsmStrip][ld]
  double* Ls = smx + (size_t)kTrsmStrip * ld;    // [kTrsmAhead][16][ld]   L[jt*16 .. +15][0 .. jt*16)
  double* Ds = Ls + (size_t)kTrsmAhead * 16 * ld;   // [kTrsmAhead][16][20]   Di_jt
  const TrsmTask task = tasks[blockIdx.y];
  const int m0 = blockIdx.x * kTrsmStrip;
  const size_t bs = (size_t)npad * npad;
  const double* A = Lb + (size_t)task.src * bs;
  const double* Lk = Lb + (size_t)task.kframe * bs;
  const double* iT = invT + (size_t)task.kframe * npad * 16;
  double* X = T + (size_t)task.dst * bs;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int nt = npad / 16;
  const int rows = min(kTrsmStrip, npad - m0);
  // load the A strip (rows beyond the block are zero-filled)
  // (eight threads per row, 128 contiguous bytes; no index division -- npad is a run-time value and the divisions of the flat-index
  // form showed up at the top of the stall samples of this latency-bound kernel)
  for (int r = tid >> 3; r < kTrsmStrip; r += 16) {
    const bool v = r < rows;
    const double* src = A + (size_t)(v ? m0 + r : 0) * npad;
    for (int c = (tid & 7) * 2; c < npad; c += 16) cp_async16(&Xs[(size_t)r * ld + c], src + c, v);
  }
  auto stage = [&](int jt) {   // L row panel (columns [0, jt*16)) and Di of step jt into ring slot jt % kTrsmAhead; always one commit group (may be empty)
    if (jt < nt) {
      double* ls = Ls + (size_t)(jt % kTrsmAhead) * 16 * ld; double* dsm = Ds + (jt % kTrsmAhead) * 320;
      const int kw = jt * 16;
      { const int r = tid >> 3; const double* src = Lk + (size_t)(jt * 16 + r) * npad; for (int c = (tid & 7) * 2; c < kw; c += 16) cp_async16(&ls[(size_t)r * ld + c], src + c, true); }
      { const int r = tid >> 3, c = (tid & 7) * 2; cp_async16(&dsm[r * 20 + c], iT + (size_t)jt * 256 + r * 16 + c, true); }
    }
    cp_async_commit();
  };
  if constexpr (kStreamed) {
    cp_async_commit();                            // the A strip was finished by earlier levels: its own group, in flight at once
  } else {
#pragma unroll
    for (int q = 0; q < kTrsmAhead; ++q) stage(q);       // group 0 also carries the A strip
  }
  constexpr int NI = kTrsmRW / 8;                 // m8 tiles per warp
  const int wr = warp * kTrsmRW;                  // this warp's rows inside the strip
  int staged = 0, ready = 0;                      // (kStreamed) panels [0, staged) are staged; [0, ready) are known to be published
  for (int jt = 0; jt < nt; ++jt) {
    if constexpr (kStreamed) {
      if (ready < min(nt, jt + kTrsmAhead)) {     // a free ring slot may take a panel not known to be published yet: read the counter
        if (tid == 0) {
          // Waits only while panel jt itself is unpublished.  This cannot deadlock: a programmatic dependent launch starts only after
          // every CTA of the k_potrf_smem before it has executed griddepcontrol.launch_dependents, so the producer of this counter is
          // resident (or done) before any consumer exists, and it never waits on a consumer.  Launched without overlap (the un-captured
          // profiling and first multi-GPU runs, or a driver that ignores the attribute), k_potrf_smem has finished and every counter is
          // final.  The counters are zeroed in the factorisation graph before level 0, so a stale count never reads as published.
          int v = ld_acquire_gpu(progress + task.kframe);
          while (v <= jt) { __nanosleep(32); v = ld_acquire_gpu(progress + task.kframe); }
          s_ready = v;
        }
        __syncthreads();                          // thread 0's acquire orders every thread's panel loads below after the publication
        ready = s_ready;
      }
      for (; staged < min(ready, jt + kTrsmAhead); ++staged) stage(staged);   // ring slot staged % kTrsmAhead was freed by step staged - kTrsmAhead
      cp_async_wait_upto3(staged - 1 - jt);       // one group per panel after the A strip's: panel jt has landed
    } else {
      cp_async_wait<kTrsmAhead - 1>();            // groups complete in order: panel jt has landed, up to kTrsmAhead - 1 later ones may be in flight
    }
    __syncthreads();
    const double* ls = Ls + (size_t)(jt % kTrsmAhead) * 16 * ld; const double* dsm = Ds + (jt % kTrsmAhead) * 320;
    double acc[NI][2][2];
#pragma unroll
    for (int i = 0; i < NI; ++i) { acc[i][0][0] = acc[i][0][1] = acc[i][1][0] = acc[i][1][1] = 0.0; }
    // K loop over the jt finished column tiles, 16 columns (four DMMA k-steps) at a time; the fragments of tile kt + 1 are loaded
    // before the eight DMMAs of tile kt issue (a one-k-step loop exposed the shared-memory latency on every step: this kernel is a
    // 13-step latency chain on the narrow levels)
    {
      double af[2][4][NI], bf[2][4][2];
      auto frag = [&](int kt, int buf) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
#pragma unroll
          for (int i = 0; i < NI; ++i) af[buf][q][i] = Xs[(size_t)(wr + i * 8 + g) * ld + kt * 16 + q * 4 + t];
#pragma unroll
          for (int j = 0; j < 2; ++j) bf[buf][q][j] = ls[(size_t)(j * 8 + g) * ld + kt * 16 + q * 4 + t];
        }
      };
      if (jt > 0) frag(0, 0);
      for (int kt = 0; kt < jt; kt += 2) {
        if (kt + 1 < jt) frag(kt + 1, 1);
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int i = 0; i < NI; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) dmma_8x8x4(acc[i][j][0], acc[i][j][1], af[0][q][i], bf[0][q][j]);
        if (kt + 1 < jt) {
          if (kt + 2 < jt) frag(kt + 2, 0);
#pragma unroll
          for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int i = 0; i < NI; ++i)
#pragma unroll
              for (int j = 0; j < 2; ++j) dmma_8x8x4(acc[i][j][0], acc[i][j][1], af[1][q][i], bf[1][q][j]);
        }
      }
    }
    // Tt = A[:, jt] - acc, written back in place (each lane owns its C-fragment positions), then X[:, jt] = Tt * Di^T
#pragma unroll
    for (int i = 0; i < NI; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        double2* ptr = reinterpret_cast<double2*>(&Xs[(size_t)(wr + i * 8 + g) * ld + jt * 16 + j * 8 + 2 * t]);
        double2 v = *ptr; v.x -= acc[i][j][0]; v.y -= acc[i][j][1]; *ptr = v;
      }
    __syncwarp();
    double out[NI][2][2];
#pragma unroll
    for (int i = 0; i < NI; ++i) { out[i][0][0] = out[i][0][1] = out[i][1][0] = out[i][1][1] = 0.0; }
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      double af[NI], bf[2];
#pragma unroll
      for (int i = 0; i < NI; ++i) af[i] = Xs[(size_t)(wr + i * 8 + g) * ld + jt * 16 + k4 * 4 + t];
#pragma unroll
      for (int j = 0; j < 2; ++j) bf[j] = dsm[(j * 8 + g) * 20 + k4 * 4 + t];
#pragma unroll
      for (int i = 0; i < NI; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) dmma_8x8x4(out[i][j][0], out[i][j][1], af[i], bf[j]);
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < NI; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int r = wr + i * 8 + g, cidx = jt * 16 + j * 8 + 2 * t;
        const double2 v = make_double2(out[i][j][0], out[i][j][1]);
        *reinterpret_cast<double2*>(&Xs[(size_t)r * ld + cidx]) = v;
        if (r < rows) *reinterpret_cast<double2*>(&X[(size_t)(m0 + r) * npad + cidx]) = v;
      }
    __syncthreads();   // every warp is done with ring slot jt % kTrsmAhead before it is refilled
    if constexpr (!kStreamed) stage(jt + kTrsmAhead);
  }
  // k_potrf_smem has published its last panel, so it is (about) done: this wait costs nothing, and it makes the completion of this
  // kernel imply the completion of k_potrf_smem for whatever follows it with an ordinary dependency
  if constexpr (kStreamed) griddep_wait();
}


// ---------------------------------------------------------------------------
// Triangular solves as GEMVs with inv(L_kk); vectors have npad stride per frame.
// ---------------------------------------------------------------------------
// y_k = inv(L_kk) rhs_k   (grid: (ceil(npad/8), frames in level), 256 threads = 8 warps, one row per warp).  k_fwd_diag and
// k_bwd_diag do nothing when `stop` (nullable) points to a non-zero flag: the stop flag of the CG solve (rcvd_cg.cuh) they precondition.
__global__ void __launch_bounds__(256) k_fwd_diag(const double* __restrict__ invL, const double* __restrict__ rhs, double* __restrict__ y,
                                                   const int* __restrict__ frames, int npad, const int* __restrict__ stop) {
  if (stop && *stop) return;
  const int frame = frames[blockIdx.y];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= npad) return;
  const double* M = invL + (size_t)frame * npad * npad + (size_t)row * npad;
  const double* b = rhs + (size_t)frame * npad;
  double s = 0.0;
  for (int q = lane; q <= row; q += 32) s += M[q] * b[q];
  s = warp_sum(s);
  if (lane == 0) y[(size_t)frame * npad + row] = s;
}
struct SolveTask { int blk; int r; int k; };   // off-diagonal factor block index (into T), row frame, column frame
// rhs_r -= T_rk y_k      (grid: (ceil(npad/8), tasks in level))
__global__ void __launch_bounds__(256) k_fwd_update(const double* __restrict__ T, const double* __restrict__ y, double* __restrict__ rhs,
                                                     const SolveTask* __restrict__ tasks, int npad) {
  const SolveTask tk = tasks[blockIdx.y];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= npad) return;
  const double* M = T + (size_t)tk.blk * npad * npad + (size_t)row * npad;
  const double* v = y + (size_t)tk.k * npad;
  double s = 0.0;
  for (int q = lane; q < npad; q += 32) s += M[q] * v[q];
  s = warp_sum(s);
  if (lane == 0) red_add(rhs + (size_t)tk.r * npad + row, -s);
}
// y_k -= T_rk^T x_r for every factor block (r,k) of the level.
// grid: (ceil(npad/32), tasks in level); 256 threads = 32 columns x 8 row groups, coalesced row reads,
// smem reduction over the row groups, one RED per column.
__global__ void __launch_bounds__(256) k_bwd_update(const double* __restrict__ T, const double* __restrict__ x, double* __restrict__ y,
                                                     const SolveTask* __restrict__ tasks, int npad) {
  __shared__ double red[8][33];
  const SolveTask tk = tasks[blockIdx.y];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + cl;
  double acc = 0.0;
  if (j < npad) {
    const double* M = T + (size_t)tk.blk * npad * npad + j;
    const double* xr = x + (size_t)tk.r * npad;
    for (int i = rg; i < npad; i += 8) acc += M[(size_t)i * npad] * xr[i];
  }
  red[rg][cl] = acc;
  __syncthreads();
  if (rg == 0 && j < npad) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) s += red[q][cl];
    if (s != 0.0) red_add(y + (size_t)tk.k * npad + j, -s);
  }
}
// x_k = inv(L_kk)^T y_k    (grid: (ceil(npad/32), frames in level)); same thread layout
__global__ void __launch_bounds__(256) k_bwd_diag(const double* __restrict__ invL, const double* __restrict__ y, double* __restrict__ x,
                                                   const int* __restrict__ frames, int npad, const int* __restrict__ stop) {
  if (stop && *stop) return;
  __shared__ double red[8][33];
  const int frame = frames[blockIdx.y];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + cl;
  double acc = 0.0;
  if (j < npad) {
    const double* M = invL + (size_t)frame * npad * npad + j;
    const double* v = y + (size_t)frame * npad;
    const int i0 = j - (j % 8) + rg;            // first row >= j in this row group (rows < j are zero anyway)
    for (int i = (i0 < j ? i0 + 8 : i0); i < npad; i += 8) acc += M[(size_t)i * npad] * v[i];
  }
  red[rg][cl] = acc;
  __syncthreads();
  if (rg == 0 && j < npad) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) s += red[q][cl];
    x[(size_t)frame * npad + j] = s;
  }
}

// ---------------------------------------------------------------------------
// The forward + backward substitution of the narrow levels as ONE persistent dataflow kernel.  The level-scheduled version above is
// 4 launches per level (172 at config 2), each a single short wave: 1.35 ms of launch latency for ~0.3 ms of memory traffic.  Here the
// same GEMVs are tasks of a list in topological order (level-major; forward levels ascending, then backward levels descending), cut
// into kSubChunk-row (forward) / -column (backward) chunks.  A CTA takes the next task with an atomic ticket, waits on the counters its
// inputs signal, computes, signals.  Dependencies always point to EARLIER tasks of the list, which running CTAs have taken, so the
// wait loops cannot deadlock whatever the number of resident CTAs is; and the waits are per frame, not per level.
//   FDIAG(k):   y_k      = inv(L_kk) rhs_k            waits until every FUPD(k, .) chunk has landed     signals fdone[k]
//   FUPD(r,k):  rhs_r   -= T_rk y_k                    waits for fdone[k] == chunks                      signals fin[r]
//   BUPD(r,k):  y_k     -= T_rk^T x_r                  waits for bdone[r] == chunks                      signals bin[k]
//   BDIAG(k):   x_k      = inv(L_kk)^T y_k             waits for fdone[k] and every BUPD(., k) chunk     signals bdone[k]
// Vectors written by other SMs are read with ld.global.cg (L2) after the acquire; matrices are immutable during the kernel.
// ---------------------------------------------------------------------------
constexpr int kSubChunk = 64;
constexpr int kSubThreads = 256;
struct SubTask { int type; int blk; int r; int k; int chunk; };   // type 0 FDIAG, 1 FUPD, 2 BUPD, 3 BDIAG
struct SubCounters { int* ticket; int* fin; int* fdone; int* bin; int* bdone; const int* fin_need; const int* bin_need; };

__device__ __forceinline__ void sub_wait(const int* c, int need) { while (ld_acquire_gpu(c) < need) __nanosleep(20); }

__device__ __forceinline__ double2 ldcg2(const double* p) { return __ldcg(reinterpret_cast<const double2*>(p)); }

__global__ void __launch_bounds__(kSubThreads) k_substitution(const double* __restrict__ invL, const double* __restrict__ T, double* rhs, double* y, double* x,
                                                              const SubTask* __restrict__ tasks, int ntasks, SubCounters cn, int npad) {
  extern __shared__ __align__(16) double red[];   // [8][kSubChunk + 2] column partials
  __shared__ int s_task;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nchunks = (npad + kSubChunk - 1) / kSubChunk;
  const size_t bs = (size_t)npad * npad;
  for (;;) {
    if (tid == 0) s_task = atomicAdd(cn.ticket, 1);
    __syncthreads();
    const int ti = s_task;
    if (ti >= ntasks) break;
    const SubTask tk = tasks[ti];
    const int c0 = tk.chunk * kSubChunk, c1 = min(npad, c0 + kSubChunk);
    // input vector (written by other SMs: read through L2 after the acquire) and the immutable matrix block of the task
    const double* vin = tk.type == 0 ? rhs + (size_t)tk.k * npad : (tk.type == 2 ? x + (size_t)tk.r * npad : y + (size_t)tk.k * npad);
    const double* M = (tk.type == 0 || tk.type == 3) ? invL + (size_t)tk.k * bs : T + (size_t)tk.blk * bs;
    auto dep_wait = [&]() {
      if (tid == 0) {
        if (tk.type == 0) sub_wait(cn.fin + tk.k, cn.fin_need[tk.k]);
        else if (tk.type == 1) sub_wait(cn.fdone + tk.k, nchunks);
        else if (tk.type == 2) sub_wait(cn.bdone + tk.r, nchunks);
        else { sub_wait(cn.fdone + tk.k, nchunks); sub_wait(cn.bin + tk.k, cn.bin_need[tk.k]); }
      }
      __syncthreads();
    };
    // A task is one short latency-bound GEMV on the dependency chain.  Every load of a thread is issued before the first is used (a
    // row-at-a-time loop serialised eight memory latencies per warp), and the matrix part -- up to 256 columns / rows, all of it at
    // npad <= 256 -- is in flight BEFORE the wait: CTAs take tasks ahead of their inputs, so the matrix latency hides behind the wait.
    if (tk.type <= 1) {
      // rows c0 .. c1 of M times the vector: eight rows per warp, 16-byte loads
      constexpr int RW = kSubChunk / (kSubThreads / 32);
      const int r0 = c0 + warp * RW;
      double acc[RW];
#pragma unroll
      for (int i = 0; i < RW; ++i) acc[i] = 0.0;
      for (int qb = 0; qb < npad; qb += 256) {        // 4 x 64 columns per pass: 32 independent 16-byte loads per lane
        double2 m[4][RW];
#pragma unroll
        for (int qi = 0; qi < 4; ++qi) {
          const int q = qb + qi * 64 + 2 * lane;
#pragma unroll
          for (int i = 0; i < RW; ++i) {
            const int row = r0 + i;
            const int len = tk.type == 0 ? row + 1 : npad;     // inv(L) is lower triangular
            m[qi][i] = (row < c1 && q < len) ? *reinterpret_cast<const double2*>(M + (size_t)row * npad + q) : make_double2(0.0, 0.0);
            if (q + 1 >= len) m[qi][i].y = 0.0;
          }
        }
        if (qb == 0) dep_wait();
        double2 v[4];
#pragma unroll
        for (int qi = 0; qi < 4; ++qi) { const int q = qb + qi * 64 + 2 * lane; v[qi] = q < npad ? ldcg2(vin + q) : make_double2(0.0, 0.0); }
#pragma unroll
        for (int qi = 0; qi < 4; ++qi)
#pragma unroll
          for (int i = 0; i < RW; ++i) acc[i] += m[qi][i].x * v[qi].x + m[qi][i].y * v[qi].y;
      }
#pragma unroll
      for (int i = 0; i < RW; ++i) {
        const double sum = warp_sum(acc[i]);
        const int row = r0 + i;
        if (lane == 0 && row < c1) { if (tk.type == 0) y[(size_t)tk.k * npad + row] = sum; else red_add(rhs + (size_t)tk.r * npad + row, -sum); }
      }
    } else {
      // columns c0 .. c1 of M^T times the vector: 32 column pairs x 8 row groups, 512 contiguous bytes per row
      const int cl = tid & 31, rg = tid >> 5, j = c0 + 2 * cl;
      double ax = 0.0, ay = 0.0;
      // inv(L)^T: only rows i >= j contribute; the first such row of this row group
      const int ifirst = tk.type == 3 ? j + ((rg - j) & 7) : rg;
      for (int ib = ifirst; ib < npad || ib == ifirst; ib += 256) {   // 32 rows of this row group per pass, loads first
        double2 m[32];
#pragma unroll
        for (int u = 0; u < 32; ++u) { const int i = ib + 8 * u; m[u] = (i < npad && j < c1) ? *reinterpret_cast<const double2*>(M + (size_t)i * npad + j) : make_double2(0.0, 0.0); }
        if (ib == ifirst) dep_wait();
        double vi[32];
#pragma unroll
        for (int u = 0; u < 32; ++u) { const int i = ib + 8 * u; vi[u] = i < npad ? __ldcg(vin + i) : 0.0; }
#pragma unroll
        for (int u = 0; u < 32; ++u) { const int i = ib + 8 * u; ax += m[u].x * vi[u]; if (tk.type != 3 || i > j) ay += m[u].y * vi[u]; }
      }
      red[rg * (kSubChunk + 2) + 2 * cl] = ax; red[rg * (kSubChunk + 2) + 2 * cl + 1] = ay;
      __syncthreads();
      if (tid < kSubChunk && c0 + tid < c1) {
        double sum = 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) sum += red[q * (kSubChunk + 2) + tid];
        if (tk.type == 3) x[(size_t)tk.k * npad + c0 + tid] = sum; else red_add(y + (size_t)tk.k * npad + c0 + tid, -sum);
      }
    }
    // the barrier orders every thread's stores / REDs before thread 0's release (cumulativity), like cutlass::Semaphore::release
    __syncthreads();
    if (tid == 0) red_release_add(tk.type == 0 ? cn.fdone + tk.k : (tk.type == 1 ? cn.fin + tk.r : (tk.type == 2 ? cn.bin + tk.k : cn.bdone + tk.k)), 1);
  }
}

// The factorisation's kernel variants at block size npad and each kernel's dynamic shared memory: k_potrf_smem up to npad 224 (else
// k_potrf_panel + k_potrf_trail), k_trsm_ll up to 416 (else k_gemm_nt with the inverse from k_trinv), its AHEAD = 4 shape up to 272.
struct FactorKernels {
  bool potrf_smem, trsm_ll, trsm_ll4;
  size_t potrf_bytes, trsm_ll2_bytes, trsm_ll4_bytes, trinv_bytes, substitution_bytes;
  int trsm2_ctas_per_sm;   // resident k_trsm_ll<2> CTAs per SM: set by allocate_storage (rcvd_api.cu) from an occupancy query
};
inline FactorKernels factor_kernels(int npad) {
  const size_t potrf = potrf_smem_bytes(npad), ll2 = trsm_ll_smem_bytes(npad, 2), ll4 = trsm_ll_smem_bytes(npad, 4);
  const size_t trinv = (size_t)(npad * 16 + 16 * (npad + 1)) * sizeof(double);   // tile column of the inverse + staged L row panel
  const size_t sub = (size_t)8 * (kSubChunk + 2) * sizeof(double);                 // k_substitution: [8][kSubChunk + 2] column partials
  return {potrf <= kMaxDynSmem, ll2 <= kMaxDynSmem, ll4 <= kMaxDynSmem, potrf, ll2, ll4, trinv, sub, 0};
}

// ---------------------------------------------------------------------------
// Factor load: L <- S H S + D2 (lower triangle of diagonal blocks, pad diagonal = 1) for the blocks blist[0, nload), zeros in the
// padding of the fill blocks blist[nload, nload + nfill) (rows neff..npad, and columns neff..npad of rows < neff).  The interior of a
// fill block is written by its first update pass (kUpdFirstFill), which covers rows and columns < neff; the padding still holds the
// previous factorisation's values.
// grid: (ceil(npad*npad/256), nload + enough rows of CTAs for the fill padding)
// ---------------------------------------------------------------------------
struct HBlock { int lblk; int r; int c; };   // H list: lblk = destination block in L.  L list: lblk = source block in H (or -1: fill)
__global__ void __launch_bounds__(256) k_load_factor(const double* __restrict__ H, double* __restrict__ Lb, const HBlock* __restrict__ lb,
                                                      const double* __restrict__ S, const double* __restrict__ D2, int npad, int nf, int neff,
                                                      const int* __restrict__ blist, int nload, int nfill) {
  const size_t bs = (size_t)npad * npad;
  if ((int)blockIdx.y >= nload) {
    const int ph = npad - neff, per = ph * (npad + neff);     // padding elements per fill block: ph full rows, then ph columns of neff rows
    const long q = ((long)(blockIdx.y - nload) * gridDim.x + blockIdx.x) * 256 + threadIdx.x;
    if (per == 0 || q >= (long)nfill * per) return;
    const int f = (int)(q / per), e = (int)(q % per), r = e - ph * npad;
    const int i = r < 0 ? neff + e / npad : r / ph, j = r < 0 ? e % npad : neff + r % ph;
    Lb[(size_t)blist[nload + f] * bs + (size_t)i * npad + j] = 0.0;
    return;
  }
  const int bid = blist[blockIdx.y];
  const HBlock b = lb[bid];
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= npad * npad) return;
  const int i = e / npad, j = e % npad;
  double v = 0.0;
  if (b.r == b.c) {
    if (j > i) v = 0.0;
    else if (i >= nf) v = (i == j) ? 1.0 : 0.0;
    else {
      v = H[(size_t)b.lblk * bs + e] * S[(size_t)b.r * npad + i] * S[(size_t)b.c * npad + j];
      if (i == j) v += D2[(size_t)b.r * npad + i];
    }
  } else if (i < nf && j < nf) {
    v = H[(size_t)b.lblk * bs + e] * S[(size_t)b.r * npad + i] * S[(size_t)b.c * npad + j];
  }
  Lb[(size_t)bid * bs + e] = v;
}
__host__ __device__ inline int load_factor_pad_rows(int npad, int neff, int nfill) {   // grid rows of k_load_factor for the fill padding
  const long per = (long)(npad - neff) * (npad + neff), row = (long)((npad * npad + 255) / 256) * 256;
  return (int)(((long)nfill * per + row - 1) / row);
}

// out += H v over the original block structure (symmetric; diagonal blocks hold the lower triangle).
// grid: (ceil(npad/8), H blocks), one warp per row i; also accumulates the transposed part.
__global__ void __launch_bounds__(256) k_spmv_sym(const double* __restrict__ H, const HBlock* __restrict__ hb, const double* __restrict__ v,
                                                   double* __restrict__ out, int npad, const int* __restrict__ blist) {
  const int bid = blist ? blist[blockIdx.y] : blockIdx.y;   // H block id (blist: the blocks this rank owns)
  const HBlock b = hb[bid];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= npad) return;
  const double* M = H + (size_t)bid * npad * npad + (size_t)row * npad;
  const double* vc = v + (size_t)b.c * npad;
  const double vr = v[(size_t)b.r * npad + row];
  double s = 0.0;
  if (b.r == b.c) {
    for (int q = lane; q <= row; q += 32) {
      const double m = M[q];
      s += m * vc[q];
      if (q < row && m != 0.0) red_add(out + (size_t)b.c * npad + q, m * vr);
    }
  } else {
    for (int q = lane; q < npad; q += 32) {
      const double m = M[q];
      s += m * vc[q];
      if (m != 0.0 && vr != 0.0) red_add(out + (size_t)b.c * npad + q, m * vr);
    }
  }
  s = warp_sum(s);
  if (lane == 0 && s != 0.0) red_add(out + (size_t)b.r * npad + row, s);
}

}  // namespace rcvd
