// rcvd_selinv.cuh -- marginal covariance blocks by selected inversion of the block-Cholesky factor (rcvd_covariance, include/rcvd.h).
//
// With P A P^T = L L^T (rcvd_linalg.cuh; L_kk the diagonal blocks, X_rk = L_rk the off-diagonal factor blocks in T, inv(L_kk) in
// invL) the blocks Z = A^-1 on the filled pattern follow from the block Takahashi recurrence, level by level in REVERSE elimination
// order; the frames k of one level are independent.  S_k = the later frames r with a factor block (r, k) (a clique after fill):
//   1. Y_rk = sum_{j in S_k} Z_rj X_jk                    r in S_k        k_selinv_product  (Z_rj: block (r, j), (j, r)^T or Z_rr)
//   2. Z_rk = -Y_rk inv(L_kk)                             in place        k_selinv_trmm
//   3. W_kk = inv(L_kk) - sum_{j in S_k} X_jk^T Z_jk                      k_selinv_product
//      Z_kk = inv(L_kk)^T W_kk                            in place        k_selinv_trmm (the strip transposed)
// Z overwrites the factor blocks in Lb: the off-diagonal A_rk are dead after the TRSM, L_kk after k_trinv.  T and invL are only read.
// Pure host code (the task lists) and kernels; rcvd_api.cu launches them.
#pragma once
#include <algorithm>
#include <map>
#include <vector>

#include "rcvd_plan.h"

namespace rcvd {

// One 64 x 64 output tile of a block product:  Lb[dst](m0.., n0..) = base + sign * sum_{p in [first, first + count)} op(A_p) op(B_p),
// base = invL[base] (or 0 with base < 0).  Operand flags of each product: which buffer it lives in and whether it is transposed.
struct SelTile { int dst, base, first, count, m0, n0; };
enum { kSelATrans = 1, kSelAInT = 2, kSelBTrans = 4, kSelBInT = 8 };
struct SelOp { int a, b, flags; };
struct SelTrmm { int blk, frame; };          // the block of Lb multiplied in place by inv(L_frame) (right) or its transpose (left)
struct SelGather { int src, trans, r, c; };   // output block from L block src (rows of frame r, columns of frame c), transposed if trans

constexpr int kSelTile = 64, kSelK = 16, kSelLd = kSelK + 4, kSelThreads = 128;
constexpr int kSelStrip = 16;   // rows of a k_selinv_trmm strip

// The launches of one level of the sweep: step 1 tiles, step 2 trmm tasks, step 3 tiles, step 3 trmm tasks ([off, off + n) each).
struct SelLevel { int off[4], n[4]; };
struct SelPlan {
  std::vector<SelTile> tiles; std::vector<SelOp> ops; std::vector<SelTrmm> trmm;
  std::vector<SelLevel> levels;              // in launch order: the plan's levels from the last to the first
  std::vector<int> row_off, row_blk;          // per frame: the T indices of its factor row (the blocks (k, c), c eliminated earlier)
  double flops = 0.0;                         // algorithmic flops of the selected inversion at nf unknowns per frame
  long products = 0;                          // block products of steps 1 and 3
};

// The task lists of the sweep over the plan's filled pattern (single GPU: every frame of every level).
inline void make_sel_plan(SelPlan& S, const FactorPlan& P, int N, int npad, int nf) {
  S = SelPlan();
  const int nLoff = P.nLoff, nt = (npad + kSelTile - 1) / kSelTile;
  std::vector<int> pos(N);
  for (int q = 0; q < N; ++q) pos[P.elim_order[q]] = q;
  std::map<std::pair<int, int>, int> lid;    // (later frame r, earlier frame c) -> L block id
  std::vector<std::vector<int>> cs(N);       // S_k, in elimination order
  for (int t = 0; t < nLoff; ++t) { const auto& b = P.lblocks[N + t]; lid[{b.r, b.c}] = N + t; cs[b.c].push_back(b.r); }
  for (auto& v : cs) std::sort(v.begin(), v.end(), [&](int a, int b) { return pos[a] < pos[b]; });
  S.row_off.assign(N + 1, 0);
  for (int t = 0; t < nLoff; ++t) S.row_off[P.lblocks[N + t].r + 1]++;
  for (int f = 0; f < N; ++f) S.row_off[f + 1] += S.row_off[f];
  S.row_blk.assign(nLoff, 0);
  { std::vector<int> fill(S.row_off.begin(), S.row_off.end() - 1); for (int t = 0; t < nLoff; ++t) S.row_blk[fill[P.lblocks[N + t].r]++] = t; }
  auto tiles_of = [&](int dst, int base, int first, int count) {
    for (int ti = 0; ti < nt; ++ti) for (int tj = 0; tj < nt; ++tj) S.tiles.push_back({dst, base, first, count, ti * kSelTile, tj * kSelTile});
  };
  const double n3 = (double)nf * nf * nf;
  for (int l = (int)P.levels.size() - 1; l >= 0; --l) {
    const auto& lv = P.levels[l];
    SelLevel sl;
    for (int step = 0; step < 4; ++step) {
      sl.off[step] = (step & 1) ? (int)S.trmm.size() : (int)S.tiles.size();
      for (int i = 0; i < lv.nframes; ++i) {
        const int k = P.lvl_frames[lv.frame_off + i];
        const std::vector<int>& sk = cs[k];
        if (step == 0) {
          for (int r : sk) {
            const int first = (int)S.ops.size();
            for (int j : sk) {
              SelOp op;
              if (r == j) { op.a = r; op.flags = 0; }
              else if (pos[r] > pos[j]) { op.a = lid[{r, j}]; op.flags = 0; }
              else { op.a = lid[{j, r}]; op.flags = kSelATrans; }
              op.b = lid[{j, k}] - N; op.flags |= kSelBInT;
              S.ops.push_back(op);
            }
            tiles_of(lid[{r, k}], -1, first, (int)sk.size());
          }
          S.products += (long)sk.size() * sk.size(); S.flops += 2.0 * n3 * sk.size() * sk.size();
        } else if (step == 1) {
          for (int r : sk) S.trmm.push_back({lid[{r, k}], k});
          S.flops += n3 * sk.size();
        } else if (step == 2) {
          const int first = (int)S.ops.size();
          for (int j : sk) S.ops.push_back({lid[{j, k}] - N, lid[{j, k}], kSelATrans | kSelAInT});
          tiles_of(k, k, first, (int)sk.size());
          S.products += (long)sk.size(); S.flops += 2.0 * n3 * sk.size();
        } else {
          S.trmm.push_back({k, k});
          S.flops += n3;
        }
      }
      sl.n[step] = ((step & 1) ? (int)S.trmm.size() : (int)S.tiles.size()) - sl.off[step];
    }
    S.levels.push_back(sl);
  }
}

// ---------------------------------------------------------------------------
// k_selinv_product: one CTA per SelTile, 4 warps of 32 x 32 on the fp64 tensor cores (mma.sync m16n8k4), operands staged 16 deep
// through shared memory with a register prefetch of the next stage.  Each CTA sums its products in list order and writes its own
// tile: no atomics, a rerun is bitwise identical.  Lb is read (operands) and written (the target): a target is never an operand of
// the same launch.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kSelThreads) k_selinv_product(double* Lb, const double* __restrict__ T, const double* __restrict__ invL,
                                                                const SelTile* __restrict__ tiles, const SelOp* __restrict__ ops, int npad, double sign) {
  __shared__ __align__(16) double As[kSelTile * kSelLd];   // As[m][k]
  __shared__ __align__(16) double Bs[kSelTile * kSelLd];   // Bs[n][k]
  const SelTile tile = tiles[blockIdx.x];
  const size_t bs = (size_t)npad * npad;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const bool active = tile.m0 + wm < npad && tile.n0 + wn < npad;   // warp-uniform: a warp tile wholly in the padding issues no mma
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0;
  const int kchunks = npad / kSelK, nstages = tile.count * kchunks;
  double ra[8], rb[8];
  // stage s = (product s / kchunks, K chunk s % kchunks) into registers: A as [m][k], B as [n][k], zeros outside the block
  auto fetch = [&](int s) {
    const SelOp op = ops[tile.first + s / kchunks];
    const int k0 = (s % kchunks) * kSelK;
    const double* A = ((op.flags & kSelAInT) ? T : Lb) + (size_t)op.a * bs;
    const double* B = ((op.flags & kSelBInT) ? T : Lb) + (size_t)op.b * bs;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int e = tid + q * kSelThreads;
      if (op.flags & kSelATrans) { const int kk = e >> 6, m = e & 63; ra[q] = tile.m0 + m < npad ? A[(size_t)(k0 + kk) * npad + tile.m0 + m] : 0.0; }
      else { const int m = e >> 4, kk = e & 15; ra[q] = tile.m0 + m < npad ? A[(size_t)(tile.m0 + m) * npad + k0 + kk] : 0.0; }
      if (op.flags & kSelBTrans) { const int n = e >> 4, kk = e & 15; rb[q] = tile.n0 + n < npad ? B[(size_t)(tile.n0 + n) * npad + k0 + kk] : 0.0; }
      else { const int kk = e >> 6, n = e & 63; rb[q] = tile.n0 + n < npad ? B[(size_t)(k0 + kk) * npad + tile.n0 + n] : 0.0; }
    }
  };
  auto stash = [&](int s) {
    const int fl = ops[tile.first + s / kchunks].flags;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int e = tid + q * kSelThreads;
      if (fl & kSelATrans) As[(e & 63) * kSelLd + (e >> 6)] = ra[q]; else As[(e >> 4) * kSelLd + (e & 15)] = ra[q];
      if (fl & kSelBTrans) Bs[(e >> 4) * kSelLd + (e & 15)] = rb[q]; else Bs[(e & 63) * kSelLd + (e >> 6)] = rb[q];
    }
  };
  if (nstages > 0) fetch(0);
  for (int s = 0; s < nstages; ++s) {
    stash(s);
    __syncthreads();
    if (s + 1 < nstages) fetch(s + 1);
    if (active) {
#pragma unroll
      for (int k4 = 0; k4 < kSelK / 4; ++k4) {
        double a[2][2], b[4];
#pragma unroll
        for (int i = 0; i < 2; ++i) { a[i][0] = As[(wm + i * 16 + g) * kSelLd + k4 * 4 + t]; a[i][1] = As[(wm + i * 16 + 8 + g) * kSelLd + k4 * 4 + t]; }
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = Bs[(wn + j * 8 + g) * kSelLd + k4 * 4 + t];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) dmma_16x8x4(acc[i][j][0], acc[i][j][1], acc[i][j][2], acc[i][j][3], a[i][0], a[i][1], b[j]);
      }
    }
    __syncthreads();
  }
  double* C = Lb + (size_t)tile.dst * bs;
  const double* base = tile.base >= 0 ? invL + (size_t)tile.base * bs : nullptr;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = tile.m0 + wm + i * 16 + h * 8 + g;
      if (row >= npad) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = tile.n0 + wn + j * 8 + 2 * t;
        if (col >= npad) continue;
        double2 v = make_double2(sign * acc[i][j][2 * h], sign * acc[i][j][2 * h + 1]);
        if (base) { const double2 b0 = *reinterpret_cast<const double2*>(base + (size_t)row * npad + col); v.x += b0.x; v.y += b0.y; }
        *reinterpret_cast<double2*>(C + (size_t)row * npad + col) = v;
      }
    }
}

// ---------------------------------------------------------------------------
// k_selinv_trmm: Y <- sign * Y inv(L_kk) in place (left = 0), or W <- sign * inv(L_kk)^T W (left = 1, computed as (W^T inv(L_kk))^T).
// grid (npad / 16 strips, tasks): a CTA stages its 16-row strip of Y (16-column strip of W, transposed) in shared memory, so it reads
// all of its strip before it writes any of it, and no other CTA touches the strip.  inv(L_kk) is lower triangular (k_trinv writes
// zeros above the diagonal), so output column block c0 sums rows q >= c0 only.  Each warp owns 8-column blocks, m16n8k4 DMMA.
// ---------------------------------------------------------------------------
__host__ __device__ inline size_t sel_trmm_smem_bytes(int npad) { return (size_t)kSelStrip * (npad + 4) * sizeof(double); }
__global__ void __launch_bounds__(kSelThreads) k_selinv_trmm(double* __restrict__ Lb, const double* __restrict__ invL, const SelTrmm* __restrict__ tasks,
                                                             int npad, double sign, int left) {
  extern __shared__ __align__(16) double Ys[];   // [16][npad + 4]
  const int ld = npad + 4;
  const SelTrmm task = tasks[blockIdx.y];
  double* Y = Lb + (size_t)task.blk * npad * npad;
  const double* M = invL + (size_t)task.frame * npad * npad;
  const int s0 = blockIdx.x * kSelStrip, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  for (int e = tid; e < kSelStrip * npad; e += kSelThreads) {
    if (left) { const int q = e >> 4, i = e & 15; Ys[i * ld + q] = Y[(size_t)q * npad + s0 + i]; }
    else { const int i = e / npad, q = e % npad; Ys[i * ld + q] = Y[(size_t)(s0 + i) * npad + q]; }
  }
  __syncthreads();
  for (int c0 = warp * 8; c0 < npad; c0 += 4 * 8) {
    double c[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 4
    for (int q = c0; q < npad; q += 4)
      dmma_16x8x4(c[0], c[1], c[2], c[3], Ys[g * ld + q + t], Ys[(g + 8) * ld + q + t], __ldg(M + (size_t)(q + t) * npad + c0 + g));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = s0 + g + 8 * h, col = c0 + 2 * t;
      if (left) { Y[(size_t)col * npad + i] = sign * c[2 * h]; Y[(size_t)(col + 1) * npad + i] = sign * c[2 * h + 1]; }
      else *reinterpret_cast<double2*>(Y + (size_t)i * npad + col) = make_double2(sign * c[2 * h], sign * c[2 * h + 1]);
    }
  }
}

// ---------------------------------------------------------------------------
// k_selinv_scale: the scaling of the covariance factorisation.  S = diag(H)^-1/2 and D2 = 0 on the free parameters; S = 0 and D2 = 1
// (a decoupled unit pivot) on the zeroed ones: held (hold), padding, and -- with the masks given -- parameters no residual touches
// (active) and frames out of range (in_range).  A free parameter with a zero diagonal gets S = 0, D2 = 0: a zero pivot.
// ---------------------------------------------------------------------------
__global__ void k_selinv_scale(const double* __restrict__ H, const uint8_t* __restrict__ hold, const uint8_t* __restrict__ active,
                               const uint8_t* __restrict__ in_range, double* __restrict__ S, double* __restrict__ D2, int N, int npad, int nf) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * npad) return;
  const int f = i / npad, l = i % npad;
  const bool zeroed = l >= nf || hold[i] || (active && !active[i]) || (in_range && !in_range[f]);
  const double d = H[(size_t)f * npad * npad + (size_t)l * npad + l];
  S[i] = zeroed || !(d > 0.0) ? 0.0 : 1.0 / sqrt(d);
  D2[i] = zeroed ? 1.0 : 0.0;
}

// ---------------------------------------------------------------------------
// k_selinv_pivots: the pivot of every row of the factorisation, recomputed from the factor as
//   d_i = A_ii - sum_{factor row blocks X_kc} |X_kc(i, :)|^2 - sum_{q < i} L_kk(i, q)^2,   A = S H S + D2.
// Equal to L_kk(i, i)^2 where the factorisation succeeded; at a non-positive pivot the Cholesky kernels flag the failure and go on with
// a unit pivot, and this recomputes the value they replaced (rows after the first failure are not meaningful).
// grid (ceil(nf / 8), N), one warp per row, lanes over columns.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_selinv_pivots(const double* __restrict__ H, const double* __restrict__ Lb, const double* __restrict__ T,
                                                       const double* __restrict__ S, const double* __restrict__ D2, const int* __restrict__ row_off,
                                                       const int* __restrict__ row_blk, int npad, int nf, double* __restrict__ piv) {
  const int k = blockIdx.y, i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= nf) return;
  const size_t bs = (size_t)npad * npad;
  double s = 0.0;
  for (int b = row_off[k]; b < row_off[k + 1]; ++b) {
    const double* x = T + (size_t)row_blk[b] * bs + (size_t)i * npad;
    for (int j = lane; j < npad; j += 32) s += x[j] * x[j];
  }
  const double* l = Lb + (size_t)k * bs + (size_t)i * npad;
  for (int q = lane; q < i; q += 32) s += l[q] * l[q];
  s = warp_sum(s);
  if (lane == 0) {
    const double si = S[(size_t)k * npad + i];
    piv[(size_t)k * npad + i] = H[(size_t)k * bs + (size_t)i * npad + i] * si * si + D2[(size_t)k * npad + i] - s;
  }
}

// ---------------------------------------------------------------------------
// k_selinv_gather: output block b = S_r Z S_c restricted to the nf unknowns, in the requested orientation.  Each entry is computed in
// the stored block's orientation, so the (a, b) and (b, a) blocks are exact transposes; a diagonal block is symmetrised,
// (Z_pq + Z_qp) / 2 with p >= q.  Zeroed parameters (S = 0) give exact zeros.  grid (ceil(nf^2 / 256), blocks).
// ---------------------------------------------------------------------------
__global__ void k_selinv_gather(const double* __restrict__ Lb, const double* __restrict__ S, const SelGather* __restrict__ list, int npad, int nf,
                                double* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nf * nf) return;
  const SelGather gb = list[blockIdx.y];
  const int i = e / nf, j = e % nf;
  int ri = gb.trans ? j : i, ci = gb.trans ? i : j;
  const double* Z = Lb + (size_t)gb.src * npad * npad;
  double z;
  if (gb.r == gb.c) { const int p = max(ri, ci), q = min(ri, ci); z = 0.5 * (Z[(size_t)p * npad + q] + Z[(size_t)q * npad + p]); ri = p; ci = q; }
  else z = Z[(size_t)ri * npad + ci];
  const double sr = S[(size_t)gb.r * npad + ri], sc = S[(size_t)gb.c * npad + ci];
  out[(size_t)blockIdx.y * nf * nf + e] = (sr == 0.0 || sc == 0.0) ? 0.0 : z * sr * sc;
}

}  // namespace rcvd
