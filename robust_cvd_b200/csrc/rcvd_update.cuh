// rcvd_update.cuh -- Schur-complement updates of the block Cholesky, A_rc -= sum_k X_rk X_ck^T, as a persistent
// TMA-fed fp64 tensor-core kernel (the dominant kernel of an LM iteration at BASELINE config 2).
//
// The reference leaves this arithmetic to Ceres' SPARSE_NORMAL_CHOLESKY (lib/PoseOptimizer.cpp:956); here it is
// the supernodal update step of our own factorisation (rcvd_linalg.cuh).  wgmma has no fp64 kind, so the MMA is
// mma.sync.m16n8k4.f64 (DMMA; two 8-row units of the warp tile per instruction); what is Hopper-native is the data movement:
//   * operands are fetched by the TMA (cp.async.bulk.tensor.2d, one elected producer thread) straight from the
//     row-major factor blocks into a 5-deep shared-memory ring, completion signalled on mbarriers (no cp.async
//     groups, no __syncthreads in the K loop);
//   * the TMA box is [rows][16 doubles] = 128-byte rows with the 128-byte swizzle (16-byte chunk index XOR row & 7).  A first
//     version used [rows][4 doubles] boxes (32-byte rows, conflict-free by construction): same speed as the cp.async
//     kernel k_gemm_nt, the DMMA warps starved on the full barriers -- the TMA is bound by row requests, not bytes.  With 128-byte
//     rows the fragment loads stay conflict-free by feeding the m8n8k4 fragment row g with tile row pi(g) = 2 (g & 3) + (g >> 2):
//     the 16 lanes of a half-warp then touch 16 distinct 8-byte slots of the 128-byte bank window.  The same permutation on
//     the B side permutes the accumulator columns; one shuffle per accumulator pair restores adjacent column pairs for
//     16-byte read-modify-writes of the target;
//   * once the producer has issued an item's last stage (the DMMA warps are then at most one ring of stages from its end), it
//     prefetches the target rows into L2 (cp.async.bulk.prefetch, one per row) for the epilogue's read-modify-write.  The products
//     are summed from zero and subtracted from the target once, at the end: accumulating onto the target instead rounds every DMMA
//     step at the target's magnitude, and on diagonal blocks, where the target dominates the products, the componentwise backward
//     error of the factor measured 72-83 u against 64 u.  The first pass into a fill block neither prefetches nor reads the target
//     (it has no value yet): it stores 0 - products;
//   * persistent CTAs walk a list of (target tile, source-pair list) work items, so the producer prefetches the next item's first
//     stages while the DMMA warps are in the epilogue of the previous one.  The plan orders a launch's items so that each wave reads
//     few distinct operand strips (L2 reuse) and every CTA gets the same work (rcvd_plan.h, order_update_items);
//   * a single warp issues DMMAs far below the SM's rate, so a lone 4-warp tile is latency-bound (1300 DMMAs per warp at
//     K = 200 on the narrow-level launches of the factorisation): TWO teams of four DMMA warps take alternate K stages of the same
//     tile, team 1 hands its partial accumulators to team 0 through shared memory (named barriers, no __syncthreads) and goes on
//     to the next item while team 0 does the read-modify-write of the target;
//   * tiles are 80 x 80 (5 x 5 m8n8 units for each of the 2 x 2 warps: balanced), the remainder of the block last:
//     neff = 200 -> 80 + 80 + 40, not 64 + 64 + 64 + 8.
#pragma once
#include "rcvd_linalg.cuh"
#include "rcvd_ptx.cuh"

namespace rcvd {

struct UpdItem {
  int dst;            // target L block
  int first, count;   // source pairs [first, first + count) of (T index of X_rk, T index of X_ck)
  short m0, n0;       // tile origin inside the block
  short mrows, ncols; // valid extent (multiples of 8)
  int flags;          // kUpdSymDiag | kUpdFirstFill
};
constexpr int kUpdSymDiag = 1;     // diagonal tile of a symmetric target: the strictly-upper warp tile is neither read nor written
constexpr int kUpdFirstFill = 2;   // first pass into a fill block: the target holds no value yet, the item writes it without reading it

// Two shapes of the same kernel (template TEAMS):
//   TEAMS = 1: 4 DMMA warps + producer, 5-stage ring, two CTAs per SM            -- launches with more items than the machine holds
//   TEAMS = 2: two teams of 4 DMMA warps + producer, 8-stage ring, one CTA per SM -- launches of a few items (the narrow levels of the
//              factorisation), where a lone 4-warp tile is bound by the DMMA issue rate of a single warp
constexpr int kUpdMaxTile = 80;       // rows / columns of a CTA tile (<= 5 m8n8 units per warp and dimension)
constexpr int kUpdPartial = 4 * 25 * 32 * 2;   // doubles: team 1's accumulators on their way to team 0
template <int TEAMS> struct UpdShape { static constexpr int stages = TEAMS == 2 ? 8 : 5, threads = TEAMS * 128 + 32, ctas = TEAMS == 2 ? 1 : 2; };
// CTAs of a launch of n items: the two-team shape (one CTA per item) up to one item per SM, else the one-team shape, two CTAs per SM.
// CTA b walks the items b, b + ctas, b + 2 ctas, ...: a "wave" of `ctas` consecutive items runs at about the same time.
inline int upd_ctas(int n, int num_sms) { return n <= num_sms ? n : (n < 2 * num_sms ? n : 2 * num_sms); }
__host__ __device__ inline size_t upd_smem_bytes(int rb, int teams) {
  const int stages = teams == 2 ? 8 : 5;
  return (size_t)stages * 2 * rb * 16 * sizeof(double) + (teams == 2 ? (size_t)kUpdPartial * sizeof(double) : 0) + 2 * stages * sizeof(uint64_t) + 1024;
}

// One k4 step of the warp tile: pairs of 8-row units as m16n8k4 (one instruction per pair and column unit), an odd last unit as m8n8k4.
template <int NI, int NJ>
__device__ __forceinline__ void upd_mma(const double (&af)[NI], const double (&bf)[NJ], double (&acc)[5][5][2]) {
#pragma unroll
  for (int i = 0; i + 1 < NI; i += 2)
#pragma unroll
    for (int j = 0; j < NJ; ++j) dmma_16x8x4(acc[i][j][0], acc[i][j][1], acc[i + 1][j][0], acc[i + 1][j][1], af[i], af[i + 1], bf[j]);
  if (NI & 1) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) dmma_8x8x4(acc[NI - 1][j][0], acc[NI - 1][j][1], af[NI - 1], bf[j]);
  }
}

// One K stage (16 deep, k4n <= 4 steps of 4) of a warp's (NI*8) x (NJ*8) tile.  As/Bs: byte pointers to this lane's row inside
// the swizzled [rb][128 B] tiles; kc[k4] = byte offset of this lane's (k4, t) element inside its row (swizzle applied).
template <int NI, int NJ>
__device__ __forceinline__ void upd_stage(const unsigned char* __restrict__ As, const unsigned char* __restrict__ Bs, const int (&kc)[4], int k4n, double (&acc)[5][5][2]) {
  if (k4n == 4) {
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      double af[NI], bf[NJ];
#pragma unroll
      for (int i = 0; i < NI; ++i) af[i] = *reinterpret_cast<const double*>(As + kc[k4] + i * 1024);
#pragma unroll
      for (int j = 0; j < NJ; ++j) bf[j] = *reinterpret_cast<const double*>(Bs + kc[k4] + j * 1024);
      upd_mma<NI, NJ>(af, bf, acc);
    }
  } else {
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      if (k4 < k4n) {
        double af[NI], bf[NJ];
#pragma unroll
        for (int i = 0; i < NI; ++i) af[i] = *reinterpret_cast<const double*>(As + kc[k4] + i * 1024);
#pragma unroll
        for (int j = 0; j < NJ; ++j) bf[j] = *reinterpret_cast<const double*>(Bs + kc[k4] + j * 1024);
        upd_mma<NI, NJ>(af, bf, acc);
      }
    }
  }
}

// Lane (g, t) holds accumulator columns pi(2t), pi(2t+1) of every 8-wide unit = {0,2}, {4,6}, {1,3}, {5,7} for t = 0..3: lanes t and
// t ^ 2 swap one value each so that every lane owns an adjacent pair (t = 0: 0,1  t = 2: 2,3  t = 1: 4,5  t = 3: 6,7).
// fresh: the first pass into a fill block, whose target is 0 (not read).
template <int NI, int NJ>
__device__ __forceinline__ void upd_epilogue(double* __restrict__ C, int npad, const double (&acc)[5][5][2], int t, const double* __restrict__ part, bool fresh) {
  const bool hi = (t & 2) != 0;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    double2 v[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) v[j] = fresh ? make_double2(0.0, 0.0) : *reinterpret_cast<const double2*>(C + (size_t)i * 8 * npad + j * 8);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      double a0 = acc[i][j][0], a1 = acc[i][j][1];
      if (part) { const double2 q = *reinterpret_cast<const double2*>(part + (size_t)(i * 5 + j) * 64); a0 += q.x; a1 += q.y; }   // team 1's share
      const double give = hi ? a0 : a1;
      const double got = __shfl_xor_sync(0xffffffffu, give, 2);
      const double lo = hi ? got : a0, up = hi ? a1 : got;
      v[j].x -= lo; v[j].y -= up;
      *reinterpret_cast<double2*>(C + (size_t)i * 8 * npad + j * 8) = v[j];
    }
  }
}
template <int NI, int NJ>
__device__ __forceinline__ void upd_store_partial(double* __restrict__ part, const double (&acc)[5][5][2]) {
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) *reinterpret_cast<double2*>(part + (size_t)(i * 5 + j) * 64) = make_double2(acc[i][j][0], acc[i][j][1]);
}

#define RCVD_UPD_CASES(M) \
  M(1, 1) M(1, 2) M(1, 3) M(1, 4) M(1, 5) M(2, 1) M(2, 2) M(2, 3) M(2, 4) M(2, 5) M(3, 1) M(3, 2) M(3, 3) M(3, 4) M(3, 5) \
  M(4, 1) M(4, 2) M(4, 3) M(4, 4) M(4, 5) M(5, 1) M(5, 2) M(5, 3) M(5, 4) M(5, 5)

// dst[it.dst] (tile) -= sum_p T[pairs[p].x] (rows m0..) * T[pairs[p].y] (rows n0..)^T over k < neff (an item flagged kUpdFirstFill: = 0 - sum).
// tmap: 2-D view of the T buffer, inner dimension = k (npad doubles per row), outer = block * npad + row; box = [rb][16], 128-B swizzle.
// dbg: timing experiments (results invalid); the solver passes 0.  The argument and its branches stay because without them ptxas
// allocates the K loop differently and spills its counters (CUDA 12.9): the update GEMMs measured 5-7 % slower at configs 2 and 4
// (H100 80GB HBM3, 700 W power limit).
template <int TEAMS>
__global__ void __launch_bounds__(UpdShape<TEAMS>::threads, UpdShape<TEAMS>::ctas) k_update_tma(const __grid_constant__ CUtensorMap tmap, double* __restrict__ dst,
                                                               const UpdItem* __restrict__ items, int nitems, const int2* __restrict__ pairs,
                                                               int npad, int neff, int rb, int dbg) {
  // The ring must start on a 1 KB boundary (swizzle atom = 8 rows x 128 B).  It is addressed as the extern array itself: rounding the
  // pointer up through an integer makes the compiler lose the shared address space and emit generic LD.E.64 for every fragment load.
  extern __shared__ __align__(1024) unsigned char ring[];
  // a programmatic dependent launch (the next narrow level's k_potrf_smem, which waits for this grid before reading) may take the SMs
  // this launch drains
  griddep_launch_dependents();
  if (smem_u32(ring) & 1023u) __trap();
  constexpr int kUpdStages = UpdShape<TEAMS>::stages;
  const int tile_bytes = rb * 128, stage_bytes = 2 * tile_bytes;                     // A tile then B tile, [rb][16 doubles]
  double* partial = reinterpret_cast<double*>(ring + (size_t)kUpdStages * stage_bytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(partial + (TEAMS == 2 ? kUpdPartial : 0));
  uint64_t* empty = full + kUpdStages;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int s = 0; s < kUpdStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  const int nk = (neff + 15) >> 4;
  const size_t bs = (size_t)npad * npad;
  if (warp == 4 * TEAMS) {
    // ---------------- producer: one thread drives the TMA ----------------
    if (lane != 0 || (dbg & 1)) return;          // dbg bit 0 (timing experiment only): no loads, the DMMA warps run on whatever is in shared memory
    int stage = 0; uint32_t phase = 0;
    for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
      const UpdItem it = items[w];
      for (int p = 0; p < it.count; ++p) {
        const int2 pr = pairs[it.first + p];
        const int rowA = pr.x * npad + it.m0, rowB = pr.y * npad + it.n0;
        for (int kk = 0; kk < nk; ++kk) {
          mbar_wait(&empty[stage], phase ^ 1);
          unsigned char* sa = ring + (size_t)stage * stage_bytes;
          mbar_expect_tx(&full[stage], (uint32_t)stage_bytes);
          tma_load_2d(sa, &tmap, &full[stage], kk * 16, rowA);
          tma_load_2d(sa + tile_bytes, &tmap, &full[stage], kk * 16, rowB);
          if (++stage == kUpdStages) { stage = 0; phase ^= 1; }
        }
      }
      // The item's last stage is issued, so the DMMA warps are at most kUpdStages stages from its end: prefetch the target rows into
      // L2 for the epilogue's read (not the first pass into a fill block, which does not read it; not the skipped upper warp tile).
      // One-team shape only: in the two-team shape this code alone makes ptxas spill accumulators between the DMMAs of the K loop.
      if (TEAMS == 1 && !(it.flags & kUpdFirstFill)) {
        const int hm = ((it.mrows >> 3) + 1) >> 1 << 3, hn = ((it.ncols >> 3) + 1) >> 1 << 3;
        const double* row = dst + (size_t)it.dst * bs + (size_t)it.m0 * npad + it.n0;
        for (int r = 0; r < it.mrows; ++r, row += npad) {
          const int bytes = ((it.flags & kUpdSymDiag) && r < hm ? hn : it.ncols) * 8;
          prefetch_l2_bulk(row, bytes);
        }
      }
    }
    return;
  }
  // ---------------- consumers: two teams of 2 x 2 DMMA warps; team = parity of the K stage ----------------
  const int team = warp >> 2, tw = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  const int pg = ((g & 3) << 1) | (g >> 2);                    // tile row (and column) fed to fragment index g
  int kc[4];
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4) kc[k4] = (((2 * k4 + (t >> 1)) ^ pg) << 4) + ((t & 1) << 3);
  const int wr = tw >> 1, wc = tw & 1;
  double* mypart = partial + (size_t)tw * (25 * 64) + lane * 2;     // [team-warp][unit][lane][2]
  if (TEAMS == 2 && team == 0) named_bar_arrive<2, 256>();     // "partial buffer is free" for team 1's first item
  int stage = 0; uint32_t phase = 0; unsigned sidx = 0;         // sidx: running stage counter (its parity picks the team)
  for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
    const UpdItem it = items[w];
    const int hm = ((it.mrows >> 3) + 1) >> 1 << 3, hn = ((it.ncols >> 3) + 1) >> 1 << 3;   // rows of warp-row 0 / columns of warp-column 0
    const int wm = wr * hm, wn = wc * hn;
    int ni = wr ? (it.mrows - hm) >> 3 : hm >> 3, nj = wc ? (it.ncols - hn) >> 3 : hn >> 3;
    if ((it.flags & kUpdSymDiag) && wr == 0 && wc == 1) ni = 0;         // strictly above the diagonal of a symmetric target
    if (ni == 0 || nj == 0) { ni = 0; nj = 0; }
    double acc[5][5][2];
#pragma unroll
    for (int i = 0; i < 5; ++i)
#pragma unroll
      for (int j = 0; j < 5; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }
    const int code = ni * 8 + nj;
    const int steps = it.count * nk;
    int kk = 0;
    for (int s = 0; s < steps; ++s, ++sidx) {
      if (TEAMS == 1 || (int)(sidx & 1u) == team) {
        if (!(dbg & 1)) mbar_wait(&full[stage], phase);
        const int k4n = min(4, (neff - kk * 16 + 3) >> 2);
        const unsigned char* sa = ring + (size_t)stage * stage_bytes + (size_t)(wm + pg) * 128;
        const unsigned char* sb = ring + (size_t)stage * stage_bytes + tile_bytes + (size_t)(wn + pg) * 128;
        switch (code) {
#define RCVD_UPD_STAGE(NI_, NJ_) case NI_ * 8 + NJ_: upd_stage<NI_, NJ_>(sa, sb, kc, k4n, acc); break;
          RCVD_UPD_CASES(RCVD_UPD_STAGE)
#undef RCVD_UPD_STAGE
          default: break;
        }
        __syncwarp();
        if (lane == 0 && !(dbg & 1)) mbar_arrive(&empty[stage]);
      }
      if (++stage == kUpdStages) { stage = 0; phase ^= 1; }
      if (++kk == nk) kk = 0;
    }
    if (TEAMS == 2 && team == 1) {
      // hand the partial accumulators to team 0 and go on with the next item
      named_bar_sync<2, 256>();                                // team 0 has consumed the previous partials
      switch (code) {
#define RCVD_UPD_PART(NI_, NJ_) case NI_ * 8 + NJ_: upd_store_partial<NI_, NJ_>(mypart, acc); break;
        RCVD_UPD_CASES(RCVD_UPD_PART)
#undef RCVD_UPD_PART
        default: break;
      }
      named_bar_arrive<1, 256>();                              // "partials are in shared memory"
      continue;
    }
    if (TEAMS == 2) named_bar_sync<1, 256>();
    if (dbg & 2) { if (acc[0][0][0] == 1.2345e300) dst[0] = acc[4][4][1] + acc[2][3][0]; if (TEAMS == 2) named_bar_arrive<2, 256>(); continue; }   // timing experiment: no read-modify-write of the target
    double* C = dst + (size_t)it.dst * bs + (size_t)(it.m0 + wm + pg) * npad + it.n0 + wn + ((t & 1) << 2) + (t & 2);
    const bool fresh = (it.flags & kUpdFirstFill) != 0;
    switch (code) {
#define RCVD_UPD_EPI(NI_, NJ_) case NI_ * 8 + NJ_: upd_epilogue<NI_, NJ_>(C, npad, acc, t, TEAMS == 2 ? mypart : nullptr, fresh); break;
      RCVD_UPD_CASES(RCVD_UPD_EPI)
#undef RCVD_UPD_EPI
      default: break;
    }
    if (TEAMS == 2) named_bar_arrive<2, 256>();                // partial buffer free again
  }
}

}  // namespace rcvd
