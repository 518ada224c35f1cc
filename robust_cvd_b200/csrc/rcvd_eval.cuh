// rcvd_eval.cuh -- residual / Jacobian / normal-equation evaluation kernels.
//
// Each residual family runs in one of the modes of EvalMode: the cost alone (LM step acceptance), cost + gradient (the bounded
// line search), cost + gradient + normal matrix, marking the parameters its rows reference (the active mask), or writing every
// residual block's rows to its own slot of a RowOut (rcvd_evaluate_rows).
//   k_pairs<MODE>        : flow constraints, StaticSceneCost residual + analytic Jacobian + Cauchy correction + scatter of J^T J
//                          and J^T r (reference hot loop D, lib/PoseOptimizer.cpp:237-308 evaluated by Ceres autodiff at :1198);
//                          every transform / intrinsics mode
//   k_accumulate_fast, k_accumulate_runs : the CostGradH pair kernels of the default configuration (pose block on the tensor cores)
//   k_regularisers<MODE> : scale / deform / spatial / focal / position rows (:488-656, :1341-1549)
//   k_triplets<MODE>     : scene-flow smoothness rows (:1242-1339)
//   k_depth_pairs<MODE>  : pairwise depth normalisation, DisparityDissimilarityCost rows (:425-462, added at :1005-1095)
// The partial costs of all families meet in one deterministic two-stage reduction (k_reduce_partials).
#pragma once
#include <type_traits>
#include "rcvd_device.cuh"
#include "rcvd_ptx.cuh"

namespace rcvd {

constexpr int kTile = 128;          // constraints per CTA tile (all from one group: a directed pair or a triplet centre)

enum class EvalMode { Cost, CostGrad, CostGradH, MarkActive, Rows };

// Output of the Rows mode.  Block b of a family (its slot: the caller's record order, or the regulariser row order of
// rcvd_row_layout) owns r[b*m .. b*m+m) and rho[b]: the unrobustified residual and rho(|r|^2) of the block's loss.  With the
// Jacobian (the kernels' JAC flag) row i = b*m + q also owns K column slots cols / jac[i*K .. i*K+K): the global column (the caller's
// frame * nf + local parameter) and dr_q / dx of every non-constant parameter the block reaches, then index -1 and value 0.
struct RowOut {
  double* r; double* rho; int32_t* cols; double* jac;
  int K;
  const int32_t* uperm;   // internal frame -> the caller's frame
  const int32_t* slot;    // k_regularisers: kernel row id -> block slot, -1 where the id has no row
  __device__ __forceinline__ void col(size_t row, int e, int32_t c, double v) const { cols[row * K + e] = c; jac[row * K + e] = v; }
  __device__ __forceinline__ void pad(size_t row, int e) const { for (; e < K; ++e) col(row, e, -1, 0.0); }
};
// The last kernel parameter: a RowOut in the Rows mode, an empty struct in the others.
struct NoRows {};
template <EvalMode MODE> using RowArg = typename std::conditional<MODE == EvalMode::Rows, RowOut, NoRows>::type;

// One constraint family on the device: groups of consecutive records (a group is a directed frame pair, or a triplet's centre
// frame), cut into tiles of <= kTile records of one group.  Tile t is CTA t of the family's kernel.
struct RecordTiles {
  const float* records;         // [n][record width]
  const int32_t* group_frames;  // [groups][frames per group], internal frame ids
  const int32_t* tile_group;    // [T]
  const int64_t* tile_begin;    // [T] first record
  const int32_t* tile_count;    // [T] records
};

struct DevProblem {
  rcvd_config cfg;
  Layout L;
  int N;
  RecordTiles pairs;           // static-scene pairs, records [C][6]
  RecordTiles trips;           // scene-flow smoothness triplets (optional), records [n][10]
  RecordTiles dpairs;          // pairwise depth-normalisation pairs (optional), records [n][6]
  const int32_t* blk_of;       // [N*N]: (fa,fb) -> H block id*2 + (fa is the row side), -1 if absent
  const uint8_t* in_range;     // [N]
  const double* median;        // [N]
  const double* adaptive;      // [N*G] or null
  const float* scale_locs;     // [M][2]
  int rank, nranks;            // regulariser and triplet rows are evaluated by rank f % nranks (every rank marks them all)
};

__device__ __forceinline__ bool is_const_local(const rcvd_config& c, const Layout& L, int l) {
  if (l < 6) return c.fix_poses != 0;
  if (l == 6) return c.intr_opt == RCVD_INTR_FIXED;
  if (l < L.offS) return c.fix_depth_xforms != 0;
  return c.fix_spatial_xforms != 0;
}

// Adds v to H(fa:la, fb:lb).  Diagonal blocks store the lower triangle only.
__device__ __forceinline__ void add_h(const DevProblem& p, double* H, int fa, int la, int fb, int lb, double v) {
  const int np = p.L.npad;
  if (fa == fb) {
    const int i = max(la, lb), j = min(la, lb);
    red_add(H + (size_t)fa * np * np + (size_t)i * np + j, v);
  } else {
    const int enc = p.blk_of[fa * p.N + fb];
    const size_t base = (size_t)(enc >> 1) * np * np;
    if (enc & 1) red_add(H + base + (size_t)la * np + lb, v);
    else red_add(H + base + (size_t)lb * np + la, v);
  }
}

struct StaticEval {
  double r[3];
  double rho0, scale;
};

// Front end of k_pairs: loads the record, gathers, evaluates residual (+ local Jacobian).
template <bool JAC>
__device__ __forceinline__ void eval_constraint(const DevProblem& p, const double* __restrict__ x, int f0, int f1,
                                                const float* __restrict__ rec, Gather& dg0, Gather& sg0, Gather& dg1, Gather& sg1,
                                                StaticEval& ev, double* Jl) {
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const double* pf0 = x + (size_t)f0 * L.nf; const double* pf1 = x + (size_t)f1 * L.nf;
  ObsIn o0{rec[0], rec[1], rec[2]}, o1{rec[3], rec[4], rec[5]};
  gather_depth(c, o0.ndcx, o0.ndcy, dg0); gather_depth(c, o1.ndcx, o1.ndcy, dg1);
  gather_spatial(c, o0.ndcx, o0.ndcy, sg0); gather_spatial(c, o1.ndcx, o1.ndcy, sg1);
  double phi0, phi1;
  if (c.intr_opt == RCVD_INTR_SHARED) phi0 = phi1 = x[6];          // &poseParams_[0][6], lib/PoseOptimizer.cpp:1226
  else if (c.intr_opt == RCVD_INTR_PER_FRAME) { phi0 = pf0[6]; phi1 = pf1[6]; }
  else phi0 = phi1 = c.fixed_vfocal;
  const double D0 = depth_value(c, L, dg0, o0.depth, pf0), D1 = depth_value(c, L, dg1, o1.depth, pf1);
  double u0[2], u1[2];
  warp_value(L, sg0, pf0, u0); warp_value(L, sg1, pf1, u1);
  static_scene<JAC>(c, pf0, phi0, D0, u0, pf1, phi1, D1, u1, o0, o1, ev.r, Jl);
  const double s = ev.r[0] * ev.r[0] + ev.r[1] * ev.r[1] + ev.r[2] * ev.r[2];
  double rho1;
  robust_loss(c, s, ev.rho0, rho1);
  ev.scale = sqrt(rho1);    // Corrector with rho'' <= 0: residual and Jacobian scaled by sqrt(rho')
}

// Block-level sum -> partial[blockIdx.x]  (deterministic two-stage cost reduction)
__device__ __forceinline__ void block_store_sum(double v, double* partial) {
  __shared__ double red[32];
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (wid == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    double t = lane < nw ? red[lane] : 0.0;
    t = warp_sum(t);
    if (lane == 0) *partial = t;
  }
}

// Column expansion of one row block over NF frames fr[] (pair constraints NF = 2, smoothness triplets NF = 3).  Jl: the 3 x 10 NF
// local Jacobian (per frame: pose 6, focal, depth D, warp 2).  Every column a parameter sees goes to push(frame, local column,
// 3-vector), constant parameters included -- pose, PerFrame focal, depth nodes (x src; the offset too when k = 2), spatial nodes,
// then the shared focal.
template <int NF, class Push>
__device__ __forceinline__ void for_each_column(const DevProblem& p, const int* fr, const float* __restrict__ rec, const Gather* dg, const Gather* sg,
                                                const double* Jl, Push&& push) {
  constexpr int ld = 10 * NF;           // Jacobian row stride
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  for (int side = 0; side < NF; ++side) {
    const int f = fr[side], o = side * 10;
    const double src = (double)rec[3 * side + 2];
    for (int q = 0; q < 6; ++q) push(f, q, Jl[o + q], Jl[ld + o + q], Jl[2 * ld + o + q]);
    if (c.intr_opt == RCVD_INTR_PER_FRAME) push(f, 6, Jl[o + 6], Jl[ld + o + 6], Jl[2 * ld + o + 6]);
    for (int q = 0; q < dg[side].n; ++q) {
      const double w = dg[side].w[q];
      push(f, L.offD + dg[side].idx[q] * L.k, Jl[o + 7] * w * src, Jl[ld + o + 7] * w * src, Jl[2 * ld + o + 7] * w * src);
      if (L.k == 2) push(f, L.offD + dg[side].idx[q] * 2 + 1, Jl[o + 7] * w, Jl[ld + o + 7] * w, Jl[2 * ld + o + 7] * w);
    }
    for (int q = 0; q < sg[side].n; ++q) {
      const double w = sg[side].w[q];
      push(f, L.offS + sg[side].idx[q] * 2, Jl[o + 8] * w, Jl[ld + o + 8] * w, Jl[2 * ld + o + 8] * w);
      push(f, L.offS + sg[side].idx[q] * 2 + 1, Jl[o + 9] * w, Jl[ld + o + 9] * w, Jl[2 * ld + o + 9] * w);
    }
  }
  if (c.intr_opt == RCVD_INTR_SHARED) {   // one focal for every frame: the sum of the frames' focal columns, in frame order
    double s[3];
    for (int i = 0; i < 3; ++i) { s[i] = Jl[i * ld + 6]; for (int side = 1; side < NF; ++side) s[i] += Jl[i * ld + side * 10 + 6]; }
    push(0, 6, s[0], s[1], s[2]);
  }
}

// Scatter of one row block: r the residual, sc its scale; g += J^T r over the columns of for_each_column that are not held constant,
// with WANT_H also H += J^T J (lower triangle, add_h).
template <int NF, bool WANT_H>
__device__ __forceinline__ void scatter_columns(const DevProblem& p, const int* fr, const float* __restrict__ rec, const Gather* dg, const Gather* sg,
                                                const double* Jl, const double* r, double sc, double* __restrict__ H, double* __restrict__ g) {
  constexpr int kMaxCols = 72 * NF;     // NF (6 + 1 + 16*2 + 16*2) + the shared focal, with slack
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const double r0 = r[0] * sc, r1 = r[1] * sc, r2 = r[2] * sc;
  int ef[kMaxCols]; short el[kMaxCols]; double ej[kMaxCols][3];
  int E = 0;
  for_each_column<NF>(p, fr, rec, dg, sg, Jl, [&](int f, int l, double a0, double a1, double a2) {
    if (is_const_local(c, L, l)) return;
    ef[E] = f; el[E] = (short)l; ej[E][0] = a0 * sc; ej[E][1] = a1 * sc; ej[E][2] = a2 * sc; ++E;
  });
  const int np = L.npad;
  for (int a = 0; a < E; ++a) {
    const double a0 = ej[a][0], a1 = ej[a][1], a2 = ej[a][2];
    red_add(g + (size_t)ef[a] * np + el[a], a0 * r0 + a1 * r1 + a2 * r2);
    if (WANT_H) for (int b = 0; b <= a; ++b) add_h(p, H, ef[a], el[a], ef[b], el[b], a0 * ej[b][0] + a1 * ej[b][1] + a2 * ej[b][2]);
  }
}

// Rows mode of k_pairs / k_triplets: block `slot`'s three residuals r, its rho and (JAC) its rows of for_each_column, unscaled.
template <int NF, bool JAC>
__device__ __forceinline__ void store_rows(const DevProblem& p, const RowOut& o, size_t slot, const int* fr, const float* __restrict__ rec,
                                           const Gather* dg, const Gather* sg, const double* Jl, const double* r, double rho) {
  for (int q = 0; q < 3; ++q) o.r[slot * 3 + q] = r[q];
  o.rho[slot] = rho;
  if constexpr (JAC) {
    const rcvd_config& c = p.cfg; const Layout& L = p.L;
    int E = 0;
    for_each_column<NF>(p, fr, rec, dg, sg, Jl, [&](int f, int l, double a0, double a1, double a2) {
      if (is_const_local(c, L, l)) return;
      const int32_t col = o.uperm[f] * L.nf + l;
      o.col(slot * 3, E, col, a0); o.col(slot * 3 + 1, E, col, a1); o.col(slot * 3 + 2, E, col, a2); ++E;
    });
    for (int q = 0; q < 3; ++q) o.pad(slot * 3 + q, E);
  }
}

// Marks the parameters of one frame (its row m of the mask, npad stride) that a residual reaches through pose, focal and the
// gathered depth / spatial nodes.
__device__ __forceinline__ void mark_frame(const rcvd_config& c, const Layout& L, uint8_t* m, const Gather& dg, const Gather& sg) {
  for (int q = 0; q < 6; ++q) m[q] = 1;
  if (c.intr_opt == RCVD_INTR_PER_FRAME) m[6] = 1;
  for (int q = 0; q < dg.n; ++q) for (int j = 0; j < L.k; ++j) m[L.offD + dg.idx[q] * L.k + j] = 1;
  for (int q = 0; q < sg.n; ++q) { m[L.offS + sg.idx[q] * 2] = 1; m[L.offS + sg.idx[q] * 2 + 1] = 1; }
}

// Pair constraints in every mode and every transform / intrinsics configuration; scatter with L2 reductions.  MarkActive marks
// the parameters referenced by at least one residual block (the Ceres program's parameter set, used for |x| / |step| norms).  Rows
// writes record i's rows to slot i: the records must be in the caller's order (not the run path's sorted copy).
template <EvalMode MODE, bool JAC = false>
__global__ void __launch_bounds__(kTile) k_pairs(DevProblem p, const double* __restrict__ x, double* __restrict__ H, double* __restrict__ g,
                                                 double* __restrict__ partial, uint8_t* __restrict__ mask, RowArg<MODE> rows) {
  const rcvd_config& c = p.cfg;
  const int t = blockIdx.x;
  const int pr = p.pairs.tile_group[t];
  const int f0 = p.pairs.group_frames[2 * pr], f1 = p.pairs.group_frames[2 * pr + 1];
  double cost = 0.0;
  if ((int)threadIdx.x < p.pairs.tile_count[t]) {
    const float* rec = p.pairs.records + (size_t)(p.pairs.tile_begin[t] + threadIdx.x) * 6;
    if constexpr (MODE == EvalMode::MarkActive) {
      for (int side = 0; side < 2; ++side) {
        Gather dg, sg;
        gather_depth(c, rec[side * 3], rec[side * 3 + 1], dg); gather_spatial(c, rec[side * 3], rec[side * 3 + 1], sg);
        mark_frame(c, p.L, mask + (size_t)(side ? f1 : f0) * p.L.npad, dg, sg);
      }
      if (c.intr_opt == RCVD_INTR_SHARED) mask[6] = 1;
    } else {
      StaticEval ev;
      if constexpr (MODE == EvalMode::Cost) {
        Gather dg0, sg0, dg1, sg1;   // (as four variables the frame is 8 B smaller than with the arrays below)
        eval_constraint<false>(p, x, f0, f1, rec, dg0, sg0, dg1, sg1, ev, nullptr);
      } else if constexpr (MODE == EvalMode::Rows) {
        const int fr[2] = {f0, f1}; Gather dg[2], sg[2]; double Jl[JAC ? 60 : 1];
        eval_constraint<JAC>(p, x, f0, f1, rec, dg[0], sg[0], dg[1], sg[1], ev, JAC ? Jl : nullptr);
        store_rows<2, JAC>(p, rows, (size_t)(p.pairs.tile_begin[t] + threadIdx.x), fr, rec, dg, sg, Jl, ev.r, ev.rho0);
      } else {
        const int fr[2] = {f0, f1}; Gather dg[2], sg[2]; double Jl[60];
        eval_constraint<true>(p, x, f0, f1, rec, dg[0], sg[0], dg[1], sg[1], ev, Jl);
        scatter_columns<2, MODE == EvalMode::CostGradH>(p, fr, rec, dg, sg, Jl, ev.r, ev.scale, H, g);
      }
      cost = 0.5 * ev.rho0;
    }
  }
  if (MODE != EvalMode::MarkActive && MODE != EvalMode::Rows) block_store_sum(cost, partial + t);
}

// ---------------------------------------------------------------------------
// Tensor-core pair kernels: depth transform Identity / Global / bilinear Grid with Scale value transform, identity spatial
// transform, PerFrame or Fixed intrinsics, nothing held constant -- the reference's default configuration
// (pose_optimization.py:197-207 + coarse-to-fine grids).  Per constraint the Jacobian is kept in "local" variables (pose 6,
// focal, depth D per frame); the dense 14 x 14 pose/focal normal block and its gradient are reduced over the 128 constraints
// of the tile on the fp64 tensor cores (J^T [J | r] as an m8n8k4 DMMA GEMM with K = 3 x 128 residual rows staged in shared
// memory), so they cost 119 L2 reductions per tile instead of per constraint.
// ---------------------------------------------------------------------------
constexpr int kJsLd = 20;   // k_accumulate_fast's [k][col] staging layout, 20-double rows: conflict-free DMMA fragment loads
constexpr int kRunLd = 24;  // k_accumulate_runs': 0-13 pose/focal (frame 0, frame 1), 14 r, 15 zero, 16-19 nodes of frame 0, 20-23 nodes of frame 1
constexpr int kFastSmem = (3 * kTile * kJsLd + 4 * 256) * (int)sizeof(double);
constexpr int kRunSmem = ((3 * kTile + 4) * kRunLd + 4 * 256) * (int)sizeof(double) + kTile * (int)sizeof(unsigned);

// Configurations k_accumulate_fast serves, and the subset k_accumulate_runs serves (bilinear grid, node ids fit the 16-bit halves of the sort key)
__host__ __device__ inline bool fast_path_ok(const rcvd_config& c, const Layout& L) {
  return L.k == 1 && c.spatial_type == RCVD_SPATIAL_IDENTITY && c.intr_opt != RCVD_INTR_SHARED && !c.fix_poses && !c.fix_depth_xforms &&
         !c.fix_spatial_xforms && (c.depth_type != RCVD_DEPTH_GRID || !c.depth_cubic);
}
__host__ __device__ inline bool run_path_ok(const rcvd_config& c, const Layout& L) { return fast_path_ok(c, L) && c.depth_type == RCVD_DEPTH_GRID && L.G < 65535; }

// The three H blocks a pair (f0, f1) touches: its two diagonal blocks and the cross block, stored with frame 0 or frame 1 as rows.
struct PairBlocks {
  double *H0, *H1, *Hx; bool f0rows; int np;
  // H(frame 1 ? f1 : f0, li; same frame, lj), li >= lj: diagonal blocks keep their lower triangle
  __device__ __forceinline__ void add_diag(bool frame1, int li, int lj, double v) const { red_add((frame1 ? H1 : H0) + (size_t)li * np + lj, v); }
  // H(fa:la, fb:lb) with fa = (a_f0 ? f0 : f1), fb the other frame: the one stored copy of it and of its mirror H(fb:lb, fa:la)
  __device__ __forceinline__ void add_cross(bool a_f0, int la, int lb, double v) const {
    if (a_f0 == f0rows) red_add(Hx + (size_t)la * np + lb, v); else red_add(Hx + (size_t)lb * np + la, v);
  }
};
__device__ __forceinline__ PairBlocks pair_blocks(const DevProblem& p, double* H, int f0, int f1) {
  const int np = p.L.npad; const size_t bs = (size_t)np * np;
  const int enc = p.blk_of[f0 * p.N + f1];          // cross block id*2 + (f0 is the row side)
  return PairBlocks{H + (size_t)f0 * bs, H + (size_t)f1 * bs, H + (size_t)(enc >> 1) * bs, (enc & 1) != 0, np};
}

// One constraint of the tensor-core kernels: Jl = the 3 x 20 local Jacobian scaled by sqrt(rho') (focal columns zero unless
// PerFrame), r the scaled residual, and per frame the top-left depth node of the constraint's cell with the four node weights
// times the source depth (dD/ds_i; Global depth: node 0 and w[0] only).  GRID: the caller serves bilinear grids only.
struct TcEval { double r0, r1, r2, cost; int node0, node1; double w0[4], w1[4]; };

template <bool GRID>
__device__ __forceinline__ void tc_eval(const DevProblem& p, const double* __restrict__ x, int f0, int f1, const float* __restrict__ rec, double* Jl, TcEval& e) {
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const double* pf0 = x + (size_t)f0 * L.nf; const double* pf1 = x + (size_t)f1 * L.nf;
  ObsIn o0{rec[0], rec[1], rec[2]}, o1{rec[3], rec[4], rec[5]};
  double D0 = (double)o0.depth, D1 = (double)o1.depth;
  if (!GRID && c.depth_type == RCVD_DEPTH_GLOBAL) {
    e.node0 = e.node1 = 0; e.w0[0] = D0; e.w1[0] = D1;          // dD/ds = src
    D0 *= pf0[L.offD]; D1 *= pf1[L.offD];
  } else if (GRID || c.depth_type == RCVD_DEPTH_GRID) {
    const int gx = c.depth_grid_x;
    e.node0 = bilinear_cell(o0.ndcx, o0.ndcy, gx, c.depth_grid_y, e.w0);
    e.node1 = bilinear_cell(o1.ndcx, o1.ndcy, gx, c.depth_grid_y, e.w1);
    // GridDepthFunctor::eval: res += (src * s_i) * w_i, in node order
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int dq = (q & 1) + (q >> 1) * gx;
      a0 += (D0 * pf0[L.offD + e.node0 + dq]) * e.w0[q]; a1 += (D1 * pf1[L.offD + e.node1 + dq]) * e.w1[q];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) { e.w0[q] *= D0; e.w1[q] *= D1; }          // dD/ds_i = w_i * src
    D0 = a0; D1 = a1;
  }
  const double phi0 = (c.intr_opt == RCVD_INTR_PER_FRAME) ? pf0[6] : c.fixed_vfocal;
  const double phi1 = (c.intr_opt == RCVD_INTR_PER_FRAME) ? pf1[6] : c.fixed_vfocal;
  const double u[2] = {0.0, 0.0};
  double r[3];
  static_scene<true>(c, pf0, phi0, D0, u, pf1, phi1, D1, u, o0, o1, r, Jl);
  const double s = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  double rho0, rho1;
  robust_loss(c, s, rho0, rho1);
  e.cost = 0.5 * rho0;
  const double sc = sqrt(rho1);
  e.r0 = r[0] * sc; e.r1 = r[1] * sc; e.r2 = r[2] * sc;
#pragma unroll
  for (int i = 0; i < 60; ++i) Jl[i] *= sc;
  if (c.intr_opt != RCVD_INTR_PER_FRAME) { Jl[6] = Jl[26] = Jl[46] = 0.0; Jl[16] = Jl[36] = Jl[56] = 0.0; }
}

// Stages the constraint's three [J_P | r] rows (LD doubles apart): columns 0..6 frame-0 pose+focal, 7..13 frame 1, 14 r, 15 zero
template <int LD>
__device__ __forceinline__ void stage_pose_rows(double* Js, int tid, const double* Jl, const TcEval& e) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double* row = Js + (size_t)(tid * 3 + i) * LD;
#pragma unroll
    for (int q = 0; q < 7; ++q) { row[q] = Jl[i * 20 + q]; row[7 + q] = Jl[i * 20 + 10 + q]; }
    row[14] = (i == 0) ? e.r0 : (i == 1 ? e.r1 : e.r2);
    row[15] = 0.0;
  }
}

// Ms[warp] = J_P^T [J_P | r] (16 x 16) over this warp's 96 staged residual rows, on the fp64 tensor cores
template <int LD>
__device__ __forceinline__ void pose_block_mma(const double* Js, double* Ms, int warp, int lane) {
  const int gq = lane >> 2, tq = lane & 3;
  double acc[2][2][2] = {{{0.0, 0.0}, {0.0, 0.0}}, {{0.0, 0.0}, {0.0, 0.0}}};
  const double* base = Js + (size_t)warp * 96 * LD;
#pragma unroll 4
  for (int k4 = 0; k4 < 24; ++k4) {
    const double* rowp = base + (size_t)(k4 * 4 + tq) * LD;
    const double a0 = rowp[gq], a1 = rowp[8 + gq];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) dmma_8x8x4(acc[i][j][0], acc[i][j][1], i ? a1 : a0, j ? a1 : a0);
  }
  double* mw = Ms + warp * 256;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) { mw[(i * 8 + gq) * 16 + j * 8 + 2 * tq] = acc[i][j][0]; mw[(i * 8 + gq) * 16 + j * 8 + 2 * tq + 1] = acc[i][j][1]; }
}

// Adds the sum of the four warps' M to the pair's H blocks (rows / columns 0..13) and to g (column 14)
__device__ __forceinline__ void scatter_pose_block(const double* Ms, const PairBlocks& hb, double* __restrict__ g, int f0, int f1) {
  for (int e = threadIdx.x; e < 256; e += kTile) {
    const int i = e >> 4, j = e & 15;
    if (i >= 14 || j >= 15) continue;
    const double v = Ms[e] + Ms[256 + e] + Ms[512 + e] + Ms[768 + e];
    const int li = i < 7 ? i : i - 7;
    if (j == 14) { red_add(g + (size_t)(i < 7 ? f0 : f1) * hb.np + li, v); continue; }
    const bool jf0 = j < 7; const int lj = jf0 ? j : j - 7;
    if ((i < 7) == jf0) { if (li >= lj) hb.add_diag(i >= 7, li, lj, v); }
    else if (i < 7) hb.add_cross(true, li, lj, v);   // each cross entry appears twice in M (i<7,j>=7 and mirrored); take this one
  }
}

// K1 (fast path): the spline-node columns (<= 4 nodes per frame) are expanded per thread and scattered with RED.ADD.F64.
__global__ void __launch_bounds__(kTile) k_accumulate_fast(DevProblem p, const double* __restrict__ x, double* __restrict__ H,
                                                            double* __restrict__ g, double* __restrict__ partial) {
  extern __shared__ __align__(16) double sm[];
  double* Js = sm;                                  // [3*kTile][kJsLd]
  double* Ms = sm + 3 * kTile * kJsLd;              // [4 warps][16][16]
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const int t = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int pr = p.pairs.tile_group[t];
  const int f0 = p.pairs.group_frames[2 * pr], f1 = p.pairs.group_frames[2 * pr + 1];
  const int np = L.npad, gx = c.depth_grid_x;
  const PairBlocks hb = pair_blocks(p, H, f0, f1);
  const bool active = tid < p.pairs.tile_count[t];
  const int nn = c.depth_type == RCVD_DEPTH_GRID ? 4 : (c.depth_type == RCVD_DEPTH_GLOBAL ? 1 : 0);
  double Jl[60]; TcEval e = {};
#pragma unroll
  for (int i = 0; i < 60; ++i) Jl[i] = 0.0;
  if (active) tc_eval<false>(p, x, f0, f1, p.pairs.records + (size_t)(p.pairs.tile_begin[t] + tid) * 6, Jl, e);
  stage_pose_rows<kJsLd>(Js, tid, Jl, e);
  // ---- per-thread scatter of the spline-node columns ----
  if (active && nn > 0) {
    const double r0 = e.r0, r1 = e.r1, r2 = e.r2;
    const double ca0 = Jl[7], ca1 = Jl[27], ca2 = Jl[47];      // d r / d D0
    const double cb0 = Jl[17], cb1 = Jl[37], cb2 = Jl[57];     // d r / d D1
    const double gDa = ca0 * r0 + ca1 * r1 + ca2 * r2, gDb = cb0 * r0 + cb1 * r1 + cb2 * r2;
    const double mAA = ca0 * ca0 + ca1 * ca1 + ca2 * ca2, mBB = cb0 * cb0 + cb1 * cb1 + cb2 * cb2, mAB = ca0 * cb0 + ca1 * cb1 + ca2 * cb2;
    double mPa[14], mPb[14];   // M[P, Da], M[P, Db]
#pragma unroll
    for (int q = 0; q < 7; ++q) {
      mPa[q] = Jl[q] * ca0 + Jl[20 + q] * ca1 + Jl[40 + q] * ca2;
      mPa[7 + q] = Jl[10 + q] * ca0 + Jl[30 + q] * ca1 + Jl[50 + q] * ca2;
      mPb[q] = Jl[q] * cb0 + Jl[20 + q] * cb1 + Jl[40 + q] * cb2;
      mPb[7 + q] = Jl[10 + q] * cb0 + Jl[30 + q] * cb1 + Jl[50 + q] * cb2;
    }
    const int nphi = (c.intr_opt == RCVD_INTR_PER_FRAME) ? 7 : 6;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i < nn) {
        const int la = L.offD + e.node0 + (i & 1) + (i >> 1) * gx, lb = L.offD + e.node1 + (i & 1) + (i >> 1) * gx;
        const double wa = e.w0[i], wb = e.w1[i];
        red_add(g + (size_t)f0 * np + la, gDa * wa);
        red_add(g + (size_t)f1 * np + lb, gDb * wb);
        for (int q = 0; q < nphi; ++q) {
          // node of frame 0 against pose/focal of frame 0 (same block, node row > pose col) and of frame 1 (cross block)
          hb.add_diag(false, la, q, mPa[q] * wa);
          hb.add_cross(true, la, q, mPa[7 + q] * wa);
          hb.add_diag(true, lb, q, mPb[7 + q] * wb);
          hb.add_cross(true, q, lb, mPb[q] * wb);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (j < nn) {
            const int la2 = L.offD + e.node0 + (j & 1) + (j >> 1) * gx, lb2 = L.offD + e.node1 + (j & 1) + (j >> 1) * gx;
            if (la >= la2) hb.add_diag(false, la, la2, mAA * wa * e.w0[j]);
            if (lb >= lb2) hb.add_diag(true, lb, lb2, mBB * wb * e.w1[j]);
            hb.add_cross(true, la, lb2, mAB * wa * e.w1[j]);
          }
        }
      }
    }
  }
  __syncthreads();
  pose_block_mma<kJsLd>(Js, Ms, warp, lane);
  __syncthreads();
  scatter_pose_block(Ms, hb, g, f0, f1);
  block_store_sum(e.cost, partial + t);
}

// ---------------------------------------------------------------------------
// K1 (run path): bilinear depth grid, the reference's default once coarse-to-fine has left the Global transform.
// The records of a pair are sorted by (source cell, target cell) when the problem is set up (rcvd_api.cu, device segmented sort), so
// consecutive constraints share their eight spline nodes.  A run = the constraints of one warp with the same cell pair.  Per run the
// node rows of the normal equations,
//       M[node, :] = sum_c  J_node(c)^T [ J_pose(c) | r(c) | J_node(c) ]        (8 x 24: 4 + 4 nodes against 14 pose/focal, r, 8 nodes)
// are reduced over the run on the fp64 tensor cores (m8n8k4, K = the run's residual rows staged in shared memory) and leave the SM as ONE
// reduction per entry per run (156 REDs) instead of one per constraint; the 14 x 14 pose/focal block is reduced over the whole
// 128-constraint tile as in k_accumulate_fast.  matchSeparation 10 (about three constraints per cell pair): ~53 REDs per constraint
// instead of 157; dense constraints (hundreds per cell pair): ~6.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kTile) k_accumulate_runs(DevProblem p, const double* __restrict__ x, double* __restrict__ H,
                                                            double* __restrict__ g, double* __restrict__ partial) {
  extern __shared__ __align__(16) double sm[];
  double* Js = sm;                                        // [3*kTile + 4][kRunLd]
  double* Ms = sm + (3 * kTile + 4) * kRunLd;             // [4 warps][16][16]
  unsigned* skey = reinterpret_cast<unsigned*>(Ms + 4 * 256);
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const int t = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int pr = p.pairs.tile_group[t];
  const int f0 = p.pairs.group_frames[2 * pr], f1 = p.pairs.group_frames[2 * pr + 1];
  const int np = L.npad;
  const PairBlocks hb = pair_blocks(p, H, f0, f1);
  const int gx = c.depth_grid_x;
  double cost = 0.0;
  const bool active = tid < p.pairs.tile_count[t];
  unsigned key = 0xffffffffu;
  {
    double Jl[60]; TcEval e = {};
#pragma unroll
    for (int i = 0; i < 60; ++i) Jl[i] = 0.0;
    if (active) {
      tc_eval<true>(p, x, f0, f1, p.pairs.records + (size_t)(p.pairs.tile_begin[t] + tid) * 6, Jl, e);
      key = ((unsigned)e.node0 << 16) | (unsigned)e.node1;
    }
    cost = e.cost;
    stage_pose_rows<kRunLd>(Js, tid, Jl, e);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      double* row = Js + (size_t)(tid * 3 + i) * kRunLd;
      const double ca = Jl[i * 20 + 7], cb = Jl[i * 20 + 17];            // d r_i / d D0, d r_i / d D1
#pragma unroll
      for (int q = 0; q < 4; ++q) { row[16 + q] = ca * e.w0[q]; row[20 + q] = cb * e.w1[q]; }
    }
    if (tid < 4 * kRunLd) Js[(size_t)3 * kTile * kRunLd + tid] = 0.0;     // four zero rows behind the tile (the K steps of the last run read them)
    skey[tid] = key;
  }
  __syncthreads();
  // ---- pose / focal block of the whole tile ----
  pose_block_mma<kRunLd>(Js, Ms, warp, lane);
  // ---- spline-node rows, one run at a time (runs never cross a warp: at most three extra runs per tile) ----
  {
    const int gq = lane >> 2, tq = lane & 3;
    const int c0 = warp * 32 + lane;
    const unsigned kprev = lane ? skey[c0 - 1] : ~key;
    const unsigned starts = __ballot_sync(0xffffffffu, key != kprev || lane == 0);
    unsigned rem = starts;
    const bool per_frame = c.intr_opt == RCVD_INTR_PER_FRAME;
    while (rem) {
      const int s0 = __ffs(rem) - 1; rem &= rem - 1;
      const int s1 = rem ? __ffs(rem) - 1 : 32;
      const unsigned rk = skey[warp * 32 + s0];
      if (rk == 0xffffffffu) break;                        // the padding behind the last constraint of the tile
      const int row0 = 3 * (warp * 32 + s0), row1 = 3 * (warp * 32 + s1);
      double acc[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}};
      for (int rr = row0; rr < row1; rr += 4) {
        const int row = rr + tq;
        const double* rowp = Js + (size_t)row * kRunLd;
        const bool in = row < row1;                                       // the last K step of a run reaches into the next run: masked
        const double a = in ? rowp[16 + gq] : 0.0;
#pragma unroll
        for (int nb = 0; nb < 3; ++nb) dmma_8x8x4(acc[nb][0], acc[nb][1], a, in ? rowp[nb * 8 + gq] : 0.0);
      }
      // lane (gq, tq) holds M[node gq][columns nb*8 + 2 tq, + 1]
      const int ba = (int)(rk >> 16), bb = (int)(rk & 0xffffu);
      const bool rowA = gq < 4;
      const int qn = gq & 3;
      const int ln = L.offD + (rowA ? ba : bb) + (qn & 1) + (qn >> 1) * gx;   // local column of this lane's node
      const int fn = rowA ? f0 : f1;
#pragma unroll
      for (int nb = 0; nb < 3; ++nb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = nb * 8 + 2 * tq + e;
          const double v = acc[nb][e];
          if (col < 14) {
            const int pc = col < 7 ? col : col - 7;
            if (pc == 6 && !per_frame) continue;
            const bool colA = col < 7;
            if (colA == rowA) hb.add_diag(!rowA, ln, pc, v);                                 // node row > pose column: lower triangle
            else hb.add_cross(rowA, ln, pc, v);                                                 // node against the other frame's pose: cross block
          } else if (col == 14) {
            red_add(g + (size_t)fn * np + ln, v);
          } else if (col >= 16) {
            const int m = col - 16, qm = m & 3; const bool colNodeA = m < 4;
            const int lm = L.offD + (colNodeA ? ba : bb) + (qm & 1) + (qm >> 1) * gx;
            if (colNodeA == rowA) { if (ln >= lm) hb.add_diag(!rowA, ln, lm, v); }          // same frame: lower triangle once
            else if (rowA) hb.add_cross(true, ln, lm, v);                                           // (frame-0 node, frame-1 node): once, from the frame-0 row
          }
        }
    }
  }
  __syncthreads();
  scatter_pose_block(Ms, hb, g, f0, f1);
  block_store_sum(cost, partial + t);
}

// Sort key of a record for the run path: (top-left node of the source cell) << 16 | (top-left node of the target cell)
__global__ void __launch_bounds__(256) k_record_keys(rcvd_config c, const float* __restrict__ records, long long n, unsigned* __restrict__ keys, int* __restrict__ idx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* rec = records + (size_t)i * 6;
  double w[4];   // unused: only the nodes make the key
  const unsigned ba = (unsigned)bilinear_cell(rec[0], rec[1], c.depth_grid_x, c.depth_grid_y, w);
  keys[i] = (ba << 16) | (unsigned)bilinear_cell(rec[3], rec[4], c.depth_grid_x, c.depth_grid_y, w);
  idx[i] = (int)i;
}
__global__ void __launch_bounds__(256) k_gather_records(const float* __restrict__ src, const int* __restrict__ idx, long long n, float* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 6) return;
  const long long rcd = i / 6; const int e = (int)(i % 6);
  dst[i] = src[(size_t)idx[rcd] * 6 + e];
}

// --- K3: regulariser rows ---------------------------------------------------
struct RegCounts { int scale, deform, spatial, focal, per_frame; int position_rows; int total; };

__host__ __device__ inline RegCounts reg_counts(const rcvd_config& c, const Layout& L, int N, int nscale) {
  RegCounts r;
  r.scale = (c.scale_reg > 0.0 && !c.fix_depth_xforms && (c.depth_type == RCVD_DEPTH_GLOBAL || c.depth_type == RCVD_DEPTH_GRID)) ? nscale : 0;
  r.deform = (c.depth_deform_reg > 0.0 && c.depth_type == RCVD_DEPTH_GRID)
                 ? ((c.depth_grid_x - 1) * c.depth_grid_y + c.depth_grid_x * (c.depth_grid_y - 1)) * L.k : 0;
  r.spatial = (c.spatial_deform_reg > 0.0) ? L.ns : 0;
  r.focal = (c.focal_reg > 0.0 && c.intr_opt != RCVD_INTR_FIXED) ? 1 : 0;
  r.per_frame = r.scale + r.deform + r.spatial + r.focal;
  r.position_rows = (c.position_reg > 0.0 && N >= 3) ? (N - 2) * 3 : 0;
  r.total = r.per_frame * N + r.position_rows;
  return r;
}

// Rows: row id -> slot through rows.slot; rho = r^2 (ScaledLoss weights are folded into r as sqrt(w), the other rows have no loss).
template <EvalMode MODE, bool JAC = false>
__global__ void __launch_bounds__(128) k_regularisers(DevProblem p, RegCounts rc, const double* __restrict__ x, double* __restrict__ H,
                                                      double* __restrict__ g, double* __restrict__ partial, uint8_t* __restrict__ mask,
                                                      int first_frame, int last_frame, RowArg<MODE> rows) {
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const int np = L.npad;
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  double cost = 0.0;
  int nent = 0; int ef[3] = {0, 0, 0}; int el[32]; double ed[32]; int efr[32];   // entries (frame, local, derivative)
  double r = 0.0; bool valid = false;
  if (id < rc.per_frame * p.N) {
    const int f = id / rc.per_frame; int k = id % rc.per_frame;
    const bool mine = MODE == EvalMode::MarkActive || (p.nranks <= 1) || (f % p.nranks == p.rank);
    if (p.in_range[f] && mine) {
      const double* pf = x + (size_t)f * L.nf;
      ef[0] = f;
      if (k < rc.scale) {
        // TargetDisparityCost (lib/PoseOptimizer.cpp:488-517) on the lattice of :1382-1385, ScaledLoss(scaleReg)
        const double sw = sqrt(c.scale_reg);
        const float med = (float)p.median[f];
        Gather gth; gather_depth(c, p.scale_locs[2 * k], p.scale_locs[2 * k + 1], gth);
        const double depth = depth_value(c, L, gth, med, pf);
        const bool clamped = depth < 1e-6;
        r = (1.0 / (clamped ? 1e-6 : depth) - 1.0) * sw;
        const double dd = clamped ? 0.0 : -1.0 / (depth * depth);
        for (int q = 0; q < gth.n; ++q) {
          el[nent] = L.offD + gth.idx[q] * L.k; ed[nent] = dd * gth.w[q] * (double)med * sw; efr[nent] = f; ++nent;
          if (L.k == 2) { el[nent] = L.offD + gth.idx[q] * 2 + 1; ed[nent] = dd * gth.w[q] * sw; efr[nent] = f; ++nent; }
        }
        valid = true;
      } else if ((k -= rc.scale) < rc.deform) {
        // computeGridDeformationCost (lib/DepthMapTransform.cpp:631-667) * weight (DeformationCost / Adaptive, :536-656)
        const int gx = c.depth_grid_x, gy = c.depth_grid_y;
        const int comp = k % L.k; const int e = k / L.k;
        int a, b;
        const int nh = (gx - 1) * gy;
        if (e < nh) { const int yy = e / (gx - 1), xx = e % (gx - 1) + 1; a = xx + yy * gx; b = a - 1; }
        else { const int e2 = e - nh; const int yy = e2 / gx + 1, xx = e2 % gx; a = xx + yy * gx; b = a - gx; }
        double w = c.depth_deform_reg;
        if (c.adaptive_deform > 0.0 && p.adaptive) {
          const double* aw = p.adaptive + (size_t)f * gx * gy;
          w = c.depth_deform_reg + fmax(aw[a], aw[b]) * c.adaptive_deform;
        }
        const int la = L.offD + a * L.k + comp, lb = L.offD + b * L.k + comp;
        const double va = pf[la], vb = pf[lb];
        const double aa = va < 0.0 ? -va : va, ab = vb < 0.0 ? -vb : vb;
        const bool useB = ab < aa;               // min(abs(this), abs(that)) = (that < this) ? that : this
        const double m = useB ? ab : aa;
        r = (va - vb) / m * w;
        double da = 1.0 / m, db = -1.0 / m;
        if (useB) db += -(va - vb) / (m * m) * (vb < 0.0 ? -1.0 : 1.0);
        else da += -(va - vb) / (m * m) * (va < 0.0 ? -1.0 : 1.0);
        el[0] = la; ed[0] = da * w; efr[0] = f; el[1] = lb; ed[1] = db * w; efr[1] = f; nent = 2;
        valid = true;
      } else if ((k -= rc.deform) < rc.spatial) {
        // paramsToResiduals (lib/DepthMapTransform.cpp:61-70) * spatialDeformReg
        r = pf[L.offS + k] * c.spatial_deform_reg; el[0] = L.offS + k; ed[0] = c.spatial_deform_reg; efr[0] = f; nent = 1; valid = true;
      } else {
        // TargetFocalCost (lib/PoseOptimizer.cpp:520-533), ScaledLoss(focalReg)
        const double sw = sqrt(c.focal_reg);
        r = (pf[6] - c.focal_target) * sw; el[0] = 6; ed[0] = sw; efr[0] = f; nent = 1; valid = true;
      }
    }
  } else if (id < rc.total) {
    // ParameterRegularizationCost (lib/PoseOptimizer.cpp:464-483) over in-range triplets (:1420-1426)
    const int k = id - rc.per_frame * p.N;
    const int f = k / 3, i = k % 3;
    const bool mine = MODE == EvalMode::MarkActive || (p.nranks <= 1) || (f % p.nranks == p.rank);
    if (mine && f >= first_frame && f < last_frame - 1 && p.in_range[f] && p.in_range[f + 1] && p.in_range[f + 2]) {
      const double sw = sqrt(c.position_reg);
      r = (x[(size_t)f * L.nf + i] - 2.0 * x[(size_t)(f + 1) * L.nf + i] + x[(size_t)(f + 2) * L.nf + i]) * sw;
      el[0] = i; ed[0] = sw; efr[0] = f; el[1] = i; ed[1] = -2.0 * sw; efr[1] = f + 1; el[2] = i; ed[2] = sw; efr[2] = f + 2; nent = 3;
      valid = true;
    }
  }
  if (valid) {
    cost = 0.5 * r * r;
    if (MODE == EvalMode::MarkActive) { for (int a = 0; a < nent; ++a) mask[(size_t)efr[a] * np + el[a]] = 1; }
    if (MODE == EvalMode::CostGrad || MODE == EvalMode::CostGradH) {
      for (int a = 0; a < nent; ++a) if (is_const_local(c, L, el[a])) ed[a] = 0.0;
      for (int a = 0; a < nent; ++a) {
        if (ed[a] == 0.0) continue;
        red_add(g + (size_t)efr[a] * np + el[a], ed[a] * r);
        if (MODE == EvalMode::CostGradH) for (int b = 0; b <= a; ++b) if (ed[b] != 0.0) add_h(p, H, efr[a], el[a], efr[b], el[b], ed[a] * ed[b]);
      }
    }
    if constexpr (MODE == EvalMode::Rows) {
      const int s = rows.slot[id];
      rows.r[s] = r; rows.rho[s] = r * r;
      if constexpr (JAC) {
        int E = 0;
        for (int a = 0; a < nent; ++a)
          if (!is_const_local(c, L, el[a])) { rows.col(s, E, rows.uperm[efr[a]] * L.nf + el[a], ed[a]); ++E; }
        rows.pad(s, E);
      }
    }
  }
  if (MODE != EvalMode::MarkActive && MODE != EvalMode::Rows) block_store_sum(cost, partial + blockIdx.x);
}

// --- scene-flow smoothness residual blocks (reference addSceneFlowSmoothnessLoss, lib/PoseOptimizer.cpp:1242-1339) ---
// Rows: r and J without the ScaledLoss weight w, rho = w |r|^2.
template <EvalMode MODE, bool JAC = false>
__global__ void __launch_bounds__(kTile) k_triplets(DevProblem p, const double* __restrict__ x, double* __restrict__ H, double* __restrict__ g,
                                                    double* __restrict__ partial, uint8_t* __restrict__ mask, RowArg<MODE> rows) {
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const int t = blockIdx.x;
  const int fc = p.trips.group_frames[p.trips.tile_group[t]];
  const bool mine = MODE == EvalMode::MarkActive || (p.nranks <= 1) || (fc % p.nranks == p.rank);
  double cost = 0.0;
  if ((int)threadIdx.x < p.trips.tile_count[t] && mine) {
    const float* rec = p.trips.records + (size_t)(p.trips.tile_begin[t] + threadIdx.x) * 10;
    Gather dg[3], sg[3];
    ObsIn o[3]; const double* pose[3]; double phi[3], D[3], u[3][2];
    for (int i = 0; i < 3; ++i) {
      o[i] = ObsIn{rec[3 * i], rec[3 * i + 1], rec[3 * i + 2]};
      gather_depth(c, o[i].ndcx, o[i].ndcy, dg[i]); gather_spatial(c, o[i].ndcx, o[i].ndcy, sg[i]);
      pose[i] = x + (size_t)(fc - 1 + i) * L.nf;
    }
    if (MODE == EvalMode::MarkActive) {
      for (int i = 0; i < 3; ++i) mark_frame(c, L, mask + (size_t)(fc - 1 + i) * L.npad, dg[i], sg[i]);
      if (c.intr_opt == RCVD_INTR_SHARED) mask[6] = 1;
      return;
    }
    for (int i = 0; i < 3; ++i) {
      phi[i] = (c.intr_opt == RCVD_INTR_SHARED) ? x[6] : (c.intr_opt == RCVD_INTR_PER_FRAME ? pose[i][6] : c.fixed_vfocal);
      D[i] = depth_value(c, L, dg[i], o[i].depth, pose[i]);
      warp_value(L, sg[i], pose[i], u[i]);
    }
    const double w = (double)rec[9], sw = sqrt(w);   // ScaledLoss(nullptr, w): rho' = w
    double r[3];
    if constexpr (MODE == EvalMode::Cost) {
      smooth_scene<false>(c, pose, phi, D, u, o, r, nullptr);
      cost = 0.5 * w * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    } else if constexpr (MODE == EvalMode::Rows) {
      const int fr[3] = {fc - 1, fc, fc + 1}; double Jl[JAC ? 90 : 1];
      smooth_scene<JAC>(c, pose, phi, D, u, o, r, JAC ? Jl : nullptr);
      store_rows<3, JAC>(p, rows, (size_t)(p.trips.tile_begin[t] + threadIdx.x), fr, rec, dg, sg, Jl, r, w * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]));
    } else {
      const int fr[3] = {fc - 1, fc, fc + 1}; double Jl[90];
      smooth_scene<true>(c, pose, phi, D, u, o, r, Jl);
      cost = 0.5 * w * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
      scatter_columns<3, MODE == EvalMode::CostGradH>(p, fr, rec, dg, sg, Jl, r, sw, H, g);
    }
  }
  if (MODE != EvalMode::MarkActive && MODE != EvalMode::Rows) block_store_sum(cost, partial + t);
}

// --- pairwise depth normalisation (normalizeDepth with normalizeDepthFromFirstFrame = false, lib/PoseOptimizer.cpp:1005-1095) ---
// One DisparityDissimilarityCost row per constraint (:425-462), r = 1 / max(D_a, 1e-6) - 1 / max(D_b, 1e-6), D the transformed depth
// of each end, over the depth-transform parameters of both frames; robustified as the static rows (robust_loss, sqrt(rho') corrector).
// max(D, eps) is Jet max, (D < eps) ? eps : D: a clamped end contributes no derivative.  With a Global transform every constraint of
// the tile touches the same 2k gradient and k (2k + 1) H entries (one pair): they are summed over the tile (warp shuffle, then shared
// memory) and leave the SM as one RED each.  Grid transforms scatter per constraint over the gathered nodes.
template <EvalMode MODE, bool JAC = false>
__global__ void __launch_bounds__(kTile) k_depth_pairs(DevProblem p, const double* __restrict__ x, double* __restrict__ H, double* __restrict__ g,
                                                       double* __restrict__ partial, uint8_t* __restrict__ mask, RowArg<MODE> rows) {
  const rcvd_config& c = p.cfg; const Layout& L = p.L;
  const int t = blockIdx.x, np = L.npad;
  const int pr = p.dpairs.tile_group[t];
  const int fr[2] = {p.dpairs.group_frames[2 * pr], p.dpairs.group_frames[2 * pr + 1]};
  const bool active = (int)threadIdx.x < p.dpairs.tile_count[t];
  const float* rec = p.dpairs.records + (size_t)(p.dpairs.tile_begin[t] + (active ? threadIdx.x : 0)) * 6;
  Gather dg[2];
  for (int s = 0; s < 2; ++s) {
    if (active) gather_depth(c, rec[3 * s], rec[3 * s + 1], dg[s]);
    else dg[s].n = 0;
  }
  if constexpr (MODE == EvalMode::MarkActive) {
    for (int s = 0; s < 2; ++s)
      for (int q = 0; q < dg[s].n; ++q)
        for (int j = 0; j < L.k; ++j) mask[(size_t)fr[s] * np + L.offD + dg[s].idx[q] * L.k + j] = 1;
    return;
  } else if constexpr (MODE == EvalMode::Rows) {
    if (!active) return;
    constexpr double eps = 1e-6;
    const double D0 = depth_value(c, L, dg[0], rec[2], x + (size_t)fr[0] * L.nf), D1 = depth_value(c, L, dg[1], rec[5], x + (size_t)fr[1] * L.nf);
    const bool c0 = D0 < eps, c1 = D1 < eps;
    const double r = 1.0 / (c0 ? eps : D0) - 1.0 / (c1 ? eps : D1);
    double rho0, rho1;
    robust_loss(c, r * r, rho0, rho1);
    const size_t slot = (size_t)(p.dpairs.tile_begin[t] + threadIdx.x);
    rows.r[slot] = r; rows.rho[slot] = rho0;
    if constexpr (JAC) {
      const double dr[2] = {c0 ? 0.0 : -1.0 / (D0 * D0), c1 ? 0.0 : 1.0 / (D1 * D1)};   // dr/dD of each end
      int E = 0;
      if (!c.fix_depth_xforms)
        for (int s = 0; s < 2; ++s) {
          const double src = (double)rec[3 * s + 2]; const int32_t base = rows.uperm[fr[s]] * L.nf + L.offD;
          for (int q = 0; q < dg[s].n; ++q) {
            const double w = dg[s].w[q];
            rows.col(slot, E++, base + dg[s].idx[q] * L.k, dr[s] * w * src);
            if (L.k == 2) rows.col(slot, E++, base + dg[s].idx[q] * 2 + 1, dr[s] * w);
          }
        }
      rows.pad(slot, E);
    }
  } else {
    double cost = 0.0, rs = 0.0, dr[2] = {0.0, 0.0};   // scaled residual and scaled dr/dD of each end (zero on idle threads)
    if (active) {
      constexpr double eps = 1e-6;
      const double D0 = depth_value(c, L, dg[0], rec[2], x + (size_t)fr[0] * L.nf), D1 = depth_value(c, L, dg[1], rec[5], x + (size_t)fr[1] * L.nf);
      const bool c0 = D0 < eps, c1 = D1 < eps;
      const double r = 1.0 / (c0 ? eps : D0) - 1.0 / (c1 ? eps : D1);
      double rho0, rho1;
      robust_loss(c, r * r, rho0, rho1);
      cost = 0.5 * rho0;
      const double sc = sqrt(rho1);
      rs = r * sc;
      dr[0] = c0 ? 0.0 : -sc / (D0 * D0);
      dr[1] = c1 ? 0.0 : sc / (D1 * D1);
    }
    if (MODE != EvalMode::Cost && !c.fix_depth_xforms) {
      constexpr bool WANT_H = MODE == EvalMode::CostGradH;
      if (c.depth_type == RCVD_DEPTH_GLOBAL) {
        // columns a = side * k + component (scale: dD/ds = src; shift: dD/do = 1); values: J^T r over a, then H(a, b), b <= a
        const int k = L.k, nc = 2 * k, nv = nc + (WANT_H ? nc * (nc + 1) / 2 : 0);
        double j[4];
        for (int s = 0; s < 2; ++s) { j[s * k] = dr[s] * (double)rec[3 * s + 2]; if (k == 2) j[s * k + 1] = dr[s]; }
        __shared__ double red[14][kTile / 32];
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        int i = 0;
        for (int a = 0; a < nc; ++a, ++i) { const double v = warp_sum(j[a] * rs); if (lane == 0) red[i][wid] = v; }
        if (WANT_H)
          for (int a = 0; a < nc; ++a)
            for (int b = 0; b <= a; ++b, ++i) { const double v = warp_sum(j[a] * j[b]); if (lane == 0) red[i][wid] = v; }
        __syncthreads();
        if ((int)threadIdx.x < nv) {
          i = threadIdx.x;
          double v = 0.0;
#pragma unroll
          for (int w = 0; w < kTile / 32; ++w) v += red[i][w];
          if (i < nc) red_add(g + (size_t)fr[i / k] * np + L.offD + i % k, v);
          else {
            int e = i - nc, a = 0;
            while (e > a) { e -= a + 1; ++a; }   // e-th entry of the lower triangle, row-major: (a, e)
            add_h(p, H, fr[a / k], L.offD + a % k, fr[e / k], L.offD + e % k, v);
          }
        }
      } else if (active) {
        int ef[64]; short el[64]; double ej[64];   // 2 ends x <= 16 nodes x k
        int E = 0;
        for (int s = 0; s < 2; ++s) {
          const double src = (double)rec[3 * s + 2];
          for (int q = 0; q < dg[s].n; ++q) {
            const double w = dg[s].w[q];
            ef[E] = fr[s]; el[E] = (short)(L.offD + dg[s].idx[q] * L.k); ej[E] = dr[s] * w * src; ++E;
            if (L.k == 2) { ef[E] = fr[s]; el[E] = (short)(L.offD + dg[s].idx[q] * 2 + 1); ej[E] = dr[s] * w; ++E; }
          }
        }
        for (int a = 0; a < E; ++a) {
          red_add(g + (size_t)ef[a] * np + el[a], ej[a] * rs);
          if (WANT_H) for (int b = 0; b <= a; ++b) add_h(p, H, ef[a], el[a], ef[b], el[b], ej[a] * ej[b]);
        }
      }
    }
    block_store_sum(cost, partial + t);
  }
}

// Final deterministic reduction of the per-block partial costs: out[slot] = sum(partial[0..n))
__global__ void __launch_bounds__(1024) k_reduce_partials(const double* __restrict__ partial, int n, double* __restrict__ out, int slot) {
  __shared__ double red[32];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += partial[i];
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (wid == 0) {
    double t = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.0;
    t = warp_sum(t);
    if (lane == 0) out[slot] = t;
  }
}

}  // namespace rcvd
