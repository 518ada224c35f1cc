// rcvd_api.cu -- host driver + C ABI (include/rcvd.h) of the H100 temporal-consistency solver.
//
// Replaces ceres::Solve as called from DepthVideoPoseOptimizer::poseOptimizationStep
// (reference lib/PoseOptimizer.cpp:954-962) and ::normalizeDepth (:1117-1125): Levenberg-
// Marquardt with Ceres' trust-region rules on the host, all arithmetic on the device.
// There is NO CPU fallback: without a CUDA device rcvd_problem_create fails.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <dlfcn.h>
#include <limits>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include <cub/device/device_segmented_sort.cuh>
#include "rcvd_eval.cuh"
#include "rcvd_linalg.cuh"
#include "rcvd_update.cuh"
#include "rcvd_plan.h"
#include "rcvd_cg.cuh"
#include "rcvd_selinv.cuh"
#include "rcvd_host.h"

using namespace rcvd;

static thread_local std::string g_err = "";
int set_err(int code, const char* fmt, ...) {
  char buf[512]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
  g_err = buf; return code;
}

// ---- NCCL through dlopen (plumbing only; the data path collective is one all-reduce) ----
namespace nccl {
typedef struct { char internal[128]; } UniqueId;
typedef void* Comm;
static void* lib = nullptr;
static int (*GetUniqueId)(UniqueId*) = nullptr;
static int (*CommInitRank)(Comm*, int, UniqueId, int) = nullptr;
static int (*AllReduce)(const void*, void*, size_t, int, int, Comm, cudaStream_t) = nullptr;
static int (*CommDestroy)(Comm) = nullptr;
static const char* (*GetErrorString)(int) = nullptr;
static int (*GroupStart)() = nullptr;
static int (*GroupEnd)() = nullptr;
static int (*Broadcast)(const void*, void*, size_t, int, int, Comm, cudaStream_t) = nullptr;
static int (*Reduce)(const void*, void*, size_t, int, int, int, Comm, cudaStream_t) = nullptr;
static bool load() {
  if (lib) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
  if (!lib) return false;
  GetUniqueId = (int (*)(UniqueId*))dlsym(lib, "ncclGetUniqueId");
  CommInitRank = (int (*)(Comm*, int, UniqueId, int))dlsym(lib, "ncclCommInitRank");
  AllReduce = (int (*)(const void*, void*, size_t, int, int, Comm, cudaStream_t))dlsym(lib, "ncclAllReduce");
  CommDestroy = (int (*)(Comm))dlsym(lib, "ncclCommDestroy");
  GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
  GroupStart = (int (*)())dlsym(lib, "ncclGroupStart"); GroupEnd = (int (*)())dlsym(lib, "ncclGroupEnd");
  Broadcast = (int (*)(const void*, void*, size_t, int, int, Comm, cudaStream_t))dlsym(lib, "ncclBroadcast");
  Reduce = (int (*)(const void*, void*, size_t, int, int, int, Comm, cudaStream_t))dlsym(lib, "ncclReduce");
  return GetUniqueId && CommInitRank && AllReduce && CommDestroy && GroupStart && GroupEnd && Broadcast && Reduce;
}
constexpr int kFloat64 = 8, kUint8 = 1, kSum = 0, kMax = 2;   // ncclFloat64, ncclUint8, ncclSum, ncclMax
}  // namespace nccl

// ---- small vector kernels of the LM loop ----
enum { SC_COST = 0, SC_CAND = 1, SC_GY = 2, SC_YHY = 3, SC_STEP2 = 4, SC_X2 = 5, SC_GMAX = 6, SC_GDOTD = 7, SC_DMAX = 8, SC_N = 16 };

__global__ void k_extract_diag(const double* __restrict__ H, double* __restrict__ diag, int N, int npad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * npad) return;
  const int f = i / npad, l = i % npad;
  diag[i] = H[(size_t)f * npad * npad + (size_t)l * npad + l];
}
__global__ void k_jacobi_scale(const double* __restrict__ diag, double* __restrict__ S, int n, int enable) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) S[i] = enable ? 1.0 / (1.0 + sqrt(diag[i])) : 1.0;
}
// lmdiag = clamp(S^2 diagH) (unless reuse); D2 = lmdiag / radius; gs = S g
__global__ void k_lm_prepare(const double* __restrict__ diagH, const double* __restrict__ S, const double* __restrict__ g, double* __restrict__ lmdiag,
                             double* __restrict__ D2, double* __restrict__ gs, int n, int reuse, double radius, double dmin, double dmax) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double s = S[i];
  double d = lmdiag[i];
  if (!reuse) { d = fmin(fmax(s * s * diagH[i], dmin), dmax); lmdiag[i] = d; }
  D2[i] = d / radius;
  gs[i] = s * g[i];
}
__global__ void k_mul(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ o, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] * b[i];
}
__device__ __forceinline__ double project_lb(const rcvd_config& c, const Layout& L, const uint8_t* in_range, int f, int l, double v) {
  if (c.depth_lower_bound && l >= L.offD && l < L.offS && ((l - L.offD) % L.k) == 0 && in_range[f]) return fmax(v, 0.0);
  return v;
}
// |x|^2 over active params and max-norm of the projected gradient step x - Plus(x, -g)
__global__ void __launch_bounds__(256) k_state_norms(rcvd_config cfg, Layout L, const uint8_t* __restrict__ in_range, const uint8_t* __restrict__ active,
                                                      const double* __restrict__ x, const double* __restrict__ g, double* __restrict__ scal, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double x2 = 0.0, gm = 0.0;
  if (i < N * L.nf) {
    const int f = i / L.nf, l = i % L.nf;
    const size_t v = (size_t)f * L.npad + l;
    if (active[v]) {
      x2 = x[i] * x[i];
      gm = fabs(x[i] - project_lb(cfg, L, in_range, f, l, x[i] - g[v]));
    }
  }
  x2 = warp_sum(x2);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) gm = fmax(gm, __shfl_xor_sync(0xffffffffu, gm, o));
  if ((threadIdx.x & 31) == 0) {
    red_add(scal + SC_X2, x2);
    atomicMax((unsigned long long*)(scal + SC_GMAX), (unsigned long long)__double_as_longlong(gm));
  }
}
__global__ void __launch_bounds__(256) k_dot2(const double* __restrict__ a, const double* __restrict__ b, const double* __restrict__ c,
                                               const double* __restrict__ d, int n, double* __restrict__ scal, int s0, int s1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double p = 0.0, q = 0.0;
  if (i < n) { p = a[i] * b[i]; q = c[i] * d[i]; }
  p = warp_sum(p); q = warp_sum(q);
  if ((threadIdx.x & 31) == 0) { red_add(scal + s0, p); red_add(scal + s1, q); }
}
__global__ void k_finalize_mask(rcvd_config cfg, Layout L, uint8_t* __restrict__ mask, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * L.npad) return;
  const int l = i % L.npad;
  if (l >= L.nf || is_const_local(cfg, L, l)) mask[i] = 0;
}
__global__ void k_project_state(rcvd_config cfg, Layout L, const uint8_t* __restrict__ in_range, double* __restrict__ x, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N * L.nf) x[i] = project_lb(cfg, L, in_range, i / L.nf, i % L.nf, x[i]);
}
__global__ void k_h_to_dense(const double* __restrict__ H, const HBlock* __restrict__ hb, int nblocks, double* __restrict__ out, int N, int nf, int npad, const int* __restrict__ uperm) {
  const int b = blockIdx.y;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nf * nf) return;
  const int i = e / nf, j = e % nf;
  const HBlock hbk = hb[b];
  if (hbk.r == hbk.c && j > i) return;
  const double v = H[(size_t)b * npad * npad + (size_t)i * npad + j];
  const size_t U = (size_t)N * nf;
  const int ur = uperm[hbk.r], uc = uperm[hbk.c];          // internal -> caller's frame order
  out[((size_t)ur * nf + i) * U + (size_t)uc * nf + j] = v;
  out[((size_t)uc * nf + j) * U + (size_t)ur * nf + i] = v;
}

// launch counters of enqueue_factor_solve by kernel path (rcvd_debug_linear_paths; include/rcvd_hooks.h lists the same order)
enum { LP_POTRF_SMEM = 0, LP_POTRF_PANEL, LP_TRSM_LL4, LP_TRSM_LL2, LP_TRSM_GEMM, LP_UPD_TMA1, LP_UPD_TMA2, LP_SUB_LEVEL, LP_SUB_FUSED,
       LP_TRINV, LP_OTHER, LP_UPD_TMA1_MULTI, LP_TRSM_STREAMED, LP_N };   // LP_UPD_TMA1_MULTI: k_update_tma<1> launches with fewer CTAs than
// items; LP_TRSM_STREAMED: the k_trsm_ll launches (either shape) that run beside their level's k_potrf_smem

// ---------------------------------------------------------------------------
// One constraint family: groups of `nframes` frames (a directed pair: 2, a triplet's centre: 1), each with a run of consecutive
// records of `width` floats, as the caller set them, and their tiled device copy (set_up_problem_data).
struct RecordSet {
  const int width, nframes;
  std::vector<int32_t> frames; std::vector<int64_t> offsets{0}; std::vector<float> records;
  RecordTiles dev = {}; int num_tiles = 0;
  const float* caller_records = nullptr;   // the device records in the caller's order (dev.records may be the run path's sorted copy)
  RecordSet(int width_, int nframes_) : width(width_), nframes(nframes_) {}
  int groups() const { return (int)offsets.size() - 1; }
  int64_t count() const { return offsets.back(); }
};

struct rcvd_problem {
  rcvd_config cfg; Layout L; int N = 0; int device = 0;
  cudaStream_t stream = nullptr;
  // host inputs (in_range all 1 and median all 1.0 from rcvd_problem_create on)
  std::vector<uint8_t> in_range; std::vector<double> median, adaptive;
  RecordSet pairs{6, 2}, trips{10, 1}, dpairs{6, 2};   // static-scene pairs, smoothness triplets, pairwise depth normalisation
  std::vector<int32_t> struct_pairs;   // global frame-pair graph (multi-GPU); empty -> local pairs
  int first_frame = 0, last_frame = -1;
  // device problem data
  int32_t* d_blk_of = nullptr; uint8_t *d_in_range = nullptr, *d_active = nullptr;
  double *d_median = nullptr, *d_adaptive = nullptr; float* d_scale_locs = nullptr; int nscale = 0;
  // state & vectors
  double *d_x = nullptr, *d_xc = nullptr, *d_xsave = nullptr;
  double *d_g = nullptr, *d_S = nullptr, *d_diagH = nullptr, *d_lmdiag = nullptr, *d_D2 = nullptr, *d_gs = nullptr, *d_rhs = nullptr, *d_ytmp = nullptr,
         *d_y = nullptr, *d_Sy = nullptr, *d_Hy = nullptr, *d_partial = nullptr, *d_scal = nullptr;
  double* h_scal = nullptr;   // pinned
  // d_partial holds one partial cost per CTA: the pair tiles from 0, the regulariser blocks from part_reg, the triplet tiles from
  // part_trip, the depth-pair tiles from part_dp; npartial in all
  int part_reg = 0, part_trip = 0, part_dp = 0, npartial = 0;
  // matrices
  double *d_H = nullptr, *d_Lb = nullptr, *d_T = nullptr, *d_invL = nullptr, *d_invT = nullptr;
  HBlock *d_hblocks = nullptr, *d_lblocks = nullptr; int* d_fail = nullptr;
  int* d_potrf_progress = nullptr;   // [N] tile columns of each diagonal block k_potrf_smem has published (read by the streamed k_trsm_ll)
  FactorKernels fk = {};              // the factorisation's kernel variants at this npad (allocate_storage)
  // the block-Cholesky plan (rcvd_plan.h) and its device copies
  FactorPlan plan;
  int *d_lvl_frames = nullptr; TrsmTask* d_trsm_tasks = nullptr; int2* d_upd_pairs = nullptr; SolveTask* d_fwd_tasks = nullptr;
  SubTask* d_sub_tasks = nullptr; int* d_sub_counters = nullptr; int* d_sub_need = nullptr;
  cudaGraphExec_t solve_graph = nullptr;
  bool structure_ready = false;
  // multi GPU
  int nranks = 1, rank = 0; nccl::Comm comm = nullptr;
  int64_t launches = 0, graph_launches = 0;
  int64_t pair_launches[3] = {0, 0, 0};   // rcvd_debug_pair_kernel_launches: CostGradH launches of k_pairs, k_accumulate_runs, k_accumulate_fast
  // The caller-visible state (N x nf, caller's frame order) is h_state whenever !structure_ready || state_dirty, and d_x otherwise:
  // drop_structure saves d_x to h_state before it invalidates the structure, ensure_ready uploads h_state when state_dirty.
  std::vector<double> h_state; bool state_dirty = true; bool overlap = true; int order_slack = 4;   // multiple elimination with degree slack 4 (measured at config 2: slack 1..5 -> 13.65 13.11 12.74 12.66 13.09 ms per iteration); -1: greedy minimum degree
  cudaStream_t side_stream = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  std::vector<cudaEvent_t> ev_side;   // per level, two each: recorded after the level's side-stream update launches (Level::join waits on them)
  cudaStream_t inv_stream = nullptr; cudaEvent_t ev_inv_join = nullptr;   // k_trinv, off the critical path and off the side stream's
  double *d_g2 = nullptr, *d_delta = nullptr; int* h_fail = nullptr;
  cudaEvent_t ev[8] = {nullptr};
  std::vector<void*> allocs;
  // kernel-class profiling (rcvd_debug_profile_linear): when set, enqueue_factor_solve records one event per launch
  std::vector<std::pair<int, cudaEvent_t>>* prof = nullptr;
  bool eval_only = false;   // test / bench hook: only rcvd_evaluate is used (no H, no factor storage)
  bool records_sorted = false;   // run path of the accumulate kernel (bilinear depth grid): records sorted by cell pair
  int fast_path = 1;             // rcvd_debug_set_fast_path
  bool dist_enabled = true, graph_warm = false, force_full_H = false;
  // the frames this rank factors per level, the L blocks k_load_factor writes (FactorPlan::load_lblocks), the H blocks this rank owns,
  // internal -> caller's frame ids
  int *d_lvl_own = nullptr, *d_load_lblocks = nullptr, *d_own_hblocks = nullptr, *d_uperm = nullptr;
  // TMA-fed persistent update kernel (rcvd_update.cuh)
  // d_upd_items: FactorPlan::upd_items_cost, then upd_items; upd_order (rcvd_debug_set_update_order) picks the list the launches read
  UpdItem* d_upd_items = nullptr; CUtensorMap tmapT; int num_sms = 0, upd_ipc = 0, upd_order = 1;   // upd_ipc: items-per-CTA cap of the one-team launches (0: none)
  std::vector<double> level_ms;   // last rcvd_debug_profile_linear: per level x kernel class
  // test hooks (rcvd_debug_factor_dense, rcvd_debug_linear_paths): whether a factorisation has run, per-kernel-path launch counters
  // (enqueue_factor_solve counts, graph replays add graph_paths)
  bool factored = false;
  int64_t paths[LP_N] = {0}, graph_paths[LP_N] = {0};
  // The linear solver build_structure picked for the plan (rcvd_cg.cuh): conjugate gradients when the block Cholesky's storage
  // exceeds factor_budget (-1: cholesky_budget of the device's total memory; rcvd_debug_set_factor_budget), the block Cholesky otherwise
  bool use_cg = false; int64_t factor_budget = -1; uint64_t total_mem = 0;
  LinearStorage storage = {}; int64_t linear_bytes = 0;   // both paths' needs for the plan; what allocate_storage allocated for the chosen one
  double cg_eta = kCgEta;                                  // rcvd_debug_set_cg_tolerance
  double *d_cg_r = nullptr, *d_cg_z = nullptr, *d_cg_p = nullptr, *d_cg_q = nullptr, *d_cg_slots = nullptr, *d_cg_part = nullptr;
  int *d_cg_frames = nullptr, *d_cg_off = nullptr, *d_cg_ids = nullptr; CgState* d_cg = nullptr;
  // CG iterations of the solves since the last rcvd_solve began (rcvd_problem_linear_info), and of the last solve alone
  int64_t cg_iterations = 0; int cg_max = 0, cg_capped = 0, cg_steps = 0, cg_last = 0;
  // rcvd_covariance (rcvd_selinv.cuh): the selected inversion's task lists, built at the first call on a structure and dropped with it;
  // launches of its kernels (product, trmm, pivots, gather, scale) and the last call's phase times (factorisation, selected inversion,
  // gather, ms)
  bool sel_ready = false; SelPlan sel;
  SelTile* d_sel_tiles = nullptr; SelOp* d_sel_ops = nullptr; SelTrmm* d_sel_trmm = nullptr; int *d_sel_row_off = nullptr, *d_sel_row_blk = nullptr;
  int64_t sel_launches[5] = {0}; double sel_ms[3] = {0.0, 0.0, 0.0};
  rcvd_problem() {}
};

// Every kernel this file runs for a handle is launched here, and counted in p->launches (rcvd_launch_count).
template <class... Params, class... Args>
static int launch(rcvd_problem* p, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, Args... args) {
  if (int rc = launch_kernel(kernel, grid, block, smem, s, pdl, args...)) return rc;
  p->launches += 1;
  return RCVD_OK;
}

template <class T> static int dalloc(rcvd_problem* p, T** ptr, size_t count) {
  *ptr = nullptr;
  if (count == 0) count = 1;
  // stream-ordered pool allocation: the reference calls the solver once per schedule step, so a handle's
  // gigabytes of factor storage are recycled from the pool instead of paying cudaMalloc/cudaFree per call
  cudaError_t e = cudaMallocAsync((void**)ptr, count * sizeof(T), p->stream);
  if (e != cudaSuccess) return set_err(RCVD_ERR_CUDA, "cudaMallocAsync(%zu bytes) failed: %s", count * sizeof(T), cudaGetErrorString(e));
  p->allocs.push_back(*ptr);
  return RCVD_OK;
}
template <class T> static int upload(rcvd_problem* p, T** ptr, const std::vector<T>& v) {
  int rc = dalloc(p, ptr, v.size()); if (rc) return rc;
  if (!v.empty()) CK(cudaMemcpyAsync(*ptr, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, p->stream));
  return RCVD_OK;
}
// Frame-major vectors between the caller's frame order and the internal one (internal frame i is the caller's frame uperm[i]): `count`
// elements of each frame, frames `src_stride` / `dst_stride` elements apart.  frames_to_internal fills the rest of each row with `pad`.
template <class T> static std::vector<T> frames_to_internal(const std::vector<int>& uperm, const T* src, size_t src_stride, size_t dst_stride, size_t count, T pad = T()) {
  std::vector<T> out(uperm.size() * dst_stride, pad);
  for (size_t i = 0; i < uperm.size(); ++i) std::copy_n(src + (size_t)uperm[i] * src_stride, count, out.begin() + i * dst_stride);
  return out;
}
template <class T> static void frames_to_caller(const std::vector<int>& uperm, const T* src, size_t src_stride, T* dst, size_t dst_stride, size_t count) {
  for (size_t i = 0; i < uperm.size(); ++i) std::copy_n(src + i * src_stride, count, dst + (size_t)uperm[i] * dst_stride);
}
// A device vector of src_stride doubles per internal frame -> dst, nf per frame in the caller's order.
static int download_frames(rcvd_problem* p, double* dst, const double* src, int src_stride) {
  std::vector<double> tmp((size_t)p->N * src_stride);
  CK(cudaMemcpyAsync(tmp.data(), src, tmp.size() * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  CK(cudaStreamSynchronize(p->stream));
  frames_to_caller(p->plan.uperm, tmp.data(), src_stride, dst, p->L.nf, p->L.nf);
  return RCVD_OK;
}
// The factor+solve graph captures the switches of enqueue_factor_solve and the device buffers: it goes when either changes.
static void drop_graph(rcvd_problem* p) {
  if (p->solve_graph) { cudaGraphExecDestroy(p->solve_graph); p->solve_graph = nullptr; }
}
// Every setter of something build_structure reads calls this after its own checks; the state survives (see rcvd_problem).
static int drop_structure(rcvd_problem* p) {
  if (p->structure_ready && !p->state_dirty) {
    SET_DEVICE(p->device);
    if (int rc = download_frames(p, p->h_state.data(), p->d_x, p->L.nf)) return rc;
  }
  p->state_dirty = true; p->structure_ready = false;
  return RCVD_OK;
}
static void free_all(rcvd_problem* p) {
  drop_graph(p);
  if (p->side_stream) cudaStreamSynchronize(p->side_stream);
  if (p->inv_stream) cudaStreamSynchronize(p->inv_stream);
  for (void* q : p->allocs) cudaFreeAsync(q, p->stream);
  p->allocs.clear();
  if (p->stream) cudaStreamSynchronize(p->stream);
  if (p->h_scal) { cudaFreeHost(p->h_scal); p->h_scal = nullptr; }
  p->structure_ready = false; p->factored = false; p->sel_ready = false;
}

static DevProblem dev_problem(const rcvd_problem* p) {
  DevProblem d; d.cfg = p->cfg; d.L = p->L; d.N = p->N;
  d.pairs = p->pairs.dev; d.trips = p->trips.dev; d.dpairs = p->dpairs.dev;
  d.blk_of = p->d_blk_of; d.in_range = p->d_in_range; d.median = p->d_median;
  d.adaptive = p->adaptive.empty() ? nullptr : p->d_adaptive; d.scale_locs = p->d_scale_locs;
  d.rank = p->rank; d.nranks = p->nranks;
  return d;
}

// Enqueues the four residual families on the main stream in mode MODE: pair constraints (the one place that chooses their
// kernel), regulariser rows, smoothness triplets, depth-normalisation pairs.  Their per-block partial costs fill d_partial in that
// order; MarkActive marks d_active instead.
template <EvalMode MODE>
static int enqueue_residuals(rcvd_problem* p, const double* x, double* g) {
  const DevProblem d = dev_problem(p);
  const RegCounts rcn = reg_counts(p->cfg, p->L, p->N, p->nscale);
  const int regblocks = p->part_trip - p->part_reg, ntiles = p->pairs.num_tiles;
  cudaStream_t st = p->stream; double* part = p->d_partial; int rc;
  if (ntiles > 0) {
    const bool tc = MODE == EvalMode::CostGradH && p->fast_path != 0;   // a tensor-core kernel (rcvd_debug_set_fast_path)
    int which = 0;
    if (tc && p->fast_path == 1 && p->records_sorted) { which = 1; rc = launch(p, k_accumulate_runs, ntiles, kTile, kRunSmem, st, false, d, x, p->d_H, g, part); }
    else if (tc && fast_path_ok(p->cfg, p->L)) { which = 2; rc = launch(p, k_accumulate_fast, ntiles, kTile, kFastSmem, st, false, d, x, p->d_H, g, part); }
    else rc = launch(p, k_pairs<MODE>, ntiles, kTile, 0, st, false, d, x, p->d_H, g, part, p->d_active, NoRows{});
    if (rc) return rc;
    if (MODE == EvalMode::CostGradH) p->pair_launches[which] += 1;
  }
  if (regblocks > 0 && (rc = launch(p, k_regularisers<MODE>, regblocks, 128, 0, st, false, d, rcn, x, p->d_H, g, part + p->part_reg, p->d_active,
                                    p->first_frame, p->last_frame, NoRows{}))) return rc;
  if (p->trips.num_tiles > 0 && (rc = launch(p, k_triplets<MODE>, p->trips.num_tiles, kTile, 0, st, false, d, x, p->d_H, g, part + p->part_trip, p->d_active, NoRows{}))) return rc;
  if (p->dpairs.num_tiles > 0 && (rc = launch(p, k_depth_pairs<MODE>, p->dpairs.num_tiles, kTile, 0, st, false, d, x, p->d_H, g, part + p->part_dp, p->d_active, NoRows{}))) return rc;
  return RCVD_OK;
}

// ---- structure: the plan on the device, the problem data, the storage ----
#define UP(ptr, vec) if ((rc = upload(p, &(ptr), vec))) return rc
#define DA(ptr, n) if ((rc = dalloc(p, &(ptr), (n)))) return rc
static int upload_plan(rcvd_problem* p) {
  const FactorPlan& pl = p->plan; int rc;
  UP(p->d_blk_of, pl.blk_of); UP(p->d_hblocks, pl.hblocks); UP(p->d_lblocks, pl.lblocks); UP(p->d_lvl_frames, pl.lvl_frames); UP(p->d_lvl_own, pl.lvl_own);
  UP(p->d_load_lblocks, pl.load_lblocks); UP(p->d_own_hblocks, pl.own_hblocks); UP(p->d_uperm, pl.uperm);
  UP(p->d_trsm_tasks, pl.trsm_tasks); UP(p->d_upd_pairs, pl.upd_pairs);
  UP(p->d_sub_tasks, pl.sub_tasks); UP(p->d_sub_need, pl.sub_need); DA(p->d_sub_counters, (size_t)4 * p->N + 4);
  UP(p->d_fwd_tasks, pl.fwd_tasks);
  { std::vector<UpdItem> both(pl.upd_items_cost); both.insert(both.end(), pl.upd_items.begin(), pl.upd_items.end());
    UP(p->d_upd_items, both); }
  return RCVD_OK;
}

// A family's records, its group frames in internal frame order and its tiles (<= kTile records of one group each) on the device.
// Triplet centres pass through iperm like pair frames, and k_triplets also reads the neighbours fc - 1 and fc + 1: that holds
// because make_factor_plan keeps the caller's frame order (iperm the identity) whenever there are triplets.
static int upload_record_set(rcvd_problem* p, RecordSet& s) {
  std::vector<int32_t> frames(s.frames.size()), tile_group, tile_count; std::vector<int64_t> tile_begin;
  for (size_t i = 0; i < frames.size(); ++i) frames[i] = p->plan.iperm[s.frames[i]];
  for (int i = 0; i < s.groups(); ++i)
    for (int64_t b = s.offsets[i]; b < s.offsets[i + 1]; b += kTile) { tile_group.push_back(i); tile_begin.push_back(b); tile_count.push_back((int32_t)std::min<int64_t>(kTile, s.offsets[i + 1] - b)); }
  s.num_tiles = (int)tile_group.size();
  float* rec; int32_t *fr, *tg, *tn; int64_t* tb; int rc;
  UP(rec, s.records); UP(fr, frames); UP(tg, tile_group); UP(tb, tile_begin); UP(tn, tile_count);
  s.dev = RecordTiles{rec, fr, tg, tb, tn}; s.caller_records = rec;
  return RCVD_OK;
}

// the three families on the device, the record sort of the run path, the per-frame inputs in internal frame order, the scale
// lattice, the layout of the partial costs
static int set_up_problem_data(rcvd_problem* p) {
  const int N = p->N; const Layout& L = p->L; const std::vector<int>& uperm = p->plan.uperm; int rc;
  for (RecordSet* s : {&p->pairs, &p->trips, &p->dpairs}) if ((rc = upload_record_set(p, *s))) return rc;
  p->records_sorted = false;
  if (run_path_ok(p->cfg, L) && p->pairs.count() > 0 && p->pairs.count() < (int64_t)0x7fffffff) {
    // run path of the accumulate kernel: the records of every pair sorted by (source cell, target cell) -- device segmented sort by pair
    const long long n = p->pairs.count();
    unsigned *d_k0 = nullptr, *d_k1 = nullptr; int *d_i0 = nullptr, *d_i1 = nullptr; float* d_sorted = nullptr; int64_t* d_off = nullptr; void* d_tmp = nullptr;
    if ((rc = dalloc(p, &d_k0, (size_t)n)) || (rc = dalloc(p, &d_k1, (size_t)n)) || (rc = dalloc(p, &d_i0, (size_t)n)) || (rc = dalloc(p, &d_i1, (size_t)n)) || (rc = dalloc(p, &d_sorted, (size_t)n * 6)) ||
        (rc = upload(p, &d_off, p->pairs.offsets))) return rc;
    if ((rc = launch(p, k_record_keys, (unsigned)((n + 255) / 256), 256, 0, p->stream, false, p->cfg, p->pairs.dev.records, n, d_k0, d_i0))) return rc;
    size_t tmp_bytes = 0;
    CK(cub::DeviceSegmentedSort::SortPairs(nullptr, tmp_bytes, d_k0, d_k1, d_i0, d_i1, (int)n, p->pairs.groups(), d_off, d_off + 1, p->stream));
    CK(cudaMallocAsync(&d_tmp, std::max<size_t>(tmp_bytes, 16), p->stream));
    CK(cub::DeviceSegmentedSort::SortPairs(d_tmp, tmp_bytes, d_k0, d_k1, d_i0, d_i1, (int)n, p->pairs.groups(), d_off, d_off + 1, p->stream));
    if ((rc = launch(p, k_gather_records, (unsigned)((n * 6 + 255) / 256), 256, 0, p->stream, false, p->pairs.dev.records, d_i1, n, d_sorted))) return rc;
    CK(cudaFreeAsync(d_tmp, p->stream));
    CK(cudaGetLastError());
    p->pairs.dev.records = d_sorted; p->records_sorted = true;      // (the unsorted copy stays for rcvd_evaluate_rows; it and the sort buffers go back to the pool with the handle's other allocations)
  }
  UP(p->d_in_range, frames_to_internal(uperm, p->in_range.data(), 1, 1, 1));
  UP(p->d_median, frames_to_internal(uperm, p->median.data(), 1, 1, 1));
  if (!p->adaptive.empty()) {
    const size_t G = p->adaptive.size() / N;
    UP(p->d_adaptive, frames_to_internal(uperm, p->adaptive.data(), G, G, G));
  }
  {
    // scale-regulariser lattice in float32, lib/PoseOptimizer.cpp:1382-1385
    std::vector<float> locs; const int gx = p->cfg.scale_grid_x, gy = p->cfg.scale_grid_y;
    for (int y = 0; y < gy; ++y) for (int x = 0; x < gx; ++x) {
      // host code is built without -mfma, so these float ops are not contracted
      const float fx = -1.f + 2.f * x / (gx - 1);
      const float fy = -1.f + 2.f * y / (gy - 1);
      locs.push_back(fx); locs.push_back(fy);
    }
    p->nscale = (int)(locs.size() / 2);
    UP(p->d_scale_locs, locs);
  }
  p->first_frame = 0; p->last_frame = -1;
  { bool any = false; for (int f = 0; f < N; ++f) if (p->in_range[f]) { if (!any) { p->first_frame = f; any = true; } p->last_frame = f; } }
  p->part_reg = p->pairs.num_tiles;
  p->part_trip = p->part_reg + (reg_counts(p->cfg, L, N, p->nscale).total + 127) / 128;
  p->part_dp = p->part_trip + p->trips.num_tiles;
  p->npartial = p->part_dp + p->dpairs.num_tiles;
  return RCVD_OK;
}
#undef UP

// state, vectors and matrices, the TMA map of the factor blocks, the active-parameter mask, the kernels' shared-memory limits
static int allocate_storage(rcvd_problem* p) {
  const int N = p->N; const Layout& L = p->L; const int npad = L.npad, nLoff = p->plan.nLoff; const size_t bs = (size_t)npad * npad; int rc;
  const size_t Upad = (size_t)N * npad, U = (size_t)N * L.nf;
  DA(p->d_x, U); DA(p->d_xc, U); DA(p->d_xsave, U);
  DA(p->d_g, 2 * Upad + 8); p->d_diagH = p->d_g + Upad + 8;   // [gradient | 8 scalars | diag H]: one packed all-reduce at N > 1
  DA(p->d_S, Upad); DA(p->d_lmdiag, Upad); DA(p->d_D2, Upad); DA(p->d_gs, Upad); DA(p->d_rhs, Upad);
  DA(p->d_g2, Upad + 8); DA(p->d_delta, Upad);
  DA(p->d_ytmp, Upad); DA(p->d_y, Upad); DA(p->d_Sy, Upad); DA(p->d_Hy, Upad); DA(p->d_scal, SC_N); DA(p->d_active, Upad); DA(p->d_fail, 1);
  DA(p->d_potrf_progress, (size_t)N);
  DA(p->d_partial, (size_t)p->npartial);
  // the linear solver's storage, counted in linear_bytes (linear_storage restates it from the plan)
  p->linear_bytes = 0;
#define LA(ptr, n) do { DA(ptr, n); p->linear_bytes += (int64_t)std::max<size_t>((n), 1) * sizeof(*(ptr)); } while (0)
  if (p->eval_only) { DA(p->d_H, 1); DA(p->d_Lb, 1); DA(p->d_T, 1); DA(p->d_invL, 1); DA(p->d_invT, 1); }   // cost / gradient evaluations only: no matrices
  else if (p->use_cg) {
    // H, the N damped diagonal blocks and their inverses: no fill blocks, no off-diagonal factor blocks
    const size_t nH = p->plan.hblocks.size();
    LA(p->d_H, nH * bs); LA(p->d_Lb, (size_t)N * bs); LA(p->d_invL, (size_t)N * bs); LA(p->d_invT, (size_t)N * npad * 16);
    p->d_T = nullptr;
    LA(p->d_cg_slots, 2 * nH * npad); LA(p->d_cg_r, Upad); LA(p->d_cg_z, Upad); LA(p->d_cg_p, Upad); LA(p->d_cg_q, Upad);
    LA(p->d_cg_part, (size_t)cg_partials(N)); LA(p->d_cg, 1);
    std::vector<int> off, ids, frames(N);
    cg_slot_lists(p->plan, N, off, ids);
    for (int f = 0; f < N; ++f) frames[f] = f;
    if ((rc = upload(p, &p->d_cg_off, off)) || (rc = upload(p, &p->d_cg_ids, ids)) || (rc = upload(p, &p->d_cg_frames, frames))) return rc;
    p->linear_bytes += (int64_t)(off.size() + ids.size() + frames.size()) * sizeof(int);
  } else {
    LA(p->d_H, p->plan.hblocks.size() * bs); LA(p->d_Lb, (size_t)(N + nLoff) * bs); LA(p->d_T, (size_t)std::max(nLoff, 1) * bs);
    LA(p->d_invL, (size_t)N * bs); LA(p->d_invT, (size_t)N * npad * 16);
  }
#undef LA
#undef DA
  if (!p->use_cg) {
    // 2-D TMA view of the T buffer (off-diagonal factor blocks X_rk, row-major): inner = k, outer = block * npad + row, box [rb][16], 128-B swizzle
    bool encoded = false;
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                 CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr; cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && fn && qres == cudaDriverEntryPointSuccess) {
      const cuuint64_t gdim[2] = {(cuuint64_t)npad, (cuuint64_t)std::max(nLoff, 1) * npad};
      const cuuint64_t gstr[1] = {(cuuint64_t)npad * sizeof(double)};
      const cuuint32_t box[2] = {16u, (cuuint32_t)p->plan.upd_rb};
      const cuuint32_t estr[2] = {1u, 1u};
      const CUresult r = ((EncodeFn)fn)(&p->tmapT, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, p->d_T, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      encoded = (r == CUDA_SUCCESS);
    }
    cudaGetLastError();
    if (!encoded) return set_err(RCVD_ERR_CUDA, "cuTensorMapEncodeTiled unavailable or failed: the TMA update kernel cannot run");
    CK(cudaFuncSetAttribute(k_update_tma<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)upd_smem_bytes(p->plan.upd_rb, 1)));
    CK(cudaFuncSetAttribute(k_update_tma<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)upd_smem_bytes(p->plan.upd_rb, 2)));
  }
  CK(cudaMallocHost((void**)&p->h_scal, (SC_N + 2) * sizeof(double)));
  p->h_fail = (int*)(p->h_scal + SC_N);
  CK(cudaMemsetAsync(p->d_x, 0, U * sizeof(double), p->stream));
  CK(cudaMemsetAsync(p->d_lmdiag, 0, Upad * sizeof(double), p->stream));
  CK(cudaMemsetAsync(p->d_S, 0, Upad * sizeof(double), p->stream));
  // active mask
  CK(cudaMemsetAsync(p->d_active, 0, Upad, p->stream));
  if ((rc = enqueue_residuals<EvalMode::MarkActive>(p, p->d_x, nullptr))) return rc;
  if ((rc = launch(p, k_finalize_mask, (int)((Upad + 255) / 256), 256, 0, p->stream, false, p->cfg, L, p->d_active, N))) return rc;
  if (p->nranks > 1) {   // the parameter set of the program is the union over the ranks' constraint shards (norms and stopping tests must agree on every rank)
    const int r = nccl::AllReduce(p->d_active, p->d_active, Upad, nccl::kUint8, nccl::kMax, p->comm, p->stream);
    if (r != 0) return set_err(RCVD_ERR_NCCL, "ncclAllReduce(active mask) failed");
  }
  // kernels that need > 48 KB dynamic smem
  FactorKernels& fk = p->fk = factor_kernels(npad);
  if (fk.trinv_bytes > kMaxDynSmem) return set_err(RCVD_ERR_INVALID, "frame block too large for the panel-inverse kernel (npad=%d)", npad);
  CK(cudaFuncSetAttribute(k_trinv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fk.trinv_bytes));
  CK(cudaFuncSetAttribute(k_accumulate_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmem));
  CK(cudaFuncSetAttribute(k_accumulate_runs, cudaFuncAttributeMaxDynamicSharedMemorySize, kRunSmem));
  if (fk.trsm_ll) {
    CK(cudaFuncSetAttribute(k_trsm_ll<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fk.trsm_ll2_bytes));
    CK(cudaFuncSetAttribute(k_trsm_ll<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fk.trsm_ll2_bytes));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fk.trsm2_ctas_per_sm, k_trsm_ll<2, true>, 128, fk.trsm_ll2_bytes));
  }
  if (fk.trsm_ll4) {
    CK(cudaFuncSetAttribute(k_trsm_ll<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fk.trsm_ll4_bytes));
    CK(cudaFuncSetAttribute(k_trsm_ll<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fk.trsm_ll4_bytes));
  }
  if (fk.potrf_smem) CK(cudaFuncSetAttribute(k_potrf_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fk.potrf_bytes));
  return RCVD_OK;
}

static int build_structure(rcvd_problem* p) {
  if (p->nranks > 1 && !p->dpairs.frames.empty()) return set_err(RCVD_ERR_INVALID, "depth-normalisation pairs are not sharded: they need a single-GPU problem (nranks = 1)");
  free_all(p);
  CK(cudaSetDevice(p->device));
  // the frame graph: static pairs (or the global structure of a sharded problem) and the depth-normalisation pairs
  std::vector<int32_t> graph = p->struct_pairs.empty() ? p->pairs.frames : p->struct_pairs;
  graph.insert(graph.end(), p->dpairs.frames.begin(), p->dpairs.frames.end());
  if (const char* e = make_factor_plan(p->plan, p->cfg, graph, p->trips.frames, p->order_slack, p->nranks, p->rank, p->dist_enabled, p->num_sms))
    return set_err(RCVD_ERR_INVALID, "%s", e);
  // The solver: the block Cholesky while its storage fits the budget; conjugate gradients beyond it, on one GPU (the distributed
  // factorisation of nranks > 1 spreads the factor over the ranks instead)
  p->storage = linear_storage(p->plan, p->N, p->L.npad);
  p->use_cg = p->nranks == 1 && !p->eval_only && p->storage.cholesky > (p->factor_budget >= 0 ? p->factor_budget : cholesky_budget(p->total_mem));
  while (p->ev_side.size() < 2 * p->plan.levels.size()) { cudaEvent_t e; CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); p->ev_side.push_back(e); }
  int rc;
  if ((rc = upload_plan(p)) || (rc = set_up_problem_data(p)) || (rc = allocate_storage(p))) return rc;
  CK(cudaStreamSynchronize(p->stream));
  p->structure_ready = true;
  return RCVD_OK;
}

static int allreduce(rcvd_problem* p, double* buf, size_t count) {
  if (p->nranks <= 1) return RCVD_OK;
  const int r = nccl::AllReduce(buf, buf, count, nccl::kFloat64, nccl::kSum, p->comm, p->stream);
  if (r != 0) return set_err(RCVD_ERR_NCCL, "ncclAllReduce failed: %s", nccl::GetErrorString ? nccl::GetErrorString(r) : "?");
  return RCVD_OK;
}
// One fused NCCL launch: for every rank q, segs[q] = (first, count) in units of `unit` doubles of `base` is broadcast from q (bcast) or
// summed onto q (!bcast), in place.  Every rank passes identical segments.
struct Seg { size_t first, count; };
static int grouped(rcvd_problem* p, double* base, size_t unit, const std::vector<Seg>& segs, bool bcast) {
  int r = nccl::GroupStart();
  for (size_t i = 0; i < segs.size() && r == 0; ++i) {
    if (segs[i].count == 0) continue;
    const int root = (int)(i % (size_t)p->nranks);
    double* ptr = base + segs[i].first * unit;
    r = bcast ? nccl::Broadcast(ptr, ptr, segs[i].count * unit, nccl::kFloat64, root, p->comm, p->stream)
              : nccl::Reduce(ptr, ptr, segs[i].count * unit, nccl::kFloat64, nccl::kSum, root, p->comm, p->stream);
  }
  const int r2 = nccl::GroupEnd();
  if (r == 0) r = r2;
  if (r != 0) return set_err(RCVD_ERR_NCCL, "grouped NCCL %s failed: %s", bcast ? "broadcast" : "reduce", nccl::GetErrorString ? nccl::GetErrorString(r) : "?");
  return RCVD_OK;
}

// Enqueues factorisation of (S H S + D2) and the solve y = A^{-1} gs on p->stream.
//
// Two-stream schedule (fork/join inside the captured graph): the deferred update passes of level l (U2) run on `side` concurrently
// with the later levels on `st`; the late passes (U1) of level Level::join are the first main-stream work that touches one of their
// targets, and wait for them there (the side stream runs in order: one wait covers every earlier side launch).  The explicit
// inverses run on a third stream, `inv`: on `side` they would hold back the next update launch by a k_trinv.
struct FactorSolve {
  enum { P_LOAD = 0, P_POTRF, P_TRINV, P_TRSM, P_GEMM, P_SOLVE };   // kernel classes of rcvd_debug_profile_linear
  rcvd_problem* p; const FactorPlan& pl; const FactorKernels& fk; const int N, npad, strips; cudaStream_t st, side, inv;
  int prof_level = 0;
  bool side_used = false, inv_used = false;   // work was enqueued on `side` / on `inv` since the main stream last waited for it
  int side_joined = -1;                        // the main stream has waited for the side launches (2 * level + launch) up to this one

  explicit FactorSolve(rcvd_problem* p_)
      : p(p_), pl(p_->plan), fk(p_->fk), N(p_->N), npad(p_->L.npad), strips((npad + kTrsmStrip - 1) / kTrsmStrip), st(p_->stream), side(p_->side_stream),
        inv(p_->inv_stream) {}

  void mark(int cls) {   // profiling mode only (single stream, not captured)
    if (!p->prof) return;
    cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, st); p->prof->push_back({cls < 0 ? cls : (cls | (prof_level << 8)), e});
  }
  // every kernel of the factorisation and the solve is launched here and also counted in p->paths[path]
  template <class... Params, class... Args>
  int launch(int path, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, Args... args) {
    if (int rc = ::launch(p, kernel, grid, block, smem, s, pdl, args...)) return rc;
    p->paths[path]++;
    return RCVD_OK;
  }
  // `waiter` waits for the work enqueued on `from` so far
  int wait(cudaStream_t waiter, cudaStream_t from, cudaEvent_t e) {
    CK(cudaEventRecord(e, from)); CK(cudaStreamWaitEvent(waiter, e, 0));
    return RCVD_OK;
  }
  // the main stream waits for `side` (every side launch of the levels before `level`) and `inv`
  int join_all(int level) {
    if (side_used) { if (int rc = wait(st, side, p->ev_join)) return rc; side_joined = 2 * level - 1; }
    if (inv_used) { if (int rc = wait(st, inv, p->ev_inv_join)) return rc; inv_used = false; }
    return RCVD_OK;
  }

  // A level's TRSM launch that is a single wave (the narrow levels) is streamed behind its k_potrf_smem (see trsm).
  bool trsm_deep(const Level& v) const { return strips * v.ntrsm <= p->num_sms && fk.trsm_ll4; }
  bool streamed(const Level& v) const {
    return fk.trsm_ll && v.nown > 0 && v.ntrsm > 0 && fk.potrf_smem && strips * v.ntrsm <= (trsm_deep(v) ? 1 : fk.trsm2_ctas_per_sm) * p->num_sms;
  }

  // the Cholesky of the level's diagonal blocks
  int factor_diagonal(const int* frames, int nfr, bool pdl) {
    if (fk.potrf_smem)
      return launch(LP_POTRF_SMEM, k_potrf_smem, dim3(nfr), dim3(kPotrfSmemThreads), fk.potrf_bytes, st, pdl, p->d_Lb, p->d_invT, frames, npad,
                    p->d_fail, p->d_potrf_progress);
    // large blocks: 16-wide panels, panel factor on one CTA per frame, trailing update on the whole machine
    for (int jb = 0; jb < npad / 16; ++jb) {
      if (int rc = launch(LP_POTRF_PANEL, k_potrf_panel, dim3(nfr), dim3(kPotrfThreads), 0, st, false, p->d_Lb, p->d_invT, frames, npad, jb, p->d_fail)) return rc;
      const int m = npad - (jb + 1) * 16, n64 = (m + 63) / 64;
      if (m > 0) { if (int rc = launch(LP_OTHER, k_potrf_trail, dim3(n64 * (n64 + 1) / 2, nfr), dim3(128), 0, st, false, p->d_Lb, frames, npad, jb)) return rc; }
    }
    return RCVD_OK;
  }

  // the explicit inverses of the level's diagonal blocks, then the TRSM X_rk = A_rk L_kk^-T of its off-diagonal blocks
  int trsm(const Level& lv, const int* frames, int nfr, bool chain) {
    // k_trsm_ll does not read the explicit inverse, only the (much later) substitution does: compute it off the critical path
    const bool inv_stream = fk.trsm_ll && p->overlap;
    if (inv_stream) { if (int rc = wait(inv, st, p->ev_fork)) return rc; inv_used = true; }
    if (int rc = launch(LP_TRINV, k_trinv, dim3(npad / 16, nfr), dim3(256), fk.trinv_bytes, inv_stream ? inv : st, false,
                        p->d_Lb, p->d_invT, p->d_invL, frames, npad)) return rc;
    mark(P_TRINV);
    if (lv.ntrsm == 0) return RCVD_OK;
    int rc;
    if (fk.trsm_ll) {
      // One CTA per SM fits the launch in a single wave: deep panel prefetch (AHEAD = 4); otherwise two CTAs per SM (AHEAD = 2).
      // A launch that is a single wave (`chain`: the narrow levels) starts beside its level's k_potrf_smem as a programmatic dependent
      // launch and follows the tile columns the Cholesky publishes.  The wide levels' multi-wave launches wait for the Cholesky to finish.
      const bool deep = trsm_deep(lv);
      decltype(&k_trsm_ll<2>) kernel = deep ? (chain ? k_trsm_ll<4, true> : k_trsm_ll<4>) : (chain ? k_trsm_ll<2, true> : k_trsm_ll<2>);
      if (chain) p->paths[LP_TRSM_STREAMED]++;
      rc = launch(deep ? LP_TRSM_LL4 : LP_TRSM_LL2, kernel, dim3(strips, lv.ntrsm), dim3(128), deep ? fk.trsm_ll4_bytes : fk.trsm_ll2_bytes, st, chain,
                  p->d_T, p->d_Lb, p->d_invT, p->d_trsm_tasks + lv.trsm_off, npad, chain ? p->d_potrf_progress : nullptr);
    } else {
      const int tiles = (npad + 63) / 64;
      rc = launch(LP_TRSM_GEMM, k_gemm_nt, dim3(tiles, tiles, lv.ntrsm), dim3(128), 0, st, false, p->d_T, p->d_Lb, p->d_invL,
                  p->d_trsm_tasks + lv.trsm_off, npad);
    }
    if (rc) return rc;
    mark(P_TRSM);
    return RCVD_OK;
  }

  // the persistent TMA-fed update kernel over the items [off, off + n) of the list upd_order selects
  int update(cudaStream_t s, int off, int n) {
    const UpdItem* items = p->d_upd_items + (size_t)p->upd_order * pl.upd_items.size() + off;
    if (n <= p->num_sms)   // few items: two DMMA teams per tile, one CTA per SM
      return launch(LP_UPD_TMA2, k_update_tma<2>, dim3(n), dim3(UpdShape<2>::threads), upd_smem_bytes(pl.upd_rb, 2), s, false,
                    p->tmapT, p->d_Lb, items, n, p->d_upd_pairs, npad, pl.upd_neff, pl.upd_rb, 0);
    int grid = upd_ctas(n, p->num_sms);
    if (p->upd_ipc > 0) grid = std::max(grid, (n + p->upd_ipc - 1) / p->upd_ipc);
    if (grid < n) p->paths[LP_UPD_TMA1_MULTI]++;
    return launch(LP_UPD_TMA1, k_update_tma<1>, dim3(grid), dim3(UpdShape<1>::threads), upd_smem_bytes(pl.upd_rb, 1), s, false,
                  p->tmapT, p->d_Lb, items, n, p->d_upd_pairs, npad, pl.upd_neff, pl.upd_rb, 0);
  }

  // The update passes of level li: after the waits for the earlier levels' U2 launches it needs, U1 on the main stream, then the
  // two U2 launches (on `side` when overlapping)
  int updates(int li) {
    const Level& lv = pl.levels[li];
    const bool u2 = lv.nit2[0] + lv.nit2[1] > 0;
    // Before a streamed level U2 forks only after U1: launched beside U1, U2's persistent CTAs (two per SM) took every SM that drained,
    // and the next level's k_potrf_smem, which needs a whole SM, started 15-40 us after U1 had finished.
    const bool fork_late = li + 1 < (int)pl.levels.size() && streamed(pl.levels[li + 1]);
    if (p->overlap && u2 && !fork_late) { if (int rc = wait(side, st, p->ev_fork)) return rc; }
    if (p->overlap) {   // U2 launch s of level q before U1(join[s] of q)
      int s = -1;
      for (int q = side_joined + 1; q < 2 * li; ++q) { const Level& v = pl.levels[q / 2]; if (v.nit2[q % 2] > 0 && v.join[q % 2] <= li) s = q; }
      if (s >= 0) { CK(cudaStreamWaitEvent(st, p->ev_side[s], 0)); side_joined = s; }
    }
    if (lv.nit > 0) { if (int rc = update(st, lv.it_off, lv.nit)) return rc; mark(P_GEMM); }
    if (p->overlap && u2 && fork_late) { if (int rc = wait(side, st, p->ev_fork)) return rc; }
    for (int h = 0; h < 2; ++h) if (lv.nit2[h] > 0) {
      if (int rc = update(p->overlap ? side : st, lv.it2_off[h], lv.nit2[h])) return rc;
      mark(P_GEMM);
      if (p->overlap) { CK(cudaEventRecord(p->ev_side[2 * li + h], side)); side_used = true; }
    }
    return RCVD_OK;
  }

  // distributed factorisation, levels < LB: the level's off-diagonal factor blocks from their owners to everybody (one fused NCCL launch)
  int broadcast_level(int li) {
    std::vector<Seg> segs;
    for (int q = 0; q < p->nranks; ++q) segs.push_back({(size_t)pl.tseg[(li * p->nranks + q) * 2], (size_t)pl.tseg[(li * p->nranks + q) * 2 + 1]});
    return grouped(p, p->d_T, (size_t)npad * npad, segs, true);
  }
  // phase boundary of the distributed factorisation: the owners' explicit inverses (for the replicated substitution) and their
  // blocks of the trailing matrix go to everybody; from here on every rank factors the same narrow tail
  int phase_boundary() {
    if (int rc = join_all(pl.LB)) return rc;
    const size_t bsz = (size_t)npad * npad;
    std::vector<Seg> invs, tr;
    for (int q = 0; q < p->nranks; ++q) invs.push_back({(size_t)pl.fa_off[q], (size_t)pl.fa_cnt[q]});
    for (int q = 0; q < p->nranks; ++q) tr.push_back({(size_t)pl.fb_off[q], (size_t)pl.fb_cnt[q]});
    for (int q = 0; q < p->nranks; ++q) tr.push_back({(size_t)N + (size_t)pl.bseg[2 * q], (size_t)pl.bseg[2 * q + 1]});
    if (int rc = grouped(p, p->d_invL, bsz, invs, true)) return rc;
    return grouped(p, p->d_Lb, bsz, tr, true);
  }

  // y = A^{-1} gs by GEMVs with the explicit inverses: the wide levels level by level, the levels >= sub_first_level in the persistent
  // dataflow kernel (rcvd_linalg.cuh, k_substitution)
  int substitution() {
    CK(cudaMemcpyAsync(p->d_rhs, p->d_gs, (size_t)N * npad * sizeof(double), cudaMemcpyDeviceToDevice, st));
    const int LS = pl.sub_first_level;
    int rc;
    for (int l = 0; l < LS; ++l) {
      const Level& lv = pl.levels[l];
      if ((rc = launch(LP_SUB_LEVEL, k_fwd_diag, dim3((npad + 7) / 8, lv.nframes), dim3(256), 0, st, false, p->d_invL, p->d_rhs, p->d_ytmp,
                       p->d_lvl_frames + lv.frame_off, npad, nullptr))) return rc;
      if (lv.nfwd > 0 && (rc = launch(LP_SUB_LEVEL, k_fwd_update, dim3((npad + 7) / 8, lv.nfwd), dim3(256), 0, st, false, p->d_T, p->d_ytmp, p->d_rhs,
                                      p->d_fwd_tasks + lv.fwd_off, npad))) return rc;
    }
    if (LS < (int)pl.levels.size() && !pl.sub_tasks.empty()) {
      CK(cudaMemsetAsync(p->d_sub_counters, 0, ((size_t)4 * N + 4) * sizeof(int), st));
      SubCounters cn; cn.ticket = p->d_sub_counters; cn.fin = p->d_sub_counters + 4; cn.fdone = cn.fin + N; cn.bin = cn.fdone + N; cn.bdone = cn.bin + N;
      cn.fin_need = p->d_sub_need; cn.bin_need = p->d_sub_need + N;
      const int ntasks = (int)pl.sub_tasks.size();
      if ((rc = launch(LP_SUB_FUSED, k_substitution, dim3(std::min(ntasks, p->num_sms)), dim3(kSubThreads), fk.substitution_bytes, st, false,
                       p->d_invL, p->d_T, p->d_rhs, p->d_ytmp, p->d_y, p->d_sub_tasks, ntasks, cn, npad))) return rc;
    }
    for (int l = LS - 1; l >= 0; --l) {
      const Level& lv = pl.levels[l];
      if (lv.nfwd > 0 && (rc = launch(LP_SUB_LEVEL, k_bwd_update, dim3((npad + 31) / 32, lv.nfwd), dim3(256), 0, st, false, p->d_T, p->d_y, p->d_ytmp,
                                      p->d_fwd_tasks + lv.fwd_off, npad))) return rc;
      if ((rc = launch(LP_SUB_LEVEL, k_bwd_diag, dim3((npad + 31) / 32, lv.nframes), dim3(256), 0, st, false, p->d_invL, p->d_ytmp, p->d_y,
                       p->d_lvl_frames + lv.frame_off, npad, nullptr))) return rc;
    }
    mark(P_SOLVE);
    return RCVD_OK;
  }
};

static int enqueue_factor_solve(rcvd_problem* p) {
  FactorSolve f(p);
  const FactorPlan& pl = p->plan; const int npad = p->L.npad, nlv = (int)pl.levels.size();
  f.mark(-1);
  CK(cudaMemsetAsync(p->d_potrf_progress, 0, (size_t)p->N * sizeof(int), p->stream));   // no count of the previous factorisation may read as published
  // the blocks this rank factors; of the fill blocks only the padding, their interior is written by their first update pass
  const int nfill = (int)pl.load_lblocks.size() - pl.nload;
  if (int rc = f.launch(LP_OTHER, k_load_factor, dim3((npad * npad + 255) / 256, pl.nload + load_factor_pad_rows(npad, pl.upd_neff, nfill)), dim3(256), 0,
                        p->stream, false, p->d_H, p->d_Lb, p->d_lblocks, p->d_S, p->d_D2, npad, p->L.nf, pl.upd_neff, p->d_load_lblocks, pl.nload, nfill)) return rc;
  f.mark(FactorSolve::P_LOAD);
  for (int li = 0; li < nlv; ++li) {
    const Level& lv = pl.levels[li]; f.prof_level = li;
    if (pl.dist && li == pl.LB) { if (int rc = f.phase_boundary()) return rc; }
    if (lv.nown > 0) {
      const int* frames = p->d_lvl_own + lv.own_off;      // the frames this rank factors at this level
      // On a streamed level the Cholesky is a programmatic dependent of the previous level's U1 (it waits for it with griddepcontrol.wait
      // before it reads anything), so its CTAs are resident as soon as U1's SMs drain; the previous level forked its U2 only after U1.
      const bool chain = f.streamed(lv);
      if (int rc = f.factor_diagonal(frames, lv.nown, chain && li > 0)) return rc;
      f.mark(FactorSolve::P_POTRF);
      if (int rc = f.trsm(lv, frames, lv.nown, chain)) return rc;
    }
    if (pl.dist && li < pl.LB) { if (int rc = f.broadcast_level(li)) return rc; }
    if (int rc = f.updates(li)) return rc;
  }
  if (pl.dist && pl.LB >= nlv) { if (int rc = f.phase_boundary()) return rc; }
  if (int rc = f.join_all(nlv)) return rc;
  if (int rc = f.substitution()) return rc;
  CK(cudaGetLastError());
  return RCVD_OK;
}

// factor+solve through a CUDA graph (the level schedule is ~5 launches per level)
static int factor_solve(rcvd_problem* p) {
  if (p->nranks > 1 && !p->graph_warm) {   // NCCL establishes its connections lazily on first use: not inside a stream capture
    p->graph_warm = true; p->factored = true;
    return enqueue_factor_solve(p);
  }
  if (!p->solve_graph) {
    cudaGraph_t graph;
    const int64_t l0 = p->launches;
    int64_t paths0[LP_N]; std::copy(p->paths, p->paths + LP_N, paths0);
    CK(cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal));
    int rc = enqueue_factor_solve(p);
    cudaError_t e = cudaStreamEndCapture(p->stream, &graph);
    for (int i = 0; i < LP_N; ++i) { p->graph_paths[i] = p->paths[i] - paths0[i]; p->paths[i] = paths0[i]; }
    if (rc) return rc;
    if (e != cudaSuccess) return set_err(RCVD_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    CK(cudaGraphInstantiate(&p->solve_graph, graph, 0));
    cudaGraphDestroy(graph);
    p->graph_launches = p->launches - l0;
    p->launches = l0;
  }
  CK(cudaGraphLaunch(p->solve_graph, p->stream));
  p->launches += p->graph_launches;
  for (int i = 0; i < LP_N; ++i) p->paths[i] += p->graph_paths[i];
  p->factored = true;
  return RCVD_OK;
}

// ---- block-Jacobi preconditioned conjugate gradients (rcvd_cg.cuh) ----
// The preconditioner: the damped diagonal blocks of the frames, loaded, factored and inverted by the block Cholesky's per-frame kernels
// over every frame at once -- the factorisation of the edgeless frame graph, which is exactly a block-diagonal factor.
static int enqueue_cg_preconditioner(rcvd_problem* p) {
  FactorSolve f(p);
  const int N = p->N, npad = p->L.npad;
  if (int rc = f.launch(LP_OTHER, k_load_factor, dim3((npad * npad + 255) / 256, N), dim3(256), 0, p->stream, false, p->d_H, p->d_Lb, p->d_lblocks,
                        p->d_S, p->d_D2, npad, p->L.nf, p->plan.upd_neff, p->d_cg_frames, N, 0)) return rc;
  if (int rc = f.factor_diagonal(p->d_cg_frames, N, false)) return rc;
  return f.launch(LP_TRINV, k_trinv, dim3(npad / 16, N), dim3(256), p->fk.trinv_bytes, p->stream, false, p->d_Lb, p->d_invT, p->d_invL, p->d_cg_frames, npad);
}

// out = (S H S + D2) v and the per-frame partials of v.out; nothing once cg->stop is set (cg null: unconditionally)
static int enqueue_cg_product(rcvd_problem* p, const double* v, double* out, const CgState* cg) {
  const int N = p->N, npad = p->L.npad, nf = p->L.nf, nH = (int)p->plan.hblocks.size();
  const size_t smem = (size_t)(3 * npad + 8 * 256) * sizeof(double);
  if (int rc = launch(p, k_cg_spmv, nH, kCgThreads, smem, p->stream, false, p->d_H, p->d_hblocks, p->d_S, v, p->d_cg_slots, nH, npad, nf, cg)) return rc;
  return launch(p, k_cg_gather, N, kCgThreads, 0, p->stream, false, p->d_cg_slots, p->d_cg_off, p->d_cg_ids, p->d_S, p->d_D2, v, out, p->d_cg_part, npad, nf, cg);
}

// Iteration i of the PCG on A = S H S + D2, b = gs, x = d_y (rcvd_cg.cuh gives the Ceres semantics it restates).
static int enqueue_cg_iteration(rcvd_problem* p, int i) {
  const int N = p->N, npad = p->L.npad, n = N * npad;
  cudaStream_t st = p->stream; const int* stop = &p->d_cg->stop; double* x = p->d_y; int rc;
  auto apply = [&](const double* v, double* out) { return enqueue_cg_product(p, v, out, p->d_cg); };
  auto scalar = [&](int phase, int nparts) {
    return launch(p, k_cg_scalar, 1, kCgThreads, 0, st, false, p->d_cg_part, nparts, p->d_cg, p->d_fail, phase, p->cg_eta, kCgMaxIterations);
  };
  auto step = [&](int mode) {
    return launch(p, k_cg_step, kCgDotBlocks, kCgThreads, 0, st, false, x, p->d_cg_p, p->d_cg_r, p->d_cg_q, p->d_gs, p->d_cg_part, n, mode, p->d_cg);
  };
  // z = L^-T L^-1 r, rho = r.z, p = z + beta p
  if ((rc = launch(p, k_fwd_diag, dim3((npad + 7) / 8, N), 256, 0, st, false, p->d_invL, p->d_cg_r, p->d_ytmp, p->d_cg_frames, npad, stop)) ||
      (rc = launch(p, k_bwd_diag, dim3((npad + 31) / 32, N), 256, 0, st, false, p->d_invL, p->d_ytmp, p->d_cg_z, p->d_cg_frames, npad, stop)) ||
      (rc = launch(p, k_cg_dot, kCgDotBlocks, kCgThreads, 0, st, false, p->d_cg_r, p->d_cg_z, p->d_cg_part, n, p->d_cg)) || (rc = scalar(CG_RHO, kCgDotBlocks)) ||
      (rc = launch(p, k_cg_direction, kCgDotBlocks, kCgThreads, 0, st, false, p->d_cg_z, p->d_cg_p, n, p->d_cg)))
    return rc;
  // q = A p, alpha = rho / p.q, x += alpha p, r -= alpha q (or r = b - A x), the quadratic-model test
  if ((rc = apply(p->d_cg_p, p->d_cg_q)) || (rc = scalar(CG_CURVATURE, N))) return rc;
  if (i % kCgResetPeriod != 0) rc = step(0);
  else if (!(rc = step(1)) && !(rc = apply(x, p->d_cg_q))) rc = step(2);
  return rc ? rc : scalar(CG_MODEL, kCgDotBlocks);
}

// y = A^-1 gs by PCG: the preconditioner, then iterations in chunks of kCgChunk with one read of the stop flag after each chunk.
static int cg_solve(rcvd_problem* p) {
  cudaStream_t st = p->stream; int rc;
  if ((rc = enqueue_cg_preconditioner(p)) ||
      (rc = launch(p, k_cg_init, kCgDotBlocks, kCgThreads, 0, st, false, p->d_gs, p->d_y, p->d_cg_r, p->d_cg_part, p->N * p->L.npad)) ||
      (rc = launch(p, k_cg_scalar, 1, kCgThreads, 0, st, false, p->d_cg_part, kCgDotBlocks, p->d_cg, p->d_fail, (int)CG_INIT, p->cg_eta, kCgMaxIterations)))
    return rc;
  CgState h;
  for (int i = 1;; ) {
    for (int k = 0; k < kCgChunk && i <= kCgMaxIterations; ++k, ++i) if ((rc = enqueue_cg_iteration(p, i))) return rc;
    CK(cudaMemcpyAsync(&h, p->d_cg, sizeof(h), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (h.stop || i > kCgMaxIterations) break;
  }
  p->cg_last = h.iterations; p->cg_iterations += h.iterations; p->cg_max = std::max(p->cg_max, h.iterations);
  p->cg_capped += h.capped; p->cg_steps += 1;
  return RCVD_OK;
}

// The damped solve y = (S H S + D2)^-1 gs of the path build_structure chose.
static int linear_solve(rcvd_problem* p) { return p->use_cg ? cg_solve(p) : factor_solve(p); }

// ---------------------------------------------------------------------------
// Evaluation
// ---------------------------------------------------------------------------

// Cost (-> d_scal[slot]) at state x; optionally gradient (gout, npad stride) and H.
static int enqueue_evaluate(rcvd_problem* p, const double* x, bool wantG, bool wantH, double* gout, int slot) {
  if (wantH && p->eval_only) return set_err(RCVD_ERR_INVALID, "this handle was set to evaluation-only (rcvd_debug_set_eval_only): no normal matrix");
  const Layout& L = p->L; const int N = p->N, npad = L.npad; cudaStream_t st = p->stream;
  const size_t bs = (size_t)npad * npad, Upad = (size_t)N * npad;
  if (wantH) CK(cudaMemsetAsync(p->d_H, 0, p->plan.hblocks.size() * bs * sizeof(double), st));
  if (wantG) CK(cudaMemsetAsync(gout, 0, (Upad + 8) * sizeof(double), st));
  int rc = wantH ? enqueue_residuals<EvalMode::CostGradH>(p, x, gout)
           : wantG ? enqueue_residuals<EvalMode::CostGrad>(p, x, gout) : enqueue_residuals<EvalMode::Cost>(p, x, gout);
  if (rc) return rc;
  if ((rc = launch(p, k_reduce_partials, 1, 1024, 0, st, false, p->d_partial, p->npartial, p->d_scal, slot))) return rc;
  if (p->nranks > 1) {
    if (wantG) {
      // ONE packed all-reduce: [gradient (Upad) | cost + 7 spare | diagonal of H (Upad, only with H into d_g)]
      CK(cudaMemcpyAsync(gout + Upad, p->d_scal + slot, sizeof(double), cudaMemcpyDeviceToDevice, st));
      size_t cnt = Upad + 8;
      if (wantH && gout == p->d_g) { if ((rc = launch(p, k_extract_diag, (int)((Upad + 255) / 256), 256, 0, st, false, p->d_H, p->d_diagH, N, npad))) return rc; cnt = 2 * Upad + 8; }
      if ((rc = allreduce(p, gout, cnt))) return rc;
      CK(cudaMemcpyAsync(p->d_scal + slot, gout + Upad, sizeof(double), cudaMemcpyDeviceToDevice, st));
    } else if ((rc = allreduce(p, p->d_scal + slot, 1))) return rc;
    if (wantH) {
      if (p->plan.dist && !p->force_full_H) {
        // the normal matrix is summed onto the OWNER of every block only (its frames' diagonal blocks, the off-diagonal blocks of its columns)
        std::vector<Seg> segs;
        for (int q = 0; q < p->nranks; ++q) segs.push_back({(size_t)p->plan.fa_off[q], (size_t)(p->plan.fa_cnt[q] + p->plan.fb_cnt[q])});
        for (int q = 0; q < p->nranks; ++q) segs.push_back({(size_t)p->plan.hseg[2 * q], (size_t)p->plan.hseg[2 * q + 1]});
        if ((rc = grouped(p, p->d_H, bs, segs, false))) return rc;
      } else if ((rc = allreduce(p, p->d_H, p->plan.hblocks.size() * bs))) return rc;
    }
  }
  return RCVD_OK;
}

static int ensure_ready(rcvd_problem* p) {
  if (!p->structure_ready) { if (int rc = build_structure(p)) return rc; }
  if (p->state_dirty) {
    const std::vector<double> x = frames_to_internal(p->plan.uperm, p->h_state.data(), p->L.nf, p->L.nf, p->L.nf);
    CK(cudaMemcpyAsync(p->d_x, x.data(), x.size() * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    CK(cudaStreamSynchronize(p->stream));      // x goes out of scope
    p->state_dirty = false;
  }
  return RCVD_OK;
}

static int read_scalars(rcvd_problem* p) {
  CK(cudaMemcpyAsync(p->h_scal, p->d_scal, SC_N * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  CK(cudaMemcpyAsync(p->h_fail, p->d_fail, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
  CK(cudaStreamSynchronize(p->stream));
  return RCVD_OK;
}

// ---------------------------------------------------------------------------
// Polynomial minimisation for the Armijo line search (ceres/polynomial.cc semantics)
// ---------------------------------------------------------------------------
namespace ls {
struct Sample { double x, value, gradient; bool valueValid, gradValid; };
static double evalPoly(const std::vector<double>& p, double x) { double v = 0; for (double c : p) v = v * x + c; return v; }
static bool solveDense(std::vector<std::vector<double>> A, std::vector<double> b, std::vector<double>& x) {
  const int n = (int)b.size(); std::vector<int> perm(n); for (int i = 0; i < n; ++i) perm[i] = i;
  for (int k = 0; k < n; ++k) {
    int pr = k, pc = k; double best = 0;
    for (int i = k; i < n; ++i) for (int j = k; j < n; ++j) if (std::fabs(A[i][j]) > best) { best = std::fabs(A[i][j]); pr = i; pc = j; }
    if (best == 0) return false;
    std::swap(A[k], A[pr]); std::swap(b[k], b[pr]);
    for (int i = 0; i < n; ++i) std::swap(A[i][k], A[i][pc]);
    std::swap(perm[k], perm[pc]);
    for (int i = k + 1; i < n; ++i) { const double f = A[i][k] / A[k][k]; for (int j = k; j < n; ++j) A[i][j] -= f * A[k][j]; b[i] -= f * b[k]; }
  }
  std::vector<double> y(n);
  for (int i = n - 1; i >= 0; --i) { double s = b[i]; for (int j = i + 1; j < n; ++j) s -= A[i][j] * y[j]; y[i] = s / A[i][i]; }
  x.assign(n, 0.0); for (int i = 0; i < n; ++i) x[perm[i]] = y[i];
  return true;
}
static std::vector<double> realRoots(std::vector<double> p) {
  while (!p.empty() && p[0] == 0.0) p.erase(p.begin());
  std::vector<double> out; const int d = (int)p.size() - 1; if (d < 1) return out;
  if (d == 1) { out.push_back(-p[1] / p[0]); return out; }
  if (d == 2) { const double a = p[0], b = p[1], c = p[2], D = b * b - 4 * a * c; if (D >= 0) { const double sq = std::sqrt(D); out.push_back((-b + sq) / (2 * a)); out.push_back((-b - sq) / (2 * a)); } else { out.push_back(-b / (2 * a)); out.push_back(-b / (2 * a)); } return out; }
  std::vector<std::pair<double, double>> z(d);
  for (int i = 0; i < d; ++i) { const double ang = 2 * M_PI * i / d + 0.4; z[i] = {0.9 * std::cos(ang), 0.9 * std::sin(ang)}; }
  auto cmul = [](std::pair<double, double> a, std::pair<double, double> b) { return std::make_pair(a.first * b.first - a.second * b.second, a.first * b.second + a.second * b.first); };
  auto cdiv = [](std::pair<double, double> a, std::pair<double, double> b) { const double dd = b.first * b.first + b.second * b.second; return std::make_pair((a.first * b.first + a.second * b.second) / dd, (a.second * b.first - a.first * b.second) / dd); };
  for (int it = 0; it < 500; ++it) {
    double mx = 0;
    for (int i = 0; i < d; ++i) {
      std::pair<double, double> v = {p[0], 0.0};
      for (int j = 1; j <= d; ++j) { v = cmul(v, z[i]); v.first += p[j]; }
      std::pair<double, double> den = {p[0], 0.0};
      for (int j = 0; j < d; ++j) if (j != i) den = cmul(den, {z[i].first - z[j].first, z[i].second - z[j].second});
      auto dl = cdiv(v, den); z[i].first -= dl.first; z[i].second -= dl.second;
      mx = std::max(mx, std::fabs(dl.first) + std::fabs(dl.second));
    }
    if (mx < 1e-14) break;
  }
  for (auto& r : z) out.push_back(r.first);
  return out;
}
static double minimizeInterpolating(const std::vector<Sample>& s, double xmin, double xmax) {
  int nc = 0; for (auto& q : s) { if (q.valueValid) ++nc; if (q.gradValid) ++nc; }
  const int deg = nc - 1;
  std::vector<std::vector<double>> A; std::vector<double> b;
  for (auto& q : s) {
    if (q.valueValid) { std::vector<double> row(nc); for (int j = 0; j <= deg; ++j) row[j] = std::pow(q.x, deg - j); A.push_back(row); b.push_back(q.value); }
    if (q.gradValid) { std::vector<double> row(nc); for (int j = 0; j < deg; ++j) row[j] = (deg - j) * std::pow(q.x, deg - j - 1); row[deg] = 0; A.push_back(row); b.push_back(q.gradient); }
  }
  std::vector<double> poly; if (!solveDense(A, b, poly)) return 0.5 * (xmin + xmax);
  double ox = (xmin + xmax) / 2.0, ov = evalPoly(poly, ox);
  const double vmin = evalPoly(poly, xmin); if (vmin < ov) { ov = vmin; ox = xmin; }
  const double vmax = evalPoly(poly, xmax); if (vmax < ov) { ov = vmax; ox = xmax; }
  if (poly.size() <= 2) return ox;
  std::vector<double> der;
  for (int j = 0; j < deg; ++j) der.push_back((deg - j) * poly[j]);
  for (double r : realRoots(der)) { if (r < xmin || r > xmax) continue; const double v = evalPoly(poly, r); if (v < ov) { ov = v; ox = r; } }
  return ox;
}
}  // namespace ls

__global__ void k_make_delta(const double* __restrict__ y, const double* __restrict__ S, double* __restrict__ delta, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) delta[i] = -y[i] * S[i];
}

// xc = Plus(x, alpha * delta) with bounds projection, delta = -y*S (k_make_delta); accumulates |x - xc|^2 over active params,
// g . delta and max|delta| (for the line search).  delta, g have npad stride; x, xc nf stride.
__global__ void __launch_bounds__(256) k_candidate(rcvd_config cfg, Layout L, const uint8_t* __restrict__ in_range, const uint8_t* __restrict__ active,
                                                    const double* __restrict__ x, const double* __restrict__ delta, const double* __restrict__ g,
                                                    double alpha, double* __restrict__ xc, double* __restrict__ scal, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double d2 = 0.0, gd = 0.0, dm = 0.0;
  if (i < N * L.nf) {
    const int f = i / L.nf, l = i % L.nf;
    const size_t v = (size_t)f * L.npad + l;
    const double dl = delta[v];
    const double xn = project_lb(cfg, L, in_range, f, l, x[i] + alpha * dl);
    xc[i] = xn;
    if (active[v]) { const double d = x[i] - xn; d2 = d * d; }
    gd = g[v] * dl; dm = fabs(dl);
  }
  d2 = warp_sum(d2); gd = warp_sum(gd);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dm = fmax(dm, __shfl_xor_sync(0xffffffffu, dm, o));
  if ((threadIdx.x & 31) == 0) {
    red_add(scal + SC_STEP2, d2); red_add(scal + SC_GDOTD, gd);
    atomicMax((unsigned long long*)(scal + SC_DMAX), (unsigned long long)__double_as_longlong(dm));   // dm >= 0: bit pattern is monotone
  }
}

// The three parts of an LM step.  rcvd_solve, rcvd_time_iteration and rcvd_debug_linear_residual all build their steps from them.

// Assemble: cost (SC_COST), gradient (d_g) and H at d_x, and diag H into d_diagH (at N > 1 enqueue_evaluate extracts it for its all-reduce)
static int enqueue_assemble(rcvd_problem* p) {
  if (int rc = enqueue_evaluate(p, p->d_x, true, true, p->d_g, SC_COST)) return rc;
  if (p->nranks > 1) return RCVD_OK;
  return launch(p, k_extract_diag, nblk((size_t)p->N * p->L.npad), 256, 0, p->stream, false, p->d_H, p->d_diagH, p->N, p->L.npad);
}

// Damped step: the LM diagonal (clamped S^2 diag H unless `reuse`), D2 = diagonal / radius and gs = S g; y = (S H S + D2)^-1 gs; the
// model terms gs.y (GY) and (Sy)^T H (Sy) (YHY, with H (S y) left in d_Hy) and delta = -y S.
static int enqueue_damped_step(rcvd_problem* p, const rcvd_solve_options& o, double radius, bool reuse) {
  const int npad = p->L.npad; const size_t Upad = (size_t)p->N * npad; cudaStream_t st = p->stream;
  int rc;
  if ((rc = launch(p, k_lm_prepare, nblk(Upad), 256, 0, st, false, p->d_diagH, p->d_S, p->d_g, p->d_lmdiag, p->d_D2, p->d_gs, (int)Upad, reuse ? 1 : 0, radius, o.min_lm_diagonal, o.max_lm_diagonal))) return rc;
  if ((rc = linear_solve(p))) return rc;
  if ((rc = launch(p, k_mul, nblk(Upad), 256, 0, st, false, p->d_S, p->d_y, p->d_Sy, (int)Upad))) return rc;
  CK(cudaMemsetAsync(p->d_Hy, 0, Upad * sizeof(double), st));
  if ((rc = launch(p, k_spmv_sym, dim3((npad + 7) / 8, p->plan.dist ? (int)p->plan.own_hblocks.size() : (int)p->plan.hblocks.size()), 256, 0, st, false, p->d_H, p->d_hblocks, p->d_Sy, p->d_Hy, npad, p->plan.dist ? p->d_own_hblocks : nullptr))) return rc;
  if ((rc = launch(p, k_dot2, nblk(Upad), 256, 0, st, false, p->d_gs, p->d_y, p->d_Sy, p->d_Hy, (int)Upad, p->d_scal, SC_GY, SC_YHY))) return rc;
  if (p->plan.dist && (rc = allreduce(p, p->d_scal + SC_YHY, 1))) return rc;   // every rank multiplied the H blocks it owns
  return launch(p, k_make_delta, nblk(Upad), 256, 0, st, false, p->d_y, p->d_S, p->d_delta, (int)Upad);
}

// Candidate cost: xc = Plus(x, alpha delta), then the cost at xc (SC_CAND).  `slope` (a line-search trial): also the gradient at xc
// into d_g2 and its directional derivative g(xc).delta (SC_GY).
static int enqueue_candidate_cost(rcvd_problem* p, double alpha, bool slope) {
  const size_t U = (size_t)p->N * p->L.nf, Upad = (size_t)p->N * p->L.npad;
  if (int rc = launch(p, k_candidate, nblk(U), 256, 0, p->stream, false, p->cfg, p->L, p->d_in_range, p->d_active, p->d_x, p->d_delta, p->d_g, alpha, p->d_xc, p->d_scal, p->N)) return rc;
  if (int rc = enqueue_evaluate(p, p->d_xc, slope, false, slope ? p->d_g2 : nullptr, SC_CAND)) return rc;
  if (!slope) return RCVD_OK;
  return launch(p, k_dot2, nblk(Upad), 256, 0, p->stream, false, p->d_g2, p->d_delta, p->d_g2, p->d_delta, (int)Upad, p->d_scal, SC_GY, SC_YHY);
}

static float ev_ms(cudaEvent_t a, cudaEvent_t b) { float m = 0; cudaEventElapsedTime(&m, a, b); return m; }

// ---------------------------------------------------------------------------
// Levenberg-Marquardt, Ceres semantics (TrustRegionMinimizer::Minimize restated).
// ---------------------------------------------------------------------------
static int lm_solve(rcvd_problem* p, const rcvd_solve_options& o, rcvd_solve_summary& sum) {
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  memset(&sum, 0, sizeof(sum));
  int rc = ensure_ready(p); if (rc) return rc;
  const Layout& L = p->L; const int N = p->N, npad = L.npad; const size_t Upad = (size_t)N * npad, U = (size_t)N * L.nf; cudaStream_t st = p->stream;
  const int64_t launches0 = p->launches;
  p->cg_iterations = 0; p->cg_max = 0; p->cg_capped = 0; p->cg_steps = 0;
  sum.num_constraints = p->pairs.count();
  const bool constrained = p->cfg.depth_lower_bound && L.nd > 0;
  if (constrained && (rc = launch(p, k_project_state, nblk(U), 256, 0, st, false, p->cfg, L, p->d_in_range, p->d_x, N))) return rc;
  // user-visible minimum-cost iterate
  CK(cudaMemcpyAsync(p->d_xsave, p->d_x, U * sizeof(double), cudaMemcpyDeviceToDevice, st));

  auto full_eval = [&]() -> int {   // assemble, then the norms at d_x
    CK(cudaMemsetAsync(p->d_scal, 0, SC_N * sizeof(double), st));
    CK(cudaEventRecord(p->ev[0], st));
    int r = enqueue_assemble(p); if (r) return r;
    CK(cudaEventRecord(p->ev[1], st));
    r = launch(p, k_state_norms, nblk(U), 256, 0, st, false, p->cfg, L, p->d_in_range, p->d_active, p->d_x, p->d_g, p->d_scal, N); if (r) return r;
    r = read_scalars(p); if (r) return r;
    sum.eval_ms += ev_ms(p->ev[0], p->ev[1]);
    return RCVD_OK;
  };
  if ((rc = full_eval())) return rc;
  double xCost = p->h_scal[SC_COST], xNorm = std::sqrt(p->h_scal[SC_X2]), gmax = p->h_scal[SC_GMAX];
  sum.initial_cost = xCost;
  if ((rc = launch(p, k_jacobi_scale, nblk(Upad), 256, 0, st, false, p->d_diagH, p->d_S, (int)Upad, o.jacobi_scaling))) return rc;
  double radius = o.initial_radius, decrease = 2.0; bool reuseDiag = false;
  double minimumCost = xCost;
  int iter = 0, invalid = 0; bool stepSuccessful = true;
  auto finish = [&](int term, const char* msg) { sum.termination = term; snprintf(sum.message, sizeof(sum.message), "%s", msg); };
  finish(RCVD_TERM_NO_CONVERGENCE, "");
  if (o.verbose) fprintf(stderr, "[rcvd] iter      cost      cost_change  |gradient|   |step|    tr_ratio  tr_radius\n[rcvd] %4d %.6e %10.2e %10.2e %10.2e %10.2e %10.2e\n", 0, xCost, 0.0, gmax, 0.0, 0.0, radius);
  for (;;) {
    if (stepSuccessful) {
      ++sum.num_successful_steps;
      if (xCost < minimumCost || iter == 0) { minimumCost = xCost; CK(cudaMemcpyAsync(p->d_xsave, p->d_x, U * sizeof(double), cudaMemcpyDeviceToDevice, st)); }
    } else ++sum.num_unsuccessful_steps;
    if (iter >= o.max_iterations) { finish(RCVD_TERM_NO_CONVERGENCE, "Maximum number of iterations reached."); break; }
    if (stepSuccessful && gmax <= o.gradient_tolerance) { finish(RCVD_TERM_CONVERGENCE, "Gradient tolerance reached."); break; }
    if (radius <= o.min_radius) { finish(RCVD_TERM_CONVERGENCE, "Minimum trust region radius reached."); break; }
    ++iter; stepSuccessful = false;
    // --- ComputeTrustRegionStep + candidate evaluation, one host sync ---
    CK(cudaMemsetAsync(p->d_scal, 0, SC_N * sizeof(double), st));
    CK(cudaMemsetAsync(p->d_fail, 0, sizeof(int), st));
    CK(cudaEventRecord(p->ev[2], st));
    if ((rc = enqueue_damped_step(p, o, radius, reuseDiag))) return rc;
    reuseDiag = true;
    CK(cudaEventRecord(p->ev[3], st));
    double alpha = 1.0;
    if (!constrained) {
      if ((rc = enqueue_candidate_cost(p, 1.0, false))) return rc;
      CK(cudaEventRecord(p->ev[4], st));
    }
    if ((rc = read_scalars(p))) return rc;
    sum.linear_ms += ev_ms(p->ev[2], p->ev[3]);
    if (!constrained) sum.cost_ms += ev_ms(p->ev[3], p->ev[4]);
    const double gy = p->h_scal[SC_GY], yHy = p->h_scal[SC_YHY];
    const double modelChange = gy - 0.5 * yHy;
    const bool ok = (*p->h_fail == 0) && std::isfinite(gy) && std::isfinite(yHy);
    if (!(ok && modelChange > 0.0)) {
      if (++invalid >= o.max_consecutive_invalid_steps) { finish(RCVD_TERM_FAILURE, "Number of consecutive invalid steps more than max_num_consecutive_invalid_steps."); break; }
      radius = radius / decrease; decrease *= 2.0; reuseDiag = true;
      if (o.verbose) fprintf(stderr, "[rcvd] %4d invalid step (fail=%d model=%g), radius %.3e\n", iter, *p->h_fail, modelChange, radius);
      continue;
    }
    invalid = 0;
    if (constrained) {
      // DoLineSearch: Armijo with cubic interpolation along the projected path (ceres defaults)
      auto trial = [&](double a, ls::Sample& s) -> int {
        CK(cudaMemsetAsync(p->d_scal, 0, SC_N * sizeof(double), st));
        int r = enqueue_candidate_cost(p, a, true); if (r) return r;
        r = read_scalars(p); if (r) return r;
        s.x = a; s.value = p->h_scal[SC_CAND]; s.valueValid = std::isfinite(s.value);
        s.gradient = p->h_scal[SC_GY]; s.gradValid = s.valueValid && std::isfinite(s.gradient);
        return RCVD_OK;
      };
      ls::Sample cur, prev{0, 0, 0, false, false};
      if ((rc = trial(1.0, cur))) return rc;
      const double gd = p->h_scal[SC_GDOTD], dirMax = p->h_scal[SC_DMAX];
      ls::Sample init{0.0, xCost, gd, true, true};
      int lsIter = 0; bool success = true;
      while (!cur.valueValid || cur.value > xCost + 1e-4 * gd * cur.x) {
        if (++lsIter >= 20) { success = false; break; }
        const double lo = 1e-3 * cur.x, hi = 0.6 * cur.x;
        double ss;
        if (!cur.valueValid) ss = std::min(std::max(cur.x * 0.5, lo), hi);
        else { std::vector<ls::Sample> sm{init, cur}; if (prev.valueValid) sm.push_back(prev); ss = ls::minimizeInterpolating(sm, lo, hi); }
        if (ss * dirMax < 1e-9) { success = false; break; }
        prev = cur;
        if ((rc = trial(ss, cur))) return rc;
      }
      alpha = success ? cur.x : 1.0;
      CK(cudaMemsetAsync(p->d_scal, 0, SC_N * sizeof(double), st));
      if ((rc = enqueue_candidate_cost(p, alpha, false))) return rc;
      if ((rc = read_scalars(p))) return rc;
    }
    double candCost = p->h_scal[SC_CAND];
    if (!std::isfinite(candCost)) candCost = std::numeric_limits<double>::max();
    const double stepNorm = std::sqrt(p->h_scal[SC_STEP2]);
    if (stepNorm <= o.parameter_tolerance * (xNorm + o.parameter_tolerance)) { finish(RCVD_TERM_CONVERGENCE, "Parameter tolerance reached."); break; }
    const double costChange = xCost - candCost;
    if (std::fabs(costChange) <= o.function_tolerance * xCost) { finish(RCVD_TERM_CONVERGENCE, "Function tolerance reached."); break; }
    const double relDecrease = (candCost >= std::numeric_limits<double>::max()) ? std::numeric_limits<double>::lowest() : costChange / modelChange;
    if (relDecrease > o.min_relative_decrease) {
      std::swap(p->d_x, p->d_xc);
      if ((rc = full_eval())) return rc;
      xCost = p->h_scal[SC_COST]; xNorm = std::sqrt(p->h_scal[SC_X2]); gmax = p->h_scal[SC_GMAX];
      stepSuccessful = true;
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relDecrease - 1.0, 3));
      radius = std::min(o.max_radius, radius); decrease = 2.0; reuseDiag = false;
    } else {
      radius = radius / decrease; decrease *= 2.0; reuseDiag = true;
    }
    if (o.verbose) fprintf(stderr, "[rcvd] %4d %.6e %10.2e %10.2e %10.2e %10.2e %10.2e\n", iter, stepSuccessful ? xCost : candCost, costChange, gmax, stepNorm, relDecrease, radius);
  }
  CK(cudaMemcpyAsync(p->d_x, p->d_xsave, U * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CK(cudaStreamSynchronize(st));
  sum.iterations = iter; sum.final_cost = minimumCost;
  sum.gpu_launches = p->launches - launches0;
  sum.total_ms = std::chrono::duration<double, std::milli>(clk::now() - t0).count();
  return RCVD_OK;
}

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
RCVD_API const char* rcvd_last_error(void) { return g_err.c_str(); }
RCVD_API int32_t rcvd_abi_version(void) { return 1; }
RCVD_API int32_t rcvd_frame_stride(const rcvd_config* c) { Layout L; return (c && make_layout(*c, L)) ? L.nf : -1; }
RCVD_API int32_t rcvd_depth_param_offset(const rcvd_config* c) { Layout L; return (c && make_layout(*c, L)) ? L.offD : -1; }
RCVD_API int32_t rcvd_spatial_param_offset(const rcvd_config* c) { Layout L; return (c && make_layout(*c, L)) ? L.offS : -1; }
RCVD_API void rcvd_default_solve_options(rcvd_solve_options* o) {
  o->max_iterations = 1000; o->verbose = 0; o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
  o->initial_radius = 1e4; o->max_radius = 1e16; o->min_radius = 1e-32; o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32; o->max_consecutive_invalid_steps = 5; o->jacobi_scaling = 1;
}

// cudaDeviceProp::totalGlobalMem of `device`, queried once per process: cudaGetDeviceProperties reads every property of the device, a
// cost a handle created per solve should not pay each time
static cudaError_t device_total_mem(int device, uint64_t* out) {
  static std::mutex m; static std::map<int, uint64_t> cache;
  std::lock_guard<std::mutex> lock(m);
  auto it = cache.find(device);
  if (it == cache.end()) {
    cudaDeviceProp prop;
    if (cudaError_t e = cudaGetDeviceProperties(&prop, device)) return e;
    it = cache.emplace(device, (uint64_t)prop.totalGlobalMem).first;
  }
  *out = it->second;
  return cudaSuccess;
}
RCVD_API int32_t rcvd_problem_create(const rcvd_config* cfg, int32_t device, rcvd_problem** out) {
  if (!cfg || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  Layout L;
  if (!make_layout(*cfg, L) || cfg->num_frames <= 0) return set_err(RCVD_ERR_INVALID, "unsupported transform configuration");
  if (int rc = check_device(device)) return rc;
  SET_DEVICE(device);
  {  // keep freed blocks in the device's default pool (released only on cudaDeviceReset / explicit trim)
    cudaMemPool_t pool; unsigned long long keep = ~0ull;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  rcvd_problem* p = new rcvd_problem();
  p->cfg = *cfg; p->L = L; p->N = cfg->num_frames; p->device = device;
  p->in_range.assign(p->N, 1); p->median.assign(p->N, 1.0); p->h_state.assign((size_t)p->N * L.nf, 0.0);
  cudaError_t e = cudaDeviceGetAttribute(&p->num_sms, cudaDevAttrMultiProcessorCount, device);   // read once: the plan and the launch shapes use it
  if (e == cudaSuccess) e = device_total_mem(device, &p->total_mem);                             // the solver choice (build_structure)
  if (e != cudaSuccess) { delete p; return set_err(RCVD_ERR_CUDA, "cudaDeviceGetAttribute / cudaGetDeviceProperties: %s", cudaGetErrorString(e)); }
  // the critical chain (potrf -> trsm -> next-level updates) runs at the highest priority, the overlapped updates at the lowest,
  // so that a freed SM goes to the chain first
  int prio_lo = 0, prio_hi = 0; cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  e = cudaStreamCreateWithPriority(&p->stream, cudaStreamNonBlocking, prio_hi);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&p->side_stream, cudaStreamNonBlocking, prio_lo);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&p->inv_stream, cudaStreamNonBlocking, prio_lo);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_inv_join, cudaEventDisableTiming);
  for (int i = 0; i < 8 && e == cudaSuccess; ++i) e = cudaEventCreate(&p->ev[i]);   // the timing events of rcvd_solve and the bench hooks
  if (e != cudaSuccess) { rcvd_problem_destroy(p); return set_err(RCVD_ERR_CUDA, "cudaStreamCreate / cudaEventCreate: %s", cudaGetErrorString(e)); }
  *out = p; return RCVD_OK;
}
RCVD_API void rcvd_problem_destroy(rcvd_problem* p) {
  if (!p) return;
  DevGuard dev_guard_(p->device);
  free_all(p);
  for (int i = 0; i < 8; ++i) if (p->ev[i]) cudaEventDestroy(p->ev[i]);
  if (p->comm && nccl::CommDestroy) nccl::CommDestroy(p->comm);
  if (p->ev_fork) cudaEventDestroy(p->ev_fork);
  if (p->ev_join) cudaEventDestroy(p->ev_join);
  for (cudaEvent_t e : p->ev_side) cudaEventDestroy(e);
  if (p->ev_inv_join) cudaEventDestroy(p->ev_inv_join);
  if (p->side_stream) cudaStreamDestroy(p->side_stream);
  if (p->inv_stream) cudaStreamDestroy(p->inv_stream);
  if (p->stream) cudaStreamDestroy(p->stream);
  delete p;
}
RCVD_API int32_t rcvd_problem_set_frames(rcvd_problem* p, const uint8_t* in_range, const double* median, const double* adaptive) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  const bool grid = adaptive && p->cfg.depth_type == RCVD_DEPTH_GRID;
  if (p->cfg.adaptive_deform > 0.0 && !grid) return set_err(RCVD_ERR_INVALID, "adaptive deformation cost requires node weights");
  if (int rc = drop_structure(p)) return rc;
  if (in_range) p->in_range.assign(in_range, in_range + p->N); else p->in_range.assign(p->N, 1);
  if (median) p->median.assign(median, median + p->N); else p->median.assign(p->N, 1.0);
  if (grid) p->adaptive.assign(adaptive, adaptive + (size_t)p->N * p->cfg.depth_grid_x * p->cfg.depth_grid_y); else p->adaptive.clear();
  return RCVD_OK;
}
// The setter of every family.  Everything is checked before anything is kept, so a refused call leaves the problem as it was:
// n groups of frames[n][nframes], offsets[n + 1] from 0, non-decreasing, records[offsets[n]][width].
static int32_t set_records(rcvd_problem* p, RecordSet rcvd_problem::*family, const char* what, int32_t n, const int32_t* frames, const int64_t* off,
                           const float* rec) {
  if (!p || n < 0 || (n > 0 && (!frames || !off))) return set_err(RCVD_ERR_INVALID, "bad %s arrays", what);
  RecordSet& s = p->*family;
  if (n > 0 && off[0] != 0) return set_err(RCVD_ERR_INVALID, "%s offsets must start at 0", what);
  for (int i = 0; i < n; ++i) {
    if (off[i + 1] < off[i]) return set_err(RCVD_ERR_INVALID, "%s offsets must be non-decreasing", what);
    const int32_t* f = frames + (size_t)i * s.nframes;
    const bool ok = s.nframes == 2 ? f[0] >= 0 && f[0] < p->N && f[1] >= 0 && f[1] < p->N && f[0] != f[1]   // two distinct frames
                                   : f[0] >= 1 && f[0] < p->N - 1;                                         // a centre with two neighbours
    if (!ok) return set_err(RCVD_ERR_INVALID, "bad %s group %d", what, i);
  }
  const int64_t count = n > 0 ? off[n] : 0;
  if (count > 0 && !rec) return set_err(RCVD_ERR_INVALID, "null %s records", what);
  if (int rc = drop_structure(p)) return rc;
  s.frames.assign(frames, frames + (size_t)n * s.nframes);
  if (n > 0) s.offsets.assign(off, off + n + 1); else s.offsets.assign(1, 0);
  s.records.assign(rec, rec + (size_t)count * s.width);
  return RCVD_OK;
}
RCVD_API int32_t rcvd_problem_set_constraints(rcvd_problem* p, int32_t np, const int32_t* pf, const int64_t* off, const float* rec) {
  return set_records(p, &rcvd_problem::pairs, "constraint", np, pf, off, rec);
}
RCVD_API int32_t rcvd_problem_set_triplets(rcvd_problem* p, int32_t nt, const int32_t* centers, const int64_t* off, const float* rec) {
  return set_records(p, &rcvd_problem::trips, "triplet", nt, centers, off, rec);
}
RCVD_API int32_t rcvd_problem_set_depth_pairs(rcvd_problem* p, int32_t np, const int32_t* pf, const int64_t* off, const float* rec) {
  if (p && p->nranks > 1 && np > 0) return set_err(RCVD_ERR_INVALID, "depth-normalisation pairs are not sharded: they need a single-GPU problem (nranks = 1)");
  return set_records(p, &rcvd_problem::dpairs, "depth-pair", np, pf, off, rec);
}
// Global frame-pair graph for multi-GPU runs (every rank must build the same block structure).
RCVD_API int32_t rcvd_problem_set_structure(rcvd_problem* p, int32_t np, const int32_t* pf) {
  if (!p || np < 0 || (np > 0 && !pf)) return set_err(RCVD_ERR_INVALID, "bad structure arrays");
  if (int rc = drop_structure(p)) return rc;
  p->struct_pairs.assign(pf, pf + 2 * (size_t)np);
  return RCVD_OK;
}
RCVD_API int32_t rcvd_nccl_unique_id(uint8_t out[128]) {
  if (!nccl::load()) return set_err(RCVD_ERR_NCCL, "libnccl.so.2 not found");
  nccl::UniqueId id; const int r = nccl::GetUniqueId(&id);
  if (r != 0) return set_err(RCVD_ERR_NCCL, "ncclGetUniqueId failed (%d)", r);
  memcpy(out, id.internal, 128); return RCVD_OK;
}
RCVD_API int32_t rcvd_problem_init_comm(rcvd_problem* p, int32_t nranks, int32_t rank, const uint8_t uid[128]) {
  if (!p || nranks < 1 || rank < 0 || rank >= nranks) return set_err(RCVD_ERR_INVALID, "bad rank/nranks");
  if (nranks > 1) {
    if (!nccl::load()) return set_err(RCVD_ERR_NCCL, "libnccl.so.2 not found");
    SET_DEVICE(p->device);
    nccl::UniqueId id; memcpy(id.internal, uid, 128);
    const int r = nccl::CommInitRank(&p->comm, nranks, id, rank);
    if (r != 0) return set_err(RCVD_ERR_NCCL, "ncclCommInitRank failed: %s", nccl::GetErrorString ? nccl::GetErrorString(r) : "?");
  }
  if (int rc = drop_structure(p)) return rc;
  p->nranks = nranks; p->rank = rank;
  return RCVD_OK;
}
RCVD_API int32_t rcvd_problem_set_state(rcvd_problem* p, const double* x) {
  if (!p || !x) return set_err(RCVD_ERR_INVALID, "null argument");
  p->h_state.assign(x, x + p->h_state.size()); p->state_dirty = true;
  return RCVD_OK;
}
RCVD_API int32_t rcvd_problem_get_state(rcvd_problem* p, double* x) {
  if (!p || !x) return set_err(RCVD_ERR_INVALID, "null argument");
  if (!p->structure_ready || p->state_dirty) { std::copy(p->h_state.begin(), p->h_state.end(), x); return RCVD_OK; }
  SET_DEVICE(p->device);
  return download_frames(p, x, p->d_x, p->L.nf);
}
RCVD_API int32_t rcvd_evaluate(rcvd_problem* p, double* cost, double* gradient) {
  if (!p || !cost) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  CK(cudaMemsetAsync(p->d_scal, 0, SC_N * sizeof(double), p->stream));
  rc = enqueue_evaluate(p, p->d_x, gradient != nullptr, false, p->d_g, SC_COST); if (rc) return rc;
  rc = read_scalars(p); if (rc) return rc;
  *cost = p->h_scal[SC_COST];
  return gradient ? download_frames(p, gradient, p->d_g, p->L.npad) : RCVD_OK;
}
RCVD_API int32_t rcvd_normal_matrix_dense(rcvd_problem* p, double* Hout) {
  if (!p || !Hout) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  p->force_full_H = true;                       // debug view: every rank assembles the whole matrix
  rc = enqueue_evaluate(p, p->d_x, true, true, p->d_g, SC_COST);
  p->force_full_H = false;
  if (rc) return rc;
  const size_t U = (size_t)p->N * p->L.nf;
  double* d_out = nullptr;
  CK(cudaMalloc((void**)&d_out, U * U * sizeof(double)));
  CK(cudaMemsetAsync(d_out, 0, U * U * sizeof(double), p->stream));
  rc = launch(p, k_h_to_dense, dim3(nblk((size_t)p->L.nf * p->L.nf), (int)p->plan.hblocks.size()), 256, 0, p->stream, false, p->d_H, p->d_hblocks, (int)p->plan.hblocks.size(), d_out, p->N, p->L.nf, p->L.npad, p->d_uperm);
  cudaError_t e = rc ? cudaSuccess : cudaMemcpyAsync(Hout, d_out, U * U * sizeof(double), cudaMemcpyDeviceToHost, p->stream);
  cudaStreamSynchronize(p->stream); cudaFree(d_out);
  if (rc) return rc;
  if (e != cudaSuccess) return set_err(RCVD_ERR_CUDA, "copy failed: %s", cudaGetErrorString(e));
  return RCVD_OK;
}

// ---- per-block rows (rcvd_row_layout, rcvd_evaluate_rows) ----
// Most nodes one gather returns (gather_depth, gather_spatial): a bicubic gather drops the taps beyond the grid's edge.
static int depth_taps(const rcvd_config& c) {
  if (c.depth_type == RCVD_DEPTH_IDENTITY) return 0;
  if (c.depth_type == RCVD_DEPTH_GLOBAL) return 1;
  return c.depth_cubic ? std::min(4, c.depth_grid_x) * std::min(4, c.depth_grid_y) : 4;
}
static int spatial_taps(const rcvd_config& c) {
  switch (c.spatial_type) {
    case RCVD_SPATIAL_VERTICAL_LINEAR: return 2;
    case RCVD_SPATIAL_CORNERS_BILINEAR: case RCVD_SPATIAL_BILINEAR_GRID: return 4;
    case RCVD_SPATIAL_BICUBIC_GRID: return std::min(4, c.spatial_grid_x) * std::min(4, c.spatial_grid_y);
    default: return 0;
  }
}
// The regulariser rows in the CPU oracle's order: every in-range frame in the caller's order with its scale rows, its deformation rows
// (grid node x + y*gx after node: the edge to the node on its left, then to the node above, k components each), its spatial rows and
// its focal row; then three position rows per frame triplet (f, f+1, f+2) that k_regularisers evaluates.  Returns the number of rows;
// slot (optional) receives the row of every k_regularisers row id, -1 where the id has none.  uperm: internal -> the caller's frame.
static int64_t regulariser_rows(const rcvd_problem* p, const std::vector<int>& uperm, std::vector<int32_t>* slot) {
  const rcvd_config& c = p->cfg; const Layout& L = p->L; const int N = p->N;
  const RegCounts rc = reg_counts(c, L, N, std::max(0, c.scale_grid_x) * std::max(0, c.scale_grid_y));
  std::vector<int> deform(rc.deform);      // kernel order (the horizontal edges, then the vertical ones) -> the oracle's
  if (rc.deform > 0) {
    const int gx = c.depth_grid_x, gy = c.depth_grid_y, nh = (gx - 1) * gy; int q = 0;
    for (int y = 0; y < gy; ++y) for (int x = 0; x < gx; ++x) {
      if (x > 0) for (int j = 0; j < L.k; ++j) deform[(y * (gx - 1) + x - 1) * L.k + j] = q++;
      if (y > 0) for (int j = 0; j < L.k; ++j) deform[(nh + (y - 1) * gx + x) * L.k + j] = q++;
    }
  }
  std::vector<int> rank(N, -1); int nin = 0, first = -1, last = -1;
  for (int u = 0; u < N; ++u) if (p->in_range[u]) { rank[u] = nin++; if (first < 0) first = u; last = u; }
  if (slot) slot->assign(rc.total, -1);
  for (int i = 0; i < N && slot; ++i) {
    const int u = uperm[i];
    if (rank[u] < 0) continue;
    for (int k = 0; k < rc.per_frame; ++k) {
      const int d = k - rc.scale;
      (*slot)[(size_t)i * rc.per_frame + k] = rank[u] * rc.per_frame + ((d >= 0 && d < rc.deform) ? rc.scale + deform[d] : k);
    }
  }
  int64_t n = (int64_t)nin * rc.per_frame;
  // k_regularisers' test on internal frames f (position rows keep the caller's frame order: make_factor_plan at one rank)
  auto in = [&](int f) { return p->in_range[uperm[f]] != 0; };
  for (int f = 0; rc.position_rows > 0 && f < N - 2; ++f) {
    if (f < first || f >= last - 1 || !in(f) || !in(f + 1) || !in(f + 2)) continue;
    for (int i = 0; i < 3; ++i) { if (slot) (*slot)[(size_t)rc.per_frame * N + 3 * f + i] = (int32_t)n; ++n; }
  }
  return n;
}
static rcvd_row_family row_family(const rcvd_problem* p, int family) {
  const rcvd_config& c = p->cfg; const Layout& L = p->L;
  const int depth = c.fix_depth_xforms ? 0 : depth_taps(c) * L.k, spatial = c.fix_spatial_xforms ? 0 : spatial_taps(c) * 2;
  const int frame = (c.fix_poses ? 0 : 6) + (c.intr_opt == RCVD_INTR_PER_FRAME ? 1 : 0) + depth + spatial;   // columns of one frame
  const int shared = c.intr_opt == RCVD_INTR_SHARED ? 1 : 0;
  switch (family) {
    case RCVD_ROWS_PAIRS: return {p->pairs.count(), 3, 2 * frame + shared};
    case RCVD_ROWS_TRIPLETS: return {p->trips.count(), 3, 3 * frame + shared};
    case RCVD_ROWS_DEPTH_PAIRS: return {p->dpairs.count(), 1, 2 * depth};
    default: {
      std::vector<int> identity(p->N);
      for (int i = 0; i < p->N; ++i) identity[i] = i;
      const RegCounts rc = reg_counts(c, L, p->N, std::max(0, c.scale_grid_x) * std::max(0, c.scale_grid_y));
      int K = 0;   // scale rows: the nodes of one depth gather; deformation: two nodes; spatial, focal: one parameter; position: three
      if (rc.scale) K = std::max(K, depth);
      if (rc.deform && !c.fix_depth_xforms) K = std::max(K, 2);
      if (rc.spatial && !c.fix_spatial_xforms) K = std::max(K, 1);
      if (rc.focal) K = std::max(K, 1);
      if (rc.position_rows && !c.fix_poses) K = std::max(K, 3);
      return {regulariser_rows(p, identity, nullptr), 1, K};
    }
  }
}
static int check_rows_handle(const rcvd_problem* p) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  if (p->nranks > 1) return set_err(RCVD_ERR_INVALID, "rows of a sharded problem (nranks > 1) are not available");
  return RCVD_OK;
}
// Launches the family's kernel in the Rows mode: from the caller's record order (not the run path's sorted copy), at the current state.
static int enqueue_rows(rcvd_problem* p, int family, bool jac, const RowOut& o) {
  DevProblem d = dev_problem(p);
  d.pairs.records = p->pairs.caller_records;
  const double* x = p->d_x; cudaStream_t st = p->stream;
  switch (family) {
    case RCVD_ROWS_PAIRS:
      return launch(p, jac ? k_pairs<EvalMode::Rows, true> : k_pairs<EvalMode::Rows, false>, p->pairs.num_tiles, kTile, 0, st, false,
                    d, x, nullptr, nullptr, nullptr, nullptr, o);
    case RCVD_ROWS_TRIPLETS:
      return launch(p, jac ? k_triplets<EvalMode::Rows, true> : k_triplets<EvalMode::Rows, false>, p->trips.num_tiles, kTile, 0, st, false,
                    d, x, nullptr, nullptr, nullptr, nullptr, o);
    case RCVD_ROWS_DEPTH_PAIRS:
      return launch(p, jac ? k_depth_pairs<EvalMode::Rows, true> : k_depth_pairs<EvalMode::Rows, false>, p->dpairs.num_tiles, kTile, 0, st, false,
                    d, x, nullptr, nullptr, nullptr, nullptr, o);
    default:
      return launch(p, jac ? k_regularisers<EvalMode::Rows, true> : k_regularisers<EvalMode::Rows, false>, p->part_trip - p->part_reg, 128, 0, st,
                    false, d, reg_counts(p->cfg, p->L, p->N, p->nscale), x, nullptr, nullptr, nullptr, nullptr, p->first_frame, p->last_frame, o);
  }
}
RCVD_API int32_t rcvd_row_layout(rcvd_problem* p, struct rcvd_row_layout* out) {
  if (int rc = check_rows_handle(p)) return rc;
  if (!out) return set_err(RCVD_ERR_INVALID, "null argument");
  for (int f = 0; f < RCVD_ROW_FAMILIES; ++f) out->family[f] = row_family(p, f);
  return RCVD_OK;
}
RCVD_API int32_t rcvd_evaluate_rows(rcvd_problem* p, int32_t family, double* residuals, double* rho, int32_t* cols, double* jac) {
  if (int rc = check_rows_handle(p)) return rc;
  if (family < 0 || family >= RCVD_ROW_FAMILIES) return set_err(RCVD_ERR_INVALID, "unknown row family %d", family);
  if ((cols == nullptr) != (jac == nullptr)) return set_err(RCVD_ERR_INVALID, "cols and jac go together: pass both or neither");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  rcvd_row_family fam = row_family(p, family);
  std::vector<int32_t> slot;
  if (family == RCVD_ROWS_REGULARISERS) fam.blocks = regulariser_rows(p, p->plan.uperm, &slot);
  if (fam.blocks == 0) return RCVD_OK;
  const bool want_jac = jac != nullptr;
  const size_t nb = (size_t)fam.blocks, nr = nb * fam.residuals, nj = want_jac ? nr * fam.max_cols : 0;
  // one device buffer: r [nr] | rho [nb] | jac [nj] | cols [nj] | regulariser slots
  char* buf = nullptr;
  CK(cudaMallocAsync((void**)&buf, std::max<size_t>((nr + nb + nj) * sizeof(double) + (nj + slot.size()) * sizeof(int32_t), 8), p->stream));
  RowOut o;
  o.r = (double*)buf; o.rho = o.r + nr; o.jac = o.rho + nb; o.cols = (int32_t*)(o.jac + nj);
  o.K = fam.max_cols; o.uperm = p->d_uperm; o.slot = o.cols + nj;
  auto run = [&]() -> int {
    if (!slot.empty()) CK(cudaMemcpyAsync((void*)o.slot, slot.data(), slot.size() * sizeof(int32_t), cudaMemcpyHostToDevice, p->stream));
    if (int rc2 = enqueue_rows(p, family, want_jac, o)) return rc2;
    if (residuals) CK(cudaMemcpyAsync(residuals, o.r, nr * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    if (rho) CK(cudaMemcpyAsync(rho, o.rho, nb * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    if (want_jac) {
      CK(cudaMemcpyAsync(jac, o.jac, nj * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
      CK(cudaMemcpyAsync(cols, o.cols, nj * sizeof(int32_t), cudaMemcpyDeviceToHost, p->stream));
    }
    return RCVD_OK;
  };
  rc = run();
  cudaFreeAsync(buf, p->stream);
  const cudaError_t e = cudaStreamSynchronize(p->stream);
  if (rc) return rc;
  if (e != cudaSuccess) return set_err(RCVD_ERR_CUDA, "rcvd_evaluate_rows: %s", cudaGetErrorString(e));
  return RCVD_OK;
}
// factorisation + solve of (S H S + diag(D2)) y = b with the H blocks already on the device; S == nullptr: S = 1
static int solve_loaded(rcvd_problem* p, const double* S, const double* D2, const double* b, double* y) {
  const std::vector<int>& uperm = p->plan.uperm; const int nf = p->L.nf, npad = p->L.npad; const size_t Upad = (size_t)p->N * npad;
  const std::vector<double> hs = S ? frames_to_internal(uperm, S, nf, npad, nf, 1.0) : std::vector<double>(Upad, 1.0);
  const std::vector<double> hd = frames_to_internal(uperm, D2, nf, npad, nf, 1.0), hb = frames_to_internal(uperm, b, nf, npad, nf, 0.0);
  CK(cudaMemcpyAsync(p->d_S, hs.data(), Upad * 8, cudaMemcpyHostToDevice, p->stream));
  CK(cudaMemcpyAsync(p->d_D2, hd.data(), Upad * 8, cudaMemcpyHostToDevice, p->stream));
  CK(cudaMemcpyAsync(p->d_gs, hb.data(), Upad * 8, cudaMemcpyHostToDevice, p->stream));
  CK(cudaMemsetAsync(p->d_fail, 0, sizeof(int), p->stream));
  int rc = linear_solve(p); if (rc) return rc;
  std::vector<double> hy(Upad);
  CK(cudaMemcpyAsync(hy.data(), p->d_y, Upad * 8, cudaMemcpyDeviceToHost, p->stream));
  rc = read_scalars(p); if (rc) return rc;
  frames_to_caller(uperm, hy.data(), npad, y, nf, nf);
  if (*p->h_fail) return set_err(RCVD_ERR_NUMERIC, p->use_cg ? "conjugate gradients broke down, or a diagonal block hit a non-positive pivot"
                                                          : "factorisation hit a non-positive pivot");
  return RCVD_OK;
}
// Debug/test: solve (S H S + diag(D2)) y = b with H = J^T J at the current state.
// S, D2, b, y: N*stride host doubles.
RCVD_API int32_t rcvd_debug_linear_solve(rcvd_problem* p, const double* S, const double* D2, const double* b, double* y) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  rc = enqueue_evaluate(p, p->d_x, true, true, p->d_g, SC_COST); if (rc) return rc;
  return solve_loaded(p, S, D2, b, y);
}
// Test hook: (H + diag(D2)) y = b for a caller-supplied dense symmetric H (U x U, U = N * stride, caller's frame order) through the
// production factorisation graph with S = 1.  H is scattered into the H blocks of the problem's frame graph (no evaluation); an entry
// in a frame pair the graph does not couple is an error.
// H (dense U x U, caller's frame order) into the H blocks of the handle's frame graph; an entry in a frame pair the graph does not couple
// is an error
static int scatter_matrix(rcvd_problem* p, const double* H) {
  const int N = p->N, nf = p->L.nf, npad = p->L.npad; const size_t U = (size_t)N * nf, bs = (size_t)npad * npad;
  std::vector<uint8_t> coupled((size_t)N * N, 0);
  for (const HBlock& hb : p->plan.hblocks) { const int a = p->plan.uperm[hb.r], c = p->plan.uperm[hb.c]; coupled[(size_t)a * N + c] = coupled[(size_t)c * N + a] = 1; }
  for (int a = 0; a < N; ++a) for (int c = 0; c < N; ++c) {
    if (coupled[(size_t)a * N + c]) continue;
    for (int i = 0; i < nf; ++i) for (int j = 0; j < nf; ++j)
      if (H[((size_t)a * nf + i) * U + (size_t)c * nf + j] != 0.0)
        return set_err(RCVD_ERR_INVALID, "H couples frames %d and %d, which the problem's frame graph does not couple", a, c);
  }
  std::vector<double> hH(p->plan.hblocks.size() * bs, 0.0);
  for (int h = 0; h < (int)p->plan.hblocks.size(); ++h) {        // block h holds rows of frame r, columns of frame c (internal ids)
    const int a = p->plan.uperm[p->plan.hblocks[h].r], c = p->plan.uperm[p->plan.hblocks[h].c];
    for (int i = 0; i < nf; ++i) for (int j = 0; j < nf; ++j) hH[h * bs + (size_t)i * npad + j] = H[((size_t)a * nf + i) * U + (size_t)c * nf + j];
  }
  CK(cudaMemcpyAsync(p->d_H, hH.data(), hH.size() * sizeof(double), cudaMemcpyHostToDevice, p->stream));
  return RCVD_OK;
}
static int debug_solve_matrix(rcvd_problem* p, const double* H, const double* D2, const double* b, double* y) {
  if (!p || !H || !D2 || !b || !y) return set_err(RCVD_ERR_INVALID, "null argument");
  if (p->nranks > 1) return set_err(RCVD_ERR_INVALID, "rcvd_debug_solve_matrix works on single-GPU handles only");
  if (p->eval_only) return set_err(RCVD_ERR_INVALID, "this handle was set to evaluation-only (rcvd_debug_set_eval_only): no factor storage");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  if ((rc = scatter_matrix(p, H))) return rc;
  return solve_loaded(p, nullptr, D2, b, y);
}
RCVD_API int32_t rcvd_debug_solve_matrix(rcvd_problem* p, const double* H, const double* D2, const double* b, double* y) {
  return debug_solve_matrix(p, H, D2, b, y);
}
// Test hook: the same system through the conjugate-gradient path (a handle whose structure chose it); iterations = the CG iterations run.
RCVD_API int32_t rcvd_debug_cg_solve_matrix(rcvd_problem* p, const double* H, const double* D2, const double* b, double* y, int32_t* iterations) {
  if (!p || !iterations) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  if (!p->use_cg) return set_err(RCVD_ERR_INVALID, "this handle solves with the block Cholesky: a factor budget of 0 (rcvd_debug_set_factor_budget) selects conjugate gradients");
  p->cg_last = 0;
  rc = debug_solve_matrix(p, H, D2, b, y);
  *iterations = p->cg_last;
  return rc;
}
// ---- marginal covariance blocks (rcvd_covariance; rcvd_selinv.cuh) ----
enum { SEL_PRODUCT = 0, SEL_TRMM, SEL_PIVOTS, SEL_GATHER, SEL_SCALE, SEL_N };   // rcvd_debug_covariance_launches
template <class... Params, class... Args>
static int sel_launch(rcvd_problem* p, int counter, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, Args... args) {
  if (int rc = launch(p, kernel, grid, block, smem, p->stream, false, args...)) return rc;
  p->sel_launches[counter]++;
  return RCVD_OK;
}
// The task lists of the selected inversion, once per structure
static int sel_prepare(rcvd_problem* p) {
  if (p->sel_ready) return RCVD_OK;
  make_sel_plan(p->sel, p->plan, p->N, p->L.npad, p->L.nf);
  int rc;
  if ((rc = upload(p, &p->d_sel_tiles, p->sel.tiles)) || (rc = upload(p, &p->d_sel_ops, p->sel.ops)) || (rc = upload(p, &p->d_sel_trmm, p->sel.trmm)) ||
      (rc = upload(p, &p->d_sel_row_off, p->sel.row_off)) || (rc = upload(p, &p->d_sel_row_blk, p->sel.row_blk))) return rc;
  CK(cudaFuncSetAttribute(k_selinv_trmm, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_trmm_smem_bytes(p->L.npad)));
  p->sel_ready = true;
  return RCVD_OK;
}
// The refusals that need no device
static int covariance_args(rcvd_problem* p, int32_t n, const int32_t* pairs, const double* out, double min_pivot) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  if (!out || n < 0 || (n > 0 && !pairs)) return set_err(RCVD_ERR_INVALID, "null argument");
  if (!(min_pivot >= 0.0) || !std::isfinite(min_pivot)) return set_err(RCVD_ERR_INVALID, "min_pivot must be finite and >= 0 (got %g)", min_pivot);
  if (p->nranks > 1) return set_err(RCVD_ERR_INVALID, "covariance of a sharded problem (nranks > 1) is not available");
  if (p->eval_only) return set_err(RCVD_ERR_INVALID, "this handle was set to evaluation-only (rcvd_debug_set_eval_only): no factor storage");
  for (int q = 0; q < 2 * n; ++q)
    if (pairs[q] < 0 || pairs[q] >= p->N) return set_err(RCVD_ERR_INVALID, "covariance block %d: frame %d is out of range [0, %d)", q / 2, pairs[q], p->N);
  return RCVD_OK;
}
// The refusals that need the structure, and the output blocks: a diagonal block, or the L block of an H block in either orientation
static int covariance_blocks(rcvd_problem* p, int32_t n, const int32_t* pairs, std::vector<SelGather>& gl) {
  if (p->use_cg) return set_err(RCVD_ERR_INVALID, "this handle solves with conjugate gradients (the block-Cholesky storage exceeds its budget): there is no factor to invert");
  const FactorPlan& pl = p->plan; const int N = p->N;
  gl.resize(n);
  for (int q = 0; q < n; ++q) {
    const int ia = pl.iperm[pairs[2 * q]], ib = pl.iperm[pairs[2 * q + 1]];
    if (ia == ib) { gl[q] = {ia, 0, ia, ia}; continue; }
    const int v = pl.blk_of[(size_t)ia * N + ib];
    if (v < 0) return set_err(RCVD_ERR_INVALID, "covariance block %d: frames %d and %d share no residual, so the normal matrix has no block (%d, %d)", q,
                              pairs[2 * q], pairs[2 * q + 1], pairs[2 * q], pairs[2 * q + 1]);
    const HBlock& hb = pl.hblocks[v >> 1];
    gl[q] = {hb.lblk, (v & 1) ? 0 : 1, hb.r, hb.c};
  }
  return RCVD_OK;
}
// Factorisation of S H S + D2 with the H already in d_H, the rank test, the selected inversion and the gather (see rcvd_covariance).
// problem_masks: also zero the parameters no residual touches and the frames out of range.
static int covariance_core(rcvd_problem* p, const uint8_t* hold, bool problem_masks, double min_pivot, const std::vector<SelGather>& gl, double* out,
                           double* min_pivot_seen) {
  const int N = p->N, nf = p->L.nf, npad = p->L.npad; const size_t Upad = (size_t)N * npad, nb = (size_t)nf * nf; cudaStream_t st = p->stream;
  int rc;
  if ((rc = sel_prepare(p))) return rc;
  const std::vector<uint8_t> hh = hold ? frames_to_internal<uint8_t>(p->plan.uperm, hold, nf, npad, nf, 0) : std::vector<uint8_t>(Upad, 0);
  // scratch: pivots [Upad] | output chunk | gather list | held mask
  const size_t chunk = std::max<size_t>(1, std::min<size_t>(gl.size(), ((size_t)64 << 20) / (nb * sizeof(double))));
  char* buf = nullptr;
  CK(cudaMallocAsync((void**)&buf, (Upad + chunk * nb) * sizeof(double) + std::max<size_t>(gl.size(), 1) * sizeof(SelGather) + Upad, st));
  double* d_piv = (double*)buf; double* d_out = d_piv + Upad; SelGather* d_gl = (SelGather*)(d_out + chunk * nb); uint8_t* d_hold = (uint8_t*)(d_gl + std::max<size_t>(gl.size(), 1));
  std::vector<double> piv(Upad), D2(Upad);
  const int* elim = p->plan.elim_order.data();
  int fail_frame = -1, fail_param = -1; double seen = std::numeric_limits<double>::infinity(), fail_value = 0.0;
  auto run = [&]() -> int {
    int r2;
    CK(cudaMemcpyAsync(d_hold, hh.data(), Upad, cudaMemcpyHostToDevice, st));
    if (!gl.empty()) CK(cudaMemcpyAsync(d_gl, gl.data(), gl.size() * sizeof(SelGather), cudaMemcpyHostToDevice, st));
    CK(cudaEventRecord(p->ev[0], st));
    if ((r2 = sel_launch(p, SEL_SCALE, k_selinv_scale, nblk(Upad), 256, 0, p->d_H, (const uint8_t*)d_hold, problem_masks ? (const uint8_t*)p->d_active : nullptr,
                         problem_masks ? (const uint8_t*)p->d_in_range : nullptr, p->d_S, p->d_D2, N, npad, nf))) return r2;
    CK(cudaMemsetAsync(p->d_gs, 0, Upad * sizeof(double), st));   // the factorisation graph's substitution solves for a zero right-hand side
    CK(cudaMemsetAsync(p->d_fail, 0, sizeof(int), st));
    if ((r2 = factor_solve(p))) return r2;
    if ((r2 = sel_launch(p, SEL_PIVOTS, k_selinv_pivots, dim3((nf + 7) / 8, N), 256, 0, (const double*)p->d_H, (const double*)p->d_Lb, (const double*)p->d_T,
                         (const double*)p->d_S, (const double*)p->d_D2, (const int*)p->d_sel_row_off, (const int*)p->d_sel_row_blk, npad, nf, d_piv))) return r2;
    CK(cudaEventRecord(p->ev[1], st));
    CK(cudaMemcpyAsync(piv.data(), d_piv, Upad * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(D2.data(), p->d_D2, Upad * sizeof(double), cudaMemcpyDeviceToHost, st));
    if ((r2 = read_scalars(p))) return r2;
    // the rank test: the first free parameter in elimination order whose pivot is <= min_pivot
    for (int q = 0; q < N && fail_frame < 0; ++q)
      for (int i = 0; i < nf; ++i) {
        const size_t v = (size_t)elim[q] * npad + i;
        if (D2[v] != 0.0) continue;                     // zeroed: a unit pivot of its own
        seen = std::min(seen, piv[v]);
        if (!(piv[v] > min_pivot)) { fail_frame = p->plan.uperm[elim[q]]; fail_param = i; fail_value = piv[v]; break; }
      }
    if (min_pivot_seen) *min_pivot_seen = fail_frame >= 0 ? fail_value : seen;
    if (fail_frame >= 0)
      return set_err(RCVD_ERR_NUMERIC, "covariance: the Jacobi-scaled normal matrix is rank-deficient: pivot %.3e <= min_pivot %.3e at frame %d, parameter %d "
                     "(hold the parameters of the gauge, e.g. one frame's pose)", fail_value, min_pivot, fail_frame, fail_param);
    if (*p->h_fail) return set_err(RCVD_ERR_NUMERIC, "covariance: the factorisation hit a non-positive pivot");
    // the selected inversion, levels in reverse
    CK(cudaEventRecord(p->ev[2], st));
    for (const SelLevel& sl : p->sel.levels) {
      if (sl.n[0] > 0 && (r2 = sel_launch(p, SEL_PRODUCT, k_selinv_product, sl.n[0], kSelThreads, 0, p->d_Lb, (const double*)p->d_T, (const double*)p->d_invL,
                                          (const SelTile*)p->d_sel_tiles + sl.off[0], (const SelOp*)p->d_sel_ops, npad, 1.0))) return r2;
      if (sl.n[1] > 0 && (r2 = sel_launch(p, SEL_TRMM, k_selinv_trmm, dim3(npad / kSelStrip, sl.n[1]), kSelThreads, sel_trmm_smem_bytes(npad), p->d_Lb,
                                          (const double*)p->d_invL, (const SelTrmm*)p->d_sel_trmm + sl.off[1], npad, -1.0, 0))) return r2;
      if (sl.n[2] > 0 && (r2 = sel_launch(p, SEL_PRODUCT, k_selinv_product, sl.n[2], kSelThreads, 0, p->d_Lb, (const double*)p->d_T, (const double*)p->d_invL,
                                          (const SelTile*)p->d_sel_tiles + sl.off[2], (const SelOp*)p->d_sel_ops, npad, -1.0))) return r2;
      if (sl.n[3] > 0 && (r2 = sel_launch(p, SEL_TRMM, k_selinv_trmm, dim3(npad / kSelStrip, sl.n[3]), kSelThreads, sel_trmm_smem_bytes(npad), p->d_Lb,
                                          (const double*)p->d_invL, (const SelTrmm*)p->d_sel_trmm + sl.off[3], npad, 1.0, 1))) return r2;
    }
    CK(cudaEventRecord(p->ev[3], st));
    for (size_t c0 = 0; c0 < gl.size(); c0 += chunk) {
      const size_t cnt = std::min(chunk, gl.size() - c0);
      if ((r2 = sel_launch(p, SEL_GATHER, k_selinv_gather, dim3(nblk(nb), (unsigned)cnt), 256, 0, (const double*)p->d_Lb, (const double*)p->d_S,
                           (const SelGather*)d_gl + c0, npad, nf, d_out))) return r2;
      CK(cudaMemcpyAsync(out + c0 * nb, d_out, cnt * nb * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    CK(cudaEventRecord(p->ev[4], st));
    CK(cudaStreamSynchronize(st));
    p->sel_ms[0] = ev_ms(p->ev[0], p->ev[1]); p->sel_ms[1] = ev_ms(p->ev[2], p->ev[3]); p->sel_ms[2] = ev_ms(p->ev[3], p->ev[4]);
    return RCVD_OK;
  };
  rc = run();
  p->factored = false;                // Lb holds Z now, not the factor
  cudaFreeAsync(buf, st);
  const cudaError_t e = cudaStreamSynchronize(st);
  if (rc) return rc;
  if (e != cudaSuccess) return set_err(RCVD_ERR_CUDA, "rcvd_covariance: %s", cudaGetErrorString(e));
  return RCVD_OK;
}
RCVD_API int32_t rcvd_covariance(rcvd_problem* p, const uint8_t* hold, double min_pivot, int32_t num_blocks, const int32_t* frame_pairs, double* out,
                                 double* min_pivot_seen) {
  if (int rc = covariance_args(p, num_blocks, frame_pairs, out, min_pivot)) return rc;
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  std::vector<SelGather> gl;
  if ((rc = covariance_blocks(p, num_blocks, frame_pairs, gl))) return rc;
  if ((rc = enqueue_evaluate(p, p->d_x, true, true, p->d_g, SC_COST))) return rc;
  return covariance_core(p, hold, true, min_pivot, gl, out, min_pivot_seen);
}
RCVD_API int32_t rcvd_debug_covariance_matrix(rcvd_problem* p, const double* H, const uint8_t* hold, int32_t num_blocks, const int32_t* frame_pairs,
                                              double* out) {
  if (int rc = covariance_args(p, num_blocks, frame_pairs, out, 1e-10)) return rc;
  if (!H) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  std::vector<SelGather> gl;
  if ((rc = covariance_blocks(p, num_blocks, frame_pairs, gl)) || (rc = scatter_matrix(p, H))) return rc;
  return covariance_core(p, hold, false, 1e-10, gl, out, nullptr);
}
RCVD_API int32_t rcvd_debug_covariance_launches(rcvd_problem* p, int64_t out[5]) {
  if (!p || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  std::copy(p->sel_launches, p->sel_launches + SEL_N, out);
  return RCVD_OK;
}
RCVD_API int32_t rcvd_debug_covariance_profile(rcvd_problem* p, double out[5]) {
  if (!p || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  std::copy(p->sel_ms, p->sel_ms + 3, out);
  out[3] = p->sel_ready ? p->sel.flops : 0.0; out[4] = p->sel_ready ? (double)p->sel.products : 0.0;
  return RCVD_OK;
}
// Test hook: the factor the last factorisation left on the device (see include/rcvd_hooks.h).
RCVD_API int32_t rcvd_debug_factor_dense(rcvd_problem* p, int32_t* order, double* L, double* Linv) {
  if (!p || !order || !L) return set_err(RCVD_ERR_INVALID, "null argument");
  if (p->structure_ready && p->use_cg) return set_err(RCVD_ERR_INVALID, "this handle solves with conjugate gradients: there is no factor");
  if (!p->structure_ready || !p->factored) return set_err(RCVD_ERR_INVALID, "no factorisation has run on this handle");
  if (p->plan.dist) return set_err(RCVD_ERR_INVALID, "the distributed factorisation keeps its blocks on their owners");
  SET_DEVICE(p->device);
  CK(cudaStreamSynchronize(p->side_stream)); CK(cudaStreamSynchronize(p->inv_stream)); CK(cudaStreamSynchronize(p->stream));
  const int N = p->N, nf = p->L.nf, npad = p->L.npad, nT = p->plan.nLoff; const size_t U = (size_t)N * nf, bs = (size_t)npad * npad;
  std::vector<double> hL((size_t)N * bs), hT((size_t)nT * bs);
  CK(cudaMemcpy(hL.data(), p->d_Lb, hL.size() * sizeof(double), cudaMemcpyDeviceToHost));   // the first N blocks: diagonal blocks L_kk
  if (nT > 0) CK(cudaMemcpy(hT.data(), p->d_T, hT.size() * sizeof(double), cudaMemcpyDeviceToHost));
  std::vector<size_t> off(N);
  for (int q = 0; q < N; ++q) { off[p->plan.elim_order[q]] = (size_t)q * nf; order[q] = p->plan.uperm[p->plan.elim_order[q]]; }
  std::fill(L, L + U * U, 0.0);
  for (int f = 0; f < N; ++f)                      // lower triangle only: the update epilogue may leave values above the diagonal
    for (int i = 0; i < nf; ++i) for (int j = 0; j <= i; ++j) L[(off[f] + i) * U + off[f] + j] = hL[f * bs + (size_t)i * npad + j];
  for (int t = 0; t < nT; ++t) {
    const HBlock& b = p->plan.lblocks[N + t];
    for (int i = 0; i < nf; ++i) for (int j = 0; j < nf; ++j) L[(off[b.r] + i) * U + off[b.c] + j] = hT[t * bs + (size_t)i * npad + j];
  }
  if (Linv) {
    CK(cudaMemcpy(hL.data(), p->d_invL, hL.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (int f = 0; f < N; ++f) {
      double* out = Linv + off[f] * nf;
      for (int i = 0; i < nf; ++i) for (int j = 0; j < nf; ++j) out[(size_t)i * nf + j] = j <= i ? hL[f * bs + (size_t)i * npad + j] : 0.0;
    }
  }
  return RCVD_OK;
}
RCVD_API int32_t rcvd_debug_pair_kernel_launches(rcvd_problem* p, int64_t out[3]) {
  if (!p || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  std::copy(p->pair_launches, p->pair_launches + 3, out);
  return RCVD_OK;
}
RCVD_API int32_t rcvd_debug_linear_paths(rcvd_problem* p, int64_t out[13]) {
  if (!p || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  static_assert(LP_N == 13, "include/rcvd_hooks.h documents thirteen counters");
  std::copy(p->paths, p->paths + LP_N, out);
  return RCVD_OK;
}
RCVD_API int32_t rcvd_time_accumulate(rcvd_problem* p, int32_t iters, double* ms) {
  if (!p || iters <= 0) return set_err(RCVD_ERR_INVALID, "bad argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  if ((rc = enqueue_evaluate(p, p->d_x, true, true, p->d_g, SC_COST))) return rc;   // warm-up
  CK(cudaEventRecord(p->ev[0], p->stream));
  for (int i = 0; i < iters; ++i) if ((rc = enqueue_evaluate(p, p->d_x, true, true, p->d_g, SC_COST))) return rc;
  CK(cudaEventRecord(p->ev[1], p->stream));
  CK(cudaStreamSynchronize(p->stream));
  *ms = ev_ms(p->ev[0], p->ev[1]) / iters;
  return RCVD_OK;
}
RCVD_API int32_t rcvd_time_iteration(rcvd_problem* p, int32_t iters, double radius, double* ms_iter, double* ms_acc, double* ms_lin, double* ms_cost) {
  if (!p || iters <= 0) return set_err(RCVD_ERR_INVALID, "bad argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  const size_t Upad = (size_t)p->N * p->L.npad; cudaStream_t st = p->stream;
  rcvd_solve_options o; rcvd_default_solve_options(&o);
  double ta = 0, tl = 0, tc = 0, tt = 0;
  for (int it = -1; it < iters; ++it) {   // it == -1: warm-up (also instantiates the graph)
    // the first iteration of rcvd_solve with the default options: assemble, Jacobi scaling, damped step, candidate cost
    CK(cudaMemsetAsync(p->d_scal, 0, SC_N * sizeof(double), st));
    CK(cudaMemsetAsync(p->d_fail, 0, sizeof(int), st));
    CK(cudaEventRecord(p->ev[0], st));
    if ((rc = enqueue_assemble(p))) return rc;
    if ((rc = launch(p, k_jacobi_scale, nblk(Upad), 256, 0, st, false, p->d_diagH, p->d_S, (int)Upad, o.jacobi_scaling))) return rc;
    CK(cudaEventRecord(p->ev[1], st));
    if ((rc = enqueue_damped_step(p, o, radius, false))) return rc;
    CK(cudaEventRecord(p->ev[2], st));
    if ((rc = enqueue_candidate_cost(p, 1.0, false))) return rc;
    CK(cudaEventRecord(p->ev[3], st));
    if ((rc = read_scalars(p))) return rc;
    if (it >= 0) { ta += ev_ms(p->ev[0], p->ev[1]); tl += ev_ms(p->ev[1], p->ev[2]); tc += ev_ms(p->ev[2], p->ev[3]); tt += ev_ms(p->ev[0], p->ev[3]); }
  }
  *ms_iter = tt / iters; if (ms_acc) *ms_acc = ta / iters; if (ms_lin) *ms_lin = tl / iters; if (ms_cost) *ms_cost = tc / iters;
  return RCVD_OK;
}
// Bench hook: the outputs of the last rcvd_time_iteration step (gradient, candidate state, cost, candidate cost), caller's frame order.
RCVD_API int32_t rcvd_debug_last_iteration(rcvd_problem* p, double* g, double* xc, double out[2]) {
  if (!p || !g || !xc || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  if (!p->structure_ready) return set_err(RCVD_ERR_INVALID, "no iteration has run on this handle");
  SET_DEVICE(p->device);
  int rc = read_scalars(p); if (rc) return rc;
  out[0] = p->h_scal[SC_COST]; out[1] = p->h_scal[SC_CAND];
  if ((rc = download_frames(p, g, p->d_g, p->L.npad))) return rc;
  return download_frames(p, xc, p->d_xc, p->L.nf);
}
// Bench hook: one factorisation + solve, un-captured on a single stream with one CUDA event per launch; returns the
// summed device time per kernel class: out_ms[0..5] = load, potrf, trinv, trsm, update GEMM (k_update_tma), substitution;
// out_ms[6] = number of k_update_tma launches, out_ms[7] = algorithmic flops of those GEMMs.
// reps < 0: keep the two-stream overlap (events on the main stream only: side-stream classes read ~0 and every wait for
// the side stream is charged to the next main-stream launch) -- shows where the chain is delayed by the overlapped work.
RCVD_API int32_t rcvd_debug_profile_linear(rcvd_problem* p, int32_t reps, double out_ms[8]) {
  const bool keep_overlap = reps < 0; if (reps < 0) reps = -reps;
  if (!p || !out_ms || reps == 0) return set_err(RCVD_ERR_INVALID, "bad argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  if (p->use_cg) return set_err(RCVD_ERR_INVALID, "this handle solves with conjugate gradients: there is no factorisation to profile");
  const bool ov = p->overlap; if (!keep_overlap) p->overlap = false;
  for (int i = 0; i < 8; ++i) out_ms[i] = 0.0;
  std::vector<std::pair<int, cudaEvent_t>> evs;
  p->level_ms.assign(p->plan.levels.size() * 6, 0.0);
  for (int r = -1; r < reps; ++r) {
    CK(cudaMemsetAsync(p->d_fail, 0, sizeof(int), p->stream));
    evs.clear(); p->prof = &evs;
    rc = enqueue_factor_solve(p);
    p->prof = nullptr; p->factored = true;
    cudaStreamSynchronize(p->stream); cudaStreamSynchronize(p->side_stream); cudaStreamSynchronize(p->inv_stream);
    double ngemm = 0;
    for (size_t i = 1; i < evs.size(); ++i) {
      float ms = 0; cudaEventElapsedTime(&ms, evs[i - 1].second, evs[i].second);
      const int cls = evs[i].first < 0 ? -1 : (evs[i].first & 0xff), lvl = evs[i].first < 0 ? 0 : (evs[i].first >> 8);
      if (r >= 0 && cls >= 0 && cls < 6) out_ms[cls] += ms;
      if (cls == 4) ngemm += 1;
      if (r == reps - 1 && cls >= 0 && cls < 6 && p->level_ms.size() >= (size_t)(lvl + 1) * 6) p->level_ms[(size_t)lvl * 6 + cls] += ms;
    }
    for (auto& e : evs) cudaEventDestroy(e.second);
    out_ms[6] = ngemm;
    if (rc) break;
  }
  p->overlap = ov;
  for (int i = 0; i < 6; ++i) out_ms[i] /= reps;
  out_ms[7] = p->plan.upd_flops;
  return rc;
}
// Bench hook: fp64 tensor-core (DMMA) peak of this device for one mma.sync shape, measured live with a register-only loop on all SMs:
// shape 0 = m8n8k4, 1 = m16n8k4, 2 = m16n8k8, 3 = m16n8k16.  The fastest shape is the denominator of the update-GEMM roofline.
template <int SHAPE>
__global__ void k_dmma_peak(double* out, int iters) {
  double c[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { c[i][0] = 0; c[i][1] = 0; c[i][2] = 0; c[i][3] = 0; }
  const double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (SHAPE == 0) dmma_8x8x4(c[i][0], c[i][1], a, b);
      if (SHAPE == 1) dmma_16x8x4(c[i][0], c[i][1], c[i][2], c[i][3], a, a, b);
      if (SHAPE == 2)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%4,%4,%4}, {%5,%5}, {%0,%1,%2,%3};"
                     : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3]) : "d"(a), "d"(b));
      if (SHAPE == 3)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%4,%4,%4,%4,%4,%4,%4}, {%5,%5,%5,%5}, {%0,%1,%2,%3};"
                     : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3]) : "d"(a), "d"(b));
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}
RCVD_API int32_t rcvd_debug_fp64_tensor_peak(int32_t device, int32_t shape, double* tflops) {
  if (!tflops || shape < 0 || shape > 3) return set_err(RCVD_ERR_INVALID, "bad argument");
  if (int rc = check_device(device)) return rc;
  SET_DEVICE(device);
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, device));
  const int threads = 512, blocks = prop.multiProcessorCount * 4, iters = 20000 >> shape;
  const double flops_per_mma = 512.0 * (1 << shape);      // 2*m*n*k: 512, 1024, 2048, 4096
  double* out = nullptr; CK(cudaMalloc((void**)&out, (size_t)blocks * threads * sizeof(double)));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  void (*const kernel)(double*, int) = shape == 0 ? k_dmma_peak<0> : shape == 1 ? k_dmma_peak<1> : shape == 2 ? k_dmma_peak<2> : k_dmma_peak<3>;
  double best = 0;
  int rc = RCVD_OK;
  for (int rep = 0; rep < 4; ++rep) {
    cudaEventRecord(e0);
    if ((rc = launch_kernel(kernel, blocks, threads, 0, nullptr, false, out, iters))) break;
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    const double tf = flops_per_mma * 8 * iters * (double)blocks * (threads / 32) / (ms * 1e-3) / 1e12;
    if (rep > 0 && tf > best) best = tf;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(out);
  if (rc) return rc;
  CK(cudaGetLastError());
  *tflops = best; return RCVD_OK;
}
// Test / bench hook: parity evidence at the size that is timed.  One LM trust-region step at the current state with the given radius
// (evaluate, Jacobi scaling, damped factorisation + substitution), then the residual of the linear system on the device:
//   out[0] = |(S H S + D2) y - S g| / |S g|   (k_spmv_sym over the assembled H, independent of the factorisation kernels)
//   out[1] = |S g|,  out[2] = cost,  out[3] = |g|_2,  out[4] = |y|_2,  out[5] = non-positive-pivot flag
__global__ void __launch_bounds__(256) k_lin_residual(const double* __restrict__ S, const double* __restrict__ HSy, const double* __restrict__ D2,
                                                       const double* __restrict__ y, const double* __restrict__ gs, const double* __restrict__ g,
                                                       int n, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double r2 = 0.0, b2 = 0.0, g2 = 0.0, y2 = 0.0;
  if (i < n) { const double r = S[i] * HSy[i] + D2[i] * y[i] - gs[i]; r2 = r * r; b2 = gs[i] * gs[i]; g2 = g[i] * g[i]; y2 = y[i] * y[i]; }
  r2 = warp_sum(r2); b2 = warp_sum(b2); g2 = warp_sum(g2); y2 = warp_sum(y2);
  if ((threadIdx.x & 31) == 0) { red_add(out + 0, r2); red_add(out + 1, b2); red_add(out + 2, g2); red_add(out + 3, y2); }
}
RCVD_API int32_t rcvd_debug_linear_residual(rcvd_problem* p, double radius, double out[6]) {
  if (!p || !out || !(radius > 0.0)) return set_err(RCVD_ERR_INVALID, "bad argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  const size_t Upad = (size_t)p->N * p->L.npad; cudaStream_t st = p->stream;
  rcvd_solve_options o; rcvd_default_solve_options(&o);
  CK(cudaMemsetAsync(p->d_scal, 0, SC_N * sizeof(double), st));
  CK(cudaMemsetAsync(p->d_fail, 0, sizeof(int), st));
  if ((rc = enqueue_assemble(p))) return rc;
  if ((rc = launch(p, k_jacobi_scale, nblk(Upad), 256, 0, st, false, p->d_diagH, p->d_S, (int)Upad, o.jacobi_scaling))) return rc;
  if ((rc = enqueue_damped_step(p, o, radius, false))) return rc;         // leaves H (S y) in d_Hy
  if (p->plan.dist && (rc = allreduce(p, p->d_Hy, Upad))) return rc;      // every rank multiplied only the H blocks it owns
  double* d_out = p->d_scal + 9;                                          // slots 9..12 are unused by the LM loop
  if ((rc = launch(p, k_lin_residual, nblk(Upad), 256, 0, st, false, p->d_S, p->d_Hy, p->d_D2, p->d_y, p->d_gs, p->d_g, (int)Upad, d_out))) return rc;
  if ((rc = read_scalars(p))) return rc;
  const double r2 = p->h_scal[9], b2 = p->h_scal[10];
  out[0] = b2 > 0.0 ? std::sqrt(r2 / b2) : std::sqrt(r2); out[1] = std::sqrt(b2); out[2] = p->h_scal[SC_COST];
  out[3] = std::sqrt(p->h_scal[11]); out[4] = std::sqrt(p->h_scal[12]); out[5] = (double)*p->h_fail;
  return RCVD_OK;
}
// per-level view of the last rcvd_debug_profile_linear call: out[level][6] = ms of {load, potrf, trinv, trsm, update, substitution}; returns levels
RCVD_API int32_t rcvd_debug_level_profile(rcvd_problem* p, double* out, int32_t max_levels) {
  if (!p || !out) return -1;
  const int n = std::min<int>(max_levels, (int)(p->level_ms.size() / 6));
  for (int i = 0; i < n * 6; ++i) out[i] = p->level_ms[i];
  return n;
}
RCVD_API int64_t rcvd_launch_count(rcvd_problem* p) { return p ? p->launches : 0; }
// Test / bench hook: elimination-order variant (-1 greedy minimum degree, >= 0 multiple elimination with that degree slack).
RCVD_API int32_t rcvd_debug_set_order_slack(rcvd_problem* p, int32_t slack) { if (!p) return set_err(RCVD_ERR_INVALID, "null problem"); if (int rc = drop_structure(p)) return rc; p->order_slack = slack; return RCVD_OK; }
// Test / bench hook: 0 = single-stream factorisation graph, 1 (default) = overlap non-critical updates on a second stream.
RCVD_API int32_t rcvd_debug_set_overlap(rcvd_problem* p, int32_t on) { if (!p) return set_err(RCVD_ERR_INVALID, "null problem"); p->overlap = on != 0; drop_graph(p); return RCVD_OK; }
// Test / bench hook: side_items_per_cta > 0 caps the items per CTA of the one-team update launches (a larger grid); 0 (default) = no cap.
// tma must be 1: the persistent TMA-fed kernel (k_update_tma) is the only update kernel.
RCVD_API int32_t rcvd_debug_set_update_kernel(rcvd_problem* p, int32_t tma, int32_t side_items_per_cta) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  if (!tma) return set_err(RCVD_ERR_INVALID, "the cp.async update path was removed: k_update_tma is the only update kernel");
  p->upd_ipc = side_items_per_cta; drop_graph(p); return RCVD_OK;
}
// Test / bench hook: the order of k_update_tma's items within each launch: 1 (default) = locality order, 0 = sorted by cost.
RCVD_API int32_t rcvd_debug_set_update_order(rcvd_problem* p, int32_t order) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  if (order < 0 || order > 1) return set_err(RCVD_ERR_INVALID, "update order must be 0 or 1 (got %d)", order);
  p->upd_order = order; drop_graph(p); return RCVD_OK;
}
// Test / bench hook: 1 = the handle will only evaluate cost / gradient (rcvd_evaluate): no normal matrix, no factor storage is allocated
RCVD_API int32_t rcvd_debug_set_eval_only(rcvd_problem* p, int32_t on) { if (!p) return set_err(RCVD_ERR_INVALID, "null problem"); if (int rc = drop_structure(p)) return rc; p->eval_only = on != 0; return RCVD_OK; }
// Test / bench hook (nranks > 1): 1 (default) = distributed factorisation (owner-computes phase A, reduce-to-owner of H), 0 = replicated scheme
// (all-reduce of H, factorisation replicated on every rank).
RCVD_API int32_t rcvd_debug_set_distributed(rcvd_problem* p, int32_t on) { if (!p) return set_err(RCVD_ERR_INVALID, "null problem"); if (int rc = drop_structure(p)) return rc; p->dist_enabled = on != 0; return RCVD_OK; }
RCVD_API int32_t rcvd_distribution_info(rcvd_problem* p, int32_t out[4]) {
  if (!p || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  out[0] = p->plan.dist ? 1 : 0; out[1] = p->plan.LB; out[2] = (int)p->plan.levels.size(); out[3] = p->plan.dist ? p->plan.fa_cnt[p->rank] + p->plan.fb_cnt[p->rank] : p->N;
  return RCVD_OK;
}
// Test hook: 0 = generic accumulate kernel (the tests' reference), 1 (default) = specialised kernels (run path on a bilinear depth grid),
// 2 = k_accumulate_fast even where the run path applies (sorted records are valid input for it): the only way to run its Grid branch
// below 65535 grid nodes.
RCVD_API int32_t rcvd_debug_set_fast_path(rcvd_problem* p, int32_t on) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  if (on < 0 || on > 2) return set_err(RCVD_ERR_INVALID, "fast path switch must be 0, 1 or 2 (got %d)", on);
  p->fast_path = on; return RCVD_OK;
}
RCVD_API int32_t rcvd_solve(rcvd_problem* p, const rcvd_solve_options* opt, rcvd_solve_summary* summary) {
  if (!p || !summary) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  rcvd_solve_options o; if (opt) o = *opt; else rcvd_default_solve_options(&o);
  return lm_solve(p, o, *summary);
}
// The plan of rcvd_debug_factor_plan / rcvd_debug_update_passes: host only, no handle, no device.
static int32_t debug_plan(FactorPlan& pl, const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                          int32_t order_slack, int32_t nranks, int32_t rank, int32_t num_sms) {
  if (!cfg || np < 0 || nt < 0 || (np > 0 && !pairs) || (nt > 0 && !trip_centers)) return set_err(RCVD_ERR_INVALID, "null or negative argument");
  if (nranks < 1 || rank < 0 || rank >= nranks || num_sms < 1) return set_err(RCVD_ERR_INVALID, "bad rank/nranks/num_sms");
  if (const char* e = make_factor_plan(pl, *cfg, std::vector<int32_t>(pairs, pairs + 2 * (size_t)np), std::vector<int32_t>(trip_centers, trip_centers + nt),
                                       order_slack, nranks, rank, true, num_sms))
    return set_err(RCVD_ERR_INVALID, "%s", e);
  return RCVD_OK;
}
// Test hook: the factorisation plan of a frame graph, computed on the host alone -- no handle, no device (see include/rcvd_hooks.h).
RCVD_API int32_t rcvd_debug_factor_plan(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                                        int32_t order_slack, int32_t nranks, int32_t rank, int32_t num_sms,
                                        int32_t* order, int32_t* level, int32_t* owner, int32_t* perm, int32_t out[13]) {
  if (!order || !level || !owner || !perm || !out) return set_err(RCVD_ERR_INVALID, "null or negative argument");
  FactorPlan pl;
  if (int32_t rc = debug_plan(pl, cfg, np, pairs, nt, trip_centers, order_slack, nranks, rank, num_sms)) return rc;
  const int N = cfg->num_frames;
  frames_to_caller(pl.uperm, pl.level.data(), 1, level, 1, 1); frames_to_caller(pl.uperm, pl.owner.data(), 1, owner, 1, 1);
  for (int i = 0; i < N; ++i) { order[i] = pl.uperm[pl.elim_order[i]]; perm[i] = pl.uperm[i]; }
  const int32_t v[13] = {(int32_t)pl.levels.size(), pl.nLoff, (int32_t)pl.hblocks.size(), pl.upd_targets, (int32_t)pl.upd_items.size(), (int32_t)pl.sub_tasks.size(),
                         pl.dist ? 1 : 0, pl.LB, pl.sub_first_level, (int32_t)pl.own_lblocks.size(), (int32_t)pl.own_hblocks.size(),
                         pl.dist ? pl.fa_cnt[rank] + pl.fb_cnt[rank] : N, (int32_t)pl.upd_tasks.size()};
  std::copy(v, v + 13, out);
  return RCVD_OK;
}
// Test hook: the update passes of the plan of a frame graph (see include/rcvd_hooks.h).
RCVD_API int32_t rcvd_debug_update_passes(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                                          int32_t order_slack, int32_t nranks, int32_t rank, int32_t num_sms,
                                          int32_t* passes, int32_t* sources, int32_t* join, int32_t* flags, int32_t counts[5]) {
  if (!counts) return set_err(RCVD_ERR_INVALID, "null argument");
  FactorPlan pl;
  if (int32_t rc = debug_plan(pl, cfg, np, pairs, nt, trip_centers, order_slack, nranks, rank, num_sms)) return rc;
  const int32_t need[3] = {(int32_t)pl.upd_tasks.size(), (int32_t)pl.upd_pairs.size(), 2 * (int32_t)pl.levels.size()};
  if (passes) {
    if (!sources || !join || !flags || counts[0] < need[0] || counts[1] < need[1] || counts[2] < need[2]) return set_err(RCVD_ERR_INVALID, "null or short output array");
    const int N = cfg->num_frames;
    for (size_t l = 0; l < pl.levels.size(); ++l) {
      const Level& lv = pl.levels[l];
      join[2 * l] = lv.join[0]; join[2 * l + 1] = lv.join[1];
      for (int q = lv.upd_off; q < lv.upd2_off[1] + lv.nupd2[1]; ++q) {
        const UpdPass& t = pl.upd_tasks[q];
        const HBlock& b = pl.lblocks[t.dst];
        int32_t* o = passes + 5 * (size_t)q;
        o[0] = pl.uperm[b.r]; o[1] = pl.uperm[b.c]; o[2] = (int32_t)l; o[3] = q >= lv.upd2_off[1] ? 2 : q >= lv.upd2_off[0] ? 1 : 0; o[4] = t.count;
        flags[q] = t.flags;
        for (int i = 0; i < t.count; ++i) sources[t.first + i] = pl.uperm[pl.lblocks[N + pl.upd_pairs[t.first + i].x].c];
      }
    }
  }
  std::copy(need, need + 3, counts); counts[3] = pl.TB; counts[4] = pl.upd_window;
  return RCVD_OK;
}
// Test hook: the update items of the plan of a frame graph, launch by launch (see include/rcvd_hooks.h).
RCVD_API int32_t rcvd_debug_update_items(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                                         int32_t order_slack, int32_t nranks, int32_t rank, int32_t num_sms, int32_t order,
                                         int32_t* items, int32_t* launches, int32_t* products, int32_t counts[5]) {
  if (!counts) return set_err(RCVD_ERR_INVALID, "null argument");
  if (order < 0 || order > 1) return set_err(RCVD_ERR_INVALID, "update order must be 0 or 1 (got %d)", order);
  FactorPlan pl;
  if (int32_t rc = debug_plan(pl, cfg, np, pairs, nt, trip_centers, order_slack, nranks, rank, num_sms)) return rc;
  const int32_t need[3] = {(int32_t)pl.upd_items.size(), 3 * (int32_t)pl.levels.size(), (int32_t)pl.upd_pairs.size()};
  if (items) {
    if (!launches || !products || counts[0] < need[0] || counts[1] < need[1] || counts[2] < need[2]) return set_err(RCVD_ERR_INVALID, "null or short output array");
    const std::vector<UpdItem>& v = order ? pl.upd_items : pl.upd_items_cost;
    for (size_t i = 0; i < v.size(); ++i) {
      const int32_t o[8] = {v[i].dst, v[i].first, v[i].count, v[i].m0, v[i].n0, v[i].mrows, v[i].ncols, v[i].flags};
      std::copy(o, o + 8, items + 8 * i);
    }
    for (size_t l = 0; l < pl.levels.size(); ++l) {
      const Level& lv = pl.levels[l];
      const int32_t o[6] = {lv.it_off, lv.nit, lv.it2_off[0], lv.nit2[0], lv.it2_off[1], lv.nit2[1]};
      std::copy(o, o + 6, launches + 6 * l);
    }
    for (size_t q = 0; q < pl.upd_pairs.size(); ++q) { products[2 * q] = pl.upd_pairs[q].x; products[2 * q + 1] = pl.upd_pairs[q].y; }
  }
  Layout L; make_layout(*cfg, L);
  std::copy(need, need + 3, counts); counts[3] = pl.upd_neff; counts[4] = L.npad;
  return RCVD_OK;
}
RCVD_API int32_t rcvd_problem_linear_info(rcvd_problem* p, rcvd_linear_info* out) {
  if (!p || !out) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  *out = rcvd_linear_info{};
  out->solver = p->use_cg ? RCVD_LINEAR_CG : RCVD_LINEAR_CHOLESKY;
  out->factor_blocks = p->eval_only ? 0 : p->use_cg ? p->N : p->N + p->plan.nLoff + std::max(p->plan.nLoff, 1);
  out->device_bytes = p->eval_only ? 0 : p->linear_bytes;
  out->cholesky_bytes = p->storage.cholesky; out->cg_bytes = p->storage.cg;
  out->budget_bytes = p->factor_budget >= 0 ? p->factor_budget : cholesky_budget(p->total_mem);
  out->cg_iterations = p->cg_iterations; out->cg_max_iterations = p->cg_max; out->cg_capped_steps = p->cg_capped; out->cg_solves = p->cg_steps;
  return RCVD_OK;
}
// Bench hook: mean device time (CUDA events, after one warm-up) of one CG matrix product (S H S + D2) p -- k_cg_spmv + k_cg_gather --
// with the S, D2 and direction of the handle's last CG solve.
RCVD_API int32_t rcvd_debug_time_cg_product(rcvd_problem* p, int32_t reps, double* ms) {
  if (!p || !ms || reps <= 0) return set_err(RCVD_ERR_INVALID, "bad argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  if (!p->use_cg) return set_err(RCVD_ERR_INVALID, "this handle solves with the block Cholesky");
  if ((rc = enqueue_cg_product(p, p->d_cg_p, p->d_cg_q, nullptr))) return rc;
  CK(cudaEventRecord(p->ev[0], p->stream));
  for (int i = 0; i < reps; ++i) if ((rc = enqueue_cg_product(p, p->d_cg_p, p->d_cg_q, nullptr))) return rc;
  CK(cudaEventRecord(p->ev[1], p->stream));
  CK(cudaStreamSynchronize(p->stream));
  *ms = ev_ms(p->ev[0], p->ev[1]) / reps;
  return RCVD_OK;
}
// Test hook: the storage budget of the block Cholesky (bytes; -1: the default, cholesky_budget of the device's memory).  The solver
// is chosen again when the structure is next built.
RCVD_API int32_t rcvd_debug_set_factor_budget(rcvd_problem* p, int64_t bytes) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  if (bytes < -1) return set_err(RCVD_ERR_INVALID, "factor budget must be >= 0, or -1 for the default (got %lld)", (long long)bytes);
  if (int rc = drop_structure(p)) return rc;
  p->factor_budget = bytes; return RCVD_OK;
}
// Test hook: the CG's q_tolerance eta (default kCgEta = 0.1, Ceres' Solver::Options::eta).
RCVD_API int32_t rcvd_debug_set_cg_tolerance(rcvd_problem* p, double eta) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null problem");
  if (!(eta > 0.0 && eta < 1.0)) return set_err(RCVD_ERR_INVALID, "CG tolerance must be in (0, 1) (got %g)", eta);
  p->cg_eta = eta; return RCVD_OK;
}
// Test hook: both linear solvers' device storage for the plan of a frame graph, and the one a device of device_total_bytes selects --
// host only, no handle, no device.
RCVD_API int32_t rcvd_debug_linear_storage(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                                           int32_t order_slack, uint64_t device_total_bytes, int64_t* cholesky_bytes, int64_t* cg_bytes, int32_t* solver) {
  if (!cholesky_bytes || !cg_bytes || !solver) return set_err(RCVD_ERR_INVALID, "null argument");
  FactorPlan pl;
  if (int32_t rc = debug_plan(pl, cfg, np, pairs, nt, trip_centers, order_slack, 1, 0, 132)) return rc;
  Layout L; make_layout(*cfg, L);
  const LinearStorage ls = linear_storage(pl, cfg->num_frames, L.npad);
  *cholesky_bytes = ls.cholesky; *cg_bytes = ls.cg;
  *solver = ls.cholesky > cholesky_budget(device_total_bytes) ? RCVD_LINEAR_CG : RCVD_LINEAR_CHOLESKY;
  return RCVD_OK;
}
// Structure statistics (for DESIGN.md / bench): frames, off-diagonal factor blocks, levels, H blocks, npad.
RCVD_API int32_t rcvd_structure_info(rcvd_problem* p, int32_t out[8]) {
  if (!p) return set_err(RCVD_ERR_INVALID, "null argument");
  SET_DEVICE(p->device);
  int rc = ensure_ready(p); if (rc) return rc;
  out[0] = p->N; out[1] = p->plan.nLoff; out[2] = (int)p->plan.levels.size(); out[3] = (int)p->plan.hblocks.size(); out[4] = p->L.npad; out[5] = p->L.nf; out[6] = p->pairs.num_tiles;
  out[7] = p->plan.upd_targets;
  return RCVD_OK;
}
