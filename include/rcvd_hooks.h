/* rcvd_hooks.h -- test / bench hooks exported by librcvd_b200.so.  NOT part of the drop-in boundary (include/rcvd.h):
 * nothing in the reference corresponds to these; tests/, bench.py and tools/ use them to look inside the solver. */
#ifndef RCVD_HOOKS_H_
#define RCVD_HOOKS_H_
#include "rcvd.h"
#ifdef __cplusplus
extern "C" {
#endif

/* kernels launched so far by this handle -- every one: the structure set-up, the evaluations, the LM step, the hooks' kernels and each
 * kernel of a factor+solve graph replay -- / by the filter / by the constraint builder (the "did the CUDA path run" evidence) */
int64_t rcvd_launch_count(rcvd_problem* p);
int64_t rcvd_filter_launch_count(void);
int64_t rcvd_builder_launch_count(void);
int64_t rcvd_static_flag_launch_count(void);
int64_t rcvd_tracks_launch_count(void);
int64_t rcvd_flow_mask_launch_count(void);
int64_t rcvd_flow_vis_launch_count(void);
int64_t rcvd_resize_launch_count(void);
/* rcvd_resize_area's kernels alone: the frames are uploaded once, the kernels of every output run reps times between two CUDA events,
 * and *ms is the mean device time of one pass over all the frames and outputs.  Arguments and refusals as rcvd_resize_area (the output
 * buffers are not needed); num_frames >= 1, reps >= 1. */
int32_t rcvd_debug_time_resize_area(const rcvd_resize_params* prm, int32_t device, const uint8_t* frames, int32_t reps, double* ms);
int64_t rcvd_depth_vis_launch_count(void);
/* rcvd_depth_visualize's kernels alone: the frames are uploaded once, then each pass runs reps times between two CUDA events; *ms_range
 * and *ms_color are the mean device times of one pass over all the frames (the colour pass writes rgb).  Arguments and refusals as
 * rcvd_depth_visualize with both passes; num_frames >= 1, reps >= 1. */
int32_t rcvd_debug_time_depth_visualize(const rcvd_depth_vis_params* prm, int32_t device, const void* frames, const uint8_t* colormap,
                                        int32_t reps, double* ms_range, double* ms_color);
/* rcvd_flow_masks' kernel alone: the inputs are uploaded once, the kernel (with counts) runs reps times between two CUDA events, and
 * *ms is the mean device time of one launch over all the pairs.  Arguments and refusals as rcvd_flow_masks; reps >= 1. */
int32_t rcvd_debug_time_flow_masks(const rcvd_flow_mask_params* prm, int32_t device, const int32_t* pair_frames, const float* flow_ij,
                                   const float* flow_ji, const float* colors, int32_t reps, double* ms);
int64_t rcvd_flow_register_launch_count(void);
/* rcvd_homography_warp's / rcvd_flow_unregister's kernel alone: the inputs are uploaded once, the kernel runs reps times between two
 * CUDA events, and *ms is the mean device time of one pass over all the pairs.  Arguments and refusals as the entry point (the output
 * buffer is not needed); num_pairs >= 1, reps >= 1. */
int32_t rcvd_debug_time_homography_warp(const rcvd_homography_warp_params* prm, int32_t device, const uint8_t* frames, const int32_t* pair_frames,
                                        const double* inverse, int32_t reps, double* ms);
int32_t rcvd_debug_time_flow_unregister(const rcvd_flow_unregister_params* prm, int32_t device, const float* flow, const double* h_inv,
                                        int32_t reps, double* ms);
int64_t rcvd_dynamic_mask_launch_count(void);
/* rcvd_dynamic_masks' kernels alone: the inputs are uploaded once, the kernels (with the anonymised frames when frames is non-null)
 * run reps times between two CUDA events, and *ms is the mean device time of one pass over all the frames.  Arguments and refusals as
 * rcvd_dynamic_masks (the outputs are not needed); num_frames >= 1, reps >= 1. */
int32_t rcvd_debug_time_dynamic_masks(const rcvd_dynamic_mask_params* prm, int32_t device, const int64_t* instance_offsets,
                                      const uint8_t* instances, const uint8_t* frames, int32_t reps, double* ms);
int64_t rcvd_builder_last_rounds(void);          /* selection rounds of the last rcvd_build_constraints call */

/* {frames, off-diagonal factor blocks, levels, H blocks, npad, stride, tiles, update targets ((source level, target block) pairs)} */
int32_t rcvd_structure_info(rcvd_problem* p, int32_t out[8]);

/* the block-Cholesky plan (robust_cvd_b200/csrc/rcvd_plan.h) of the frame graph of np pairs and nt triplet centres under cfg (shared
 * intrinsics, position regulariser, stride), as rank `rank` of `nranks` with the distributed factorisation enabled, on a device of
 * num_sms SMs.  Host only: no handle, no device.  Per frame, in the caller's frame ids: order[N] = elimination order, level[N] = level,
 * owner[N] = owning rank, perm[N] = caller's frame of each internal frame id.  out = {levels, off-diagonal factor blocks, H blocks,
 * update targets ((source level, target block) pairs), k_update_tma items, k_substitution tasks, distributed, first replicated level,
 * first k_substitution level, this rank's L blocks, H blocks, frames, update passes}.  An out-of-range pair or triplet centre:
 * RCVD_ERR_INVALID. */
int32_t rcvd_debug_factor_plan(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                               int32_t order_slack, int32_t nranks, int32_t rank, int32_t num_sms,
                               int32_t* order, int32_t* level, int32_t* owner, int32_t* perm, int32_t out[13]);
/* the update passes of the same plan, in launch order, caller's frame ids: passes[P][5] = {target row frame, target column frame (equal
 * on a diagonal block), apply level, stream (0: late pass, main stream; 1 / 2: deferred pass in the first / second side-stream launch of
 * its level), source count}; sources = the source frame of every product, pass after pass; join[2 * levels] = per level and side
 * launch, the level whose late passes wait for it (levels: none); flags[P] = per pass, bit 0: symmetric (diagonal) target, bit 1: the
 * first pass into a fill block, which writes the target without reading it.  counts = {passes P, products, 2 * levels, tail boundary
 * level, source levels per deferred window below the tail} on return; with passes non-null, counts[0..2] are the capacities of passes
 * and flags (in passes), sources and join on entry. */
int32_t rcvd_debug_update_passes(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                                 int32_t order_slack, int32_t nranks, int32_t rank, int32_t num_sms,
                                 int32_t* passes, int32_t* sources, int32_t* join, int32_t* flags, int32_t counts[5]);
/* the k_update_tma work items of the same plan, in the order `order` (1: locality order, the default of a handle; 0: sorted by cost
 * within each launch): items[I][8] = {target L block, first source pair, source pairs, tile row origin, tile column origin, rows,
 * columns, flags (1: diagonal tile of a symmetric target, 2: first pass into a fill block)}; launches[levels][6] = per level
 * {offset, items} of its late launch and of its two deferred launches; products[Q][2] = per source pair the T indices of X_rk and
 * X_ck.  counts = {I, 3 * levels, Q, unknowns per block the tiles cover (neff), npad} on return; with items non-null, counts[0..2]
 * are the capacities of items, launches (in pairs of ints) and products (in pairs of ints) on entry. */
int32_t rcvd_debug_update_items(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                                int32_t order_slack, int32_t nranks, int32_t rank, int32_t num_sms, int32_t order,
                                int32_t* items, int32_t* launches, int32_t* products, int32_t counts[5]);

/* y = (S H S + diag(D2))^-1 b with the current H (exercises factorisation + substitution alone) */
int32_t rcvd_debug_linear_solve(rcvd_problem* p, const double* S, const double* D2, const double* b, double* y);

/* y = (H + diag(D2))^-1 b for a dense symmetric U x U matrix H (U = N * stride, caller's frame order) through the production
 * factorisation graph, S = 1: H is scattered into the H blocks of the frame graph set by rcvd_problem_set_structure /
 * rcvd_problem_set_constraints (no evaluation).  A non-zero entry in a frame pair the graph does not couple: RCVD_ERR_INVALID;
 * a non-positive pivot: RCVD_ERR_NUMERIC. */
int32_t rcvd_debug_solve_matrix(rcvd_problem* p, const double* H, const double* D2, const double* b, double* y);
/* rcvd_debug_solve_matrix through conjugate gradients, on a handle whose structure chose them (a factor budget of 0); iterations = the
 * CG iterations run.  A handle on the Cholesky path: RCVD_ERR_INVALID; a CG breakdown or non-positive pivot: RCVD_ERR_NUMERIC. */
int32_t rcvd_debug_cg_solve_matrix(rcvd_problem* p, const double* H, const double* D2, const double* b, double* y, int32_t* iterations);
/* rcvd_covariance for a dense symmetric U x U matrix H (caller's frame order), scattered into the H blocks of the handle's frame graph
 * as rcvd_debug_solve_matrix does (no evaluation), min_pivot 1e-10.  Only the parameters in hold (nullable) are zeroed: no active
 * mask, configuration constants or frame range apply.  Refusals and the rank test as in rcvd_covariance. */
int32_t rcvd_debug_covariance_matrix(rcvd_problem* p, const double* H, const uint8_t* hold, int32_t num_blocks, const int32_t* frame_pairs,
                                     double* out);
/* launches of the covariance kernels since the handle was created: {k_selinv_product, k_selinv_trmm, k_selinv_pivots, k_selinv_gather,
 * k_selinv_scale} */
int32_t rcvd_debug_covariance_launches(rcvd_problem* p, int64_t out[5]);
/* the last rcvd_covariance call: out = {device ms of the factorisation with its rank test, of the selected inversion, of the gather and
 * copy-out; algorithmic flops of the selected inversion (2 nf^3 per block product, nf^3 per triangular multiply); its block products} */
int32_t rcvd_debug_covariance_profile(rcvd_problem* p, double out[5]);
/* The storage of both linear solvers (rcvd_linear_info) for the frame graph of np pairs and nt triplet centres under cfg, on one GPU, and
 * the solver (RCVD_LINEAR_*) a device of device_total_bytes selects.  Host only: no handle, no device. */
int32_t rcvd_debug_linear_storage(const rcvd_config* cfg, int32_t np, const int32_t* pairs, int32_t nt, const int32_t* trip_centers,
                                  int32_t order_slack, uint64_t device_total_bytes, int64_t* cholesky_bytes, int64_t* cg_bytes, int32_t* solver);
/* mean device ms of one CG matrix product (S H S + D2) p (the SpMV over the stored H blocks and the per-frame sum) over reps, with the
 * S, D2 and direction of the handle's last CG solve: the number tools/bench_long.py turns into achieved bandwidth */
int32_t rcvd_debug_time_cg_product(rcvd_problem* p, int32_t reps, double* ms);
/* what the last factorisation left on the device: order[N] = caller's frame index of each eliminated frame, in elimination order;
 * L = dense U x U lower-triangular factor of P A P^T in that order (padding stripped, strict upper triangle zero); Linv (may be null)
 * = the N * stride * stride explicit inverses of the diagonal blocks (k_trinv), same order.  RCVD_ERR_INVALID before any factorisation. */
int32_t rcvd_debug_factor_dense(rcvd_problem* p, int32_t* order, double* L, double* Linv);
/* launches of each factorisation / solve kernel path since the handle was created: {k_potrf_smem, k_potrf_panel, k_trsm_ll<4>,
 * k_trsm_ll<2>, TRSM by explicit inverse (k_gemm_nt), k_update_tma<1>, k_update_tma<2>, level-launched substitution
 * (k_fwd_* / k_bwd_*), k_substitution, k_trinv, the rest (k_load_factor, k_potrf_trail), k_update_tma<1> launches with fewer CTAs
 * than items (CTAs that walk several items), k_trsm_ll launches (either shape) streamed beside their level's k_potrf_smem} */
int32_t rcvd_debug_linear_paths(rcvd_problem* p, int64_t out[13]);
/* launches of each pair kernel that assembles the normal matrix (cost + gradient + H) since the handle was created: {k_pairs,
 * k_accumulate_runs, k_accumulate_fast}.  rcvd_debug_set_fast_path and the configuration choose among them. */
int32_t rcvd_debug_pair_kernel_launches(rcvd_problem* p, int64_t out[3]);

/* one damped LM step at the current state with trust-region `radius`; out = {|(S H S + D2) y - S g| / |S g| (device SpMV over the
 * assembled H), |S g|, cost, |g|_2, |y|_2, non-positive-pivot flag}: the parity evidence bench.py prints at the size it times */
int32_t rcvd_debug_linear_residual(rcvd_problem* p, double radius, double out[6]);

/* what the last rcvd_time_iteration step computed, in the caller's frame order: g = gradient at the state, xc = candidate state
 * of the damped LM step (N*stride doubles each); out = {cost, candidate cost}.  Read it before any other call on the handle. */
int32_t rcvd_debug_last_iteration(rcvd_problem* p, double* g, double* xc, double out[2]);

/* per-kernel-class device time of one factorisation + solve: out_ms[0..5] = load, potrf, trinv, trsm, update GEMM,
 * substitution; [6] = update-GEMM launches, [7] = their algorithmic flops.  reps > 0: serialised on one stream;
 * reps < 0: two-stream overlap kept, main-stream view. */
int32_t rcvd_debug_profile_linear(rcvd_problem* p, int32_t reps, double out_ms[8]);
/* per-level view of the last rcvd_debug_profile_linear call: out[level][6] ms of {load, potrf, trinv, trsm, update, substitution} */
int32_t rcvd_debug_level_profile(rcvd_problem* p, double* out, int32_t max_levels);
/* fp64 tensor-core (DMMA) peak of the device in TFLOP/s for one mma.sync shape (0 m8n8k4, 1 m16n8k4, 2 m16n8k8, 3 m16n8k16),
 * measured live */
int32_t rcvd_debug_fp64_tensor_peak(int32_t device, int32_t shape, double* tflops);

/* A/B switches (defaults in parentheses).  A null handle: RCVD_ERR_INVALID.  set_order_slack, set_eval_only and set_distributed
 * rebuild the structure at the next call that needs it; like every setter of rcvd.h they keep the state (rcvd_problem_get_state). */
int32_t rcvd_debug_set_fast_path(rcvd_problem* p, int32_t on);        /* (1) specialised accumulate kernels; 0 = generic kernel; 2 = k_accumulate_fast
                                                                          even where the run path applies (bilinear grids) */
int32_t rcvd_debug_set_overlap(rcvd_problem* p, int32_t on);          /* (1) two-stream factorisation graph */
int32_t rcvd_debug_set_order_slack(rcvd_problem* p, int32_t slack);   /* (4) multiple-elimination degree slack; -1 greedy */
int32_t rcvd_debug_set_eval_only(rcvd_problem* p, int32_t on);        /* (0) cost / gradient evaluations only: no matrix storage (the whole-problem check of a multi-GPU bench) */
int32_t rcvd_debug_set_distributed(rcvd_problem* p, int32_t on);      /* (1) nranks > 1: distributed factorisation; 0 = all-reduce H + replicated factorisation */
int32_t rcvd_distribution_info(rcvd_problem* p, int32_t out[4]);       /* {distributed, first replicated level, levels, frames owned by this rank} */
int32_t rcvd_debug_set_update_kernel(rcvd_problem* p, int32_t tma, int32_t side_items_per_cta); /* (1, 0) tma must be 1 (0: RCVD_ERR_INVALID, the cp.async update path was removed); items-per-CTA cap of the one-team launches (0: none) */
int32_t rcvd_debug_set_update_order(rcvd_problem* p, int32_t order);  /* (1) k_update_tma items of a launch in locality order; 0 = sorted by cost (same items, same factor) */
int32_t rcvd_debug_set_factor_budget(rcvd_problem* p, int64_t bytes); /* (-1) storage budget of the block Cholesky: -1 = 4/5 of the device's total memory;
                                                                          0 = conjugate gradients on any single-GPU problem */
int32_t rcvd_debug_set_cg_tolerance(rcvd_problem* p, double eta);     /* (0.1) the CG's quadratic-model tolerance eta, in (0, 1) */

#ifdef __cplusplus
}
#endif
#endif /* RCVD_HOOKS_H_ */
