"""Python binding (ctypes) of the C ABI in include/rcvd.h -- the H100 solver.

`Problem` is the array-level equivalent of the reference's
DepthVideoPoseOptimizer::poseOptimizationStep / normalizeDepth
(lib/PoseOptimizer.cpp:890-990, :992-1147): one non-linear least-squares
problem over per-frame [pose(6), focal, depth-transform params, spatial params].

There is no CPU fallback: if librcvd_b200.so is missing or no CUDA device is
usable, construction raises RuntimeError.
"""
import ctypes as C
import os
import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "librcvd_b200.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(the CUDA extension is mandatory, there is no CPU fallback)")
        L = C.CDLL(path)
        L.rcvd_last_error.restype = C.c_char_p
        L.rcvd_launch_count.restype = C.c_int64
        L.rcvd_problem_create.argtypes = [C.POINTER(abi.Config), C.c_int32, C.POINTER(C.c_void_p)]
        L.rcvd_problem_destroy.argtypes = [C.c_void_p]
        for name in ("rcvd_frame_stride", "rcvd_depth_param_offset", "rcvd_spatial_param_offset"):
            getattr(L, name).argtypes = [C.POINTER(abi.Config)]
        _LIB = L
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def _check(rc):
    if rc != 0:
        raise RuntimeError(f"rcvd error {rc}: {lib().rcvd_last_error().decode()}")


def frame_stride(cfg):
    return lib().rcvd_frame_stride(C.byref(cfg))


def depth_param_offset(cfg):
    return lib().rcvd_depth_param_offset(C.byref(cfg))


def spatial_param_offset(cfg):
    return lib().rcvd_spatial_param_offset(C.byref(cfg))


FACTOR_PLAN_COUNTS = ("levels", "offdiag_factor_blocks", "h_blocks", "update_targets", "update_items", "substitution_tasks",
                      "distributed", "first_replicated_level", "first_substitution_level", "rank_l_blocks", "rank_h_blocks", "rank_frames",
                      "update_passes")


def factor_plan(cfg, pairs, trip_centers=(), order_slack=4, nranks=1, rank=0, num_sms=132):
    """Test hook: the block-Cholesky plan of the frame graph of `pairs` ([P, 2] frame pairs) and `trip_centers` under cfg, computed on
    the host (no device).  Returns the per-frame arrays order, level, owner, perm (caller's frame ids; perm[i] = caller's frame of
    internal frame i) and the FACTOR_PLAN_COUNTS."""
    n = cfg.num_frames
    pf = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
    tc = np.ascontiguousarray(np.asarray(trip_centers, np.int32).reshape(-1))
    arrays = {k: np.zeros(n, np.int32) for k in ("order", "level", "owner", "perm")}
    out = (C.c_int32 * len(FACTOR_PLAN_COUNTS))()
    _check(lib().rcvd_debug_factor_plan(C.byref(cfg), C.c_int32(pf.shape[0]), _p(pf, C.c_int32), C.c_int32(tc.size), _p(tc, C.c_int32),
                                        C.c_int32(order_slack), C.c_int32(nranks), C.c_int32(rank), C.c_int32(num_sms),
                                        *(_p(a, C.c_int32) for a in arrays.values()), out))
    return {**arrays, **dict(zip(FACTOR_PLAN_COUNTS, list(out)))}


def update_passes(cfg, pairs, trip_centers=(), order_slack=4, nranks=1, rank=0, num_sms=132):
    """Test hook: the update passes of factor_plan's plan, in launch order (host only).  Returns passes [P, 5] (target row frame, target
    column frame, apply level, stream: 0 late / main, 1 or 2 deferred / the level's first or second side launch, source count), sources
    (the source frame of every product, pass after pass), join ([levels, 2]: per side launch, the level whose late passes wait for it),
    flags ([P]: bit 0 symmetric target, bit 1 the first pass into a fill block, which writes its target without reading it), tail (the
    tail boundary level) and window (source levels per window of the deferred passes)."""
    pf = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
    tc = np.ascontiguousarray(np.asarray(trip_centers, np.int32).reshape(-1))
    args = (C.byref(cfg), C.c_int32(pf.shape[0]), _p(pf, C.c_int32), C.c_int32(tc.size), _p(tc, C.c_int32),
            C.c_int32(order_slack), C.c_int32(nranks), C.c_int32(rank), C.c_int32(num_sms))
    counts = (C.c_int32 * 5)()
    _check(lib().rcvd_debug_update_passes(*args, None, None, None, None, counts))
    passes, sources, join = np.zeros((counts[0], 5), np.int32), np.zeros(counts[1], np.int32), np.zeros(counts[2], np.int32)
    flags = np.zeros(counts[0], np.int32)
    _check(lib().rcvd_debug_update_passes(*args, _p(passes, C.c_int32), _p(sources, C.c_int32), _p(join, C.c_int32), _p(flags, C.c_int32), counts))
    return {"passes": passes, "sources": sources, "join": join.reshape(-1, 2), "flags": flags, "tail": counts[3], "window": counts[4]}


UPDATE_ITEM_FIELDS = ("dst", "first", "count", "m0", "n0", "mrows", "ncols", "flags")


def update_items(cfg, pairs, trip_centers=(), order_slack=4, nranks=1, rank=0, num_sms=132, order=1):
    """Test hook: the update kernel's work items of factor_plan's plan (host only), in the order `order` (1 locality, 0 cost-sorted).
    Returns items [I, 8] (UPDATE_ITEM_FIELDS), launches [levels, 3, 2] ((offset, items) of the late launch and the two deferred
    launches of every level), products [Q, 2] (T indices of X_rk and X_ck of every source pair), neff and npad."""
    pf = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
    tc = np.ascontiguousarray(np.asarray(trip_centers, np.int32).reshape(-1))
    args = (C.byref(cfg), C.c_int32(pf.shape[0]), _p(pf, C.c_int32), C.c_int32(tc.size), _p(tc, C.c_int32),
            C.c_int32(order_slack), C.c_int32(nranks), C.c_int32(rank), C.c_int32(num_sms), C.c_int32(order))
    counts = (C.c_int32 * 5)()
    _check(lib().rcvd_debug_update_items(*args, None, None, None, counts))
    items, launches, products = np.zeros((counts[0], 8), np.int32), np.zeros((counts[1], 2), np.int32), np.zeros((counts[2], 2), np.int32)
    _check(lib().rcvd_debug_update_items(*args, _p(items, C.c_int32), _p(launches, C.c_int32), _p(products, C.c_int32), counts))
    return {"items": items, "launches": launches.reshape(-1, 3, 2), "products": products, "neff": counts[3], "npad": counts[4]}


def linear_storage(cfg, pairs, trip_centers=(), order_slack=4, device_total_bytes=0):
    """Test hook: the device storage of both linear solvers for the frame graph of `pairs` and `trip_centers` under cfg on one GPU, and
    the solver a device of device_total_bytes selects (host only, no device).  Returns {"cholesky_bytes", "cg_bytes", "solver"}
    (abi.LINEAR_*)."""
    pf = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
    tc = np.ascontiguousarray(np.asarray(trip_centers, np.int32).reshape(-1))
    chol, cg, which = C.c_int64(), C.c_int64(), C.c_int32()
    _check(lib().rcvd_debug_linear_storage(C.byref(cfg), C.c_int32(pf.shape[0]), _p(pf, C.c_int32), C.c_int32(tc.size), _p(tc, C.c_int32),
                                           C.c_int32(order_slack), C.c_uint64(device_total_bytes), C.byref(chol), C.byref(cg), C.byref(which)))
    return {"cholesky_bytes": chol.value, "cg_bytes": cg.value, "solver": which.value}


class Problem:
    def __init__(self, cfg, device=0):
        self.cfg = cfg
        self.L = lib()
        self.h = C.c_void_p()
        _check(self.L.rcvd_problem_create(C.byref(cfg), C.c_int32(device), C.byref(self.h)))
        self.N = cfg.num_frames
        self.stride = frame_stride(cfg)
        self.U = self.N * self.stride
        self.num_constraints = 0

    def close(self):
        if getattr(self, "h", None):
            self.L.rcvd_problem_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_frames(self, in_range=None, median_depth=None, adaptive_weights=None):
        ir = None if in_range is None else np.ascontiguousarray(in_range, np.uint8)
        md = None if median_depth is None else np.ascontiguousarray(median_depth, np.float64)
        aw = None if adaptive_weights is None else np.ascontiguousarray(adaptive_weights, np.float64)
        _check(self.L.rcvd_problem_set_frames(self.h, _p(ir, C.c_uint8), _p(md, C.c_double), _p(aw, C.c_double)))

    def _set_records(self, setter, frames, frames_per_group, offsets, records, width):
        """One constraint family through its C setter: frames[G, frames_per_group], offsets[G+1], records[n][width].  Returns n."""
        fr = np.ascontiguousarray(frames, np.int32).reshape(-1, frames_per_group)
        off = np.ascontiguousarray(offsets, np.int64)
        rec = np.ascontiguousarray(records, np.float32).reshape(-1, width)
        assert off.shape[0] == fr.shape[0] + 1 and off[-1] == rec.shape[0]
        _check(setter(self.h, C.c_int32(fr.shape[0]), _p(fr, C.c_int32), _p(off, C.c_int64), _p(rec, C.c_float)))
        return int(rec.shape[0])

    def set_constraints(self, pair_frames, offsets, records):
        self.num_constraints = self._set_records(self.L.rcvd_problem_set_constraints, pair_frames, 2, offsets, records, 6)

    def set_triplets(self, centers, offsets, records):
        """Scene-flow smoothness constraints (addSceneFlowSmoothnessLoss): centers[T], offsets[T+1], records[n][10]."""
        self._set_records(self.L.rcvd_problem_set_triplets, centers, 1, offsets, records, 10)

    def set_depth_pairs(self, pair_frames, offsets, records):
        """Pairwise depth-normalisation constraints (DisparityDissimilarityCost): pair_frames[P, 2], offsets[P+1], records[C][6] in the
        layout of set_constraints.  Single-GPU only."""
        self._set_records(self.L.rcvd_problem_set_depth_pairs, pair_frames, 2, offsets, records, 6)

    def set_structure(self, pair_frames):
        pf = np.ascontiguousarray(pair_frames, np.int32).reshape(-1, 2)
        _check(self.L.rcvd_problem_set_structure(self.h, C.c_int32(pf.shape[0]), _p(pf, C.c_int32)))

    def init_comm(self, nranks, rank, unique_id):
        uid = np.ascontiguousarray(unique_id, np.uint8)
        assert uid.size == 128
        _check(self.L.rcvd_problem_init_comm(self.h, C.c_int32(nranks), C.c_int32(rank), _p(uid, C.c_uint8)))

    def set_state(self, x):
        x = np.ascontiguousarray(x, np.float64).reshape(-1)
        assert x.size == self.U
        _check(self.L.rcvd_problem_set_state(self.h, _p(x, C.c_double)))

    def get_state(self):
        x = np.empty(self.U, np.float64)
        _check(self.L.rcvd_problem_get_state(self.h, _p(x, C.c_double)))
        return x.reshape(self.N, self.stride)

    def evaluate(self, gradient=False):
        cost = C.c_double()
        g = np.zeros(self.U, np.float64) if gradient else None
        _check(self.L.rcvd_evaluate(self.h, C.byref(cost), _p(g, C.c_double)))
        return (cost.value, g) if gradient else cost.value

    def normal_matrix_dense(self):
        H = np.zeros((self.U, self.U), np.float64)
        _check(self.L.rcvd_normal_matrix_dense(self.h, _p(H, C.c_double)))
        return H

    def row_layout(self):
        """Per residual family (abi.ROW_FAMILIES): {"blocks", "residuals" (m, per block), "max_cols" (k, column slots per residual)}."""
        out = abi.RowLayout()
        _check(self.L.rcvd_row_layout(self.h, C.byref(out)))
        return {name: {"blocks": f.blocks, "residuals": f.residuals, "max_cols": f.max_cols} for name, f in zip(abi.ROW_FAMILIES, out.family)}

    def rows(self, family, jacobian=False):
        """rcvd_evaluate_rows at the current state.  family: a name of abi.ROW_FAMILIES or an abi.ROWS_* value.  Returns (r [n, m],
        rho [n]) and with jacobian=True also (cols [n, m, k] int32, J [n, m, k]): one block per constraint record in the order it was
        set, or per regulariser row (include/rcvd.h gives the orders).  cols are indices into the [N * stride] state, -1 in unused slots."""
        fam = abi.ROW_FAMILIES.index(family) if isinstance(family, str) else int(family)
        if not 0 <= fam < len(abi.ROW_FAMILIES):
            raise ValueError(f"unknown row family {family!r}")
        lay = self.row_layout()[abi.ROW_FAMILIES[fam]]
        n, m, k = lay["blocks"], lay["residuals"], lay["max_cols"]
        r = np.zeros((n, m), np.float64); rho = np.zeros(n, np.float64)
        cols = np.zeros((n, m, k), np.int32) if jacobian else None
        J = np.zeros((n, m, k), np.float64) if jacobian else None
        _check(self.L.rcvd_evaluate_rows(self.h, C.c_int32(fam), _p(r, C.c_double), _p(rho, C.c_double), _p(cols, C.c_int32), _p(J, C.c_double)))
        return (r, rho, cols, J) if jacobian else (r, rho)

    def debug_linear_solve(self, S, D2, b):
        S = np.ascontiguousarray(S, np.float64); D2 = np.ascontiguousarray(D2, np.float64)
        b = np.ascontiguousarray(b, np.float64); y = np.zeros_like(b)
        _check(self.L.rcvd_debug_linear_solve(self.h, _p(S, C.c_double), _p(D2, C.c_double), _p(b, C.c_double), _p(y, C.c_double)))
        return y

    def solve_matrix(self, H, D2, b):
        """Test hook: y = (H + diag(D2))^-1 b through the production factorisation graph (S = 1) for a dense symmetric H [U, U] in the
        caller's frame order, restricted to the frame graph set by set_structure / set_constraints."""
        H = np.ascontiguousarray(H, np.float64); D2 = np.ascontiguousarray(D2, np.float64); b = np.ascontiguousarray(b, np.float64)
        assert H.shape == (self.U, self.U) and D2.size == self.U and b.size == self.U
        y = np.zeros(self.U, np.float64)
        _check(self.L.rcvd_debug_solve_matrix(self.h, _p(H, C.c_double), _p(D2, C.c_double), _p(b, C.c_double), _p(y, C.c_double)))
        return y

    def cg_solve_matrix(self, H, D2, b):
        """Test hook: solve_matrix through conjugate gradients, on a handle whose structure chose them (set_factor_budget(0)).
        Returns (y, CG iterations)."""
        H = np.ascontiguousarray(H, np.float64); D2 = np.ascontiguousarray(D2, np.float64); b = np.ascontiguousarray(b, np.float64)
        assert H.shape == (self.U, self.U) and D2.size == self.U and b.size == self.U
        y = np.zeros(self.U, np.float64); it = C.c_int32()
        _check(self.L.rcvd_debug_cg_solve_matrix(self.h, _p(H, C.c_double), _p(D2, C.c_double), _p(b, C.c_double), _p(y, C.c_double), C.byref(it)))
        return y, it.value

    def linear_info(self):
        """The linear solver the handle chose and its storage, and the CG iterations of the last solve (rcvd_linear_info; builds the
        structure if needed).  Returns a dict of abi.LinearInfo's fields."""
        out = abi.LinearInfo()
        _check(self.L.rcvd_problem_linear_info(self.h, C.byref(out)))
        return {name: getattr(out, name) for name, _ in abi.LinearInfo._fields_}

    def time_cg_product(self, reps=20):
        """Bench hook: mean device ms of one CG matrix product (S H S + D2) p, with the last CG solve's S, D2 and direction."""
        ms = C.c_double()
        _check(self.L.rcvd_debug_time_cg_product(self.h, C.c_int32(reps), C.byref(ms)))
        return ms.value

    def set_factor_budget(self, nbytes=-1):
        """Test hook: the block Cholesky's storage budget in bytes (-1: the default, 4/5 of the device's memory; 0: conjugate gradients
        on any single-GPU problem).  Takes effect when the structure is next built."""
        _check(self.L.rcvd_debug_set_factor_budget(self.h, C.c_int64(nbytes)))

    def set_cg_tolerance(self, eta=0.1):
        """Test hook: the CG's quadratic-model tolerance eta (default 0.1)."""
        _check(self.L.rcvd_debug_set_cg_tolerance(self.h, C.c_double(eta)))

    def factor_dense(self, inverses=False):
        """Test hook: (order, L, Linv) of the last factorisation -- caller's frame index of each eliminated frame, the dense lower factor
        of P A P^T in that order, and (inverses=True) the explicit inverses of its diagonal blocks [N, stride, stride], else None."""
        order = np.zeros(self.N, np.int32); Lf = np.zeros((self.U, self.U), np.float64)
        Li = np.zeros((self.N, self.stride, self.stride), np.float64) if inverses else None
        _check(self.L.rcvd_debug_factor_dense(self.h, _p(order, C.c_int32), _p(Lf, C.c_double), _p(Li, C.c_double)))
        return order, Lf, Li

    LINEAR_PATHS = ("potrf_smem", "potrf_panel", "trsm_ll4", "trsm_ll2", "trsm_gemm", "update_tma1", "update_tma2", "substitution_levels", "substitution_fused", "trinv", "other", "update_tma1_multi_item", "trsm_ll_streamed")

    def linear_paths(self):
        """Test hook: launches of each factorisation / solve kernel path since the handle was created (LINEAR_PATHS)."""
        out = (C.c_int64 * len(self.LINEAR_PATHS))()
        _check(self.L.rcvd_debug_linear_paths(self.h, out))
        return dict(zip(self.LINEAR_PATHS, list(out)))

    def solve(self, options=None):
        opt = options or abi.default_solve_options()
        s = abi.SolveSummary()
        _check(self.L.rcvd_solve(self.h, C.byref(opt), C.byref(s)))
        return s

    def time_accumulate(self, iters=10):
        ms = C.c_double()
        _check(self.L.rcvd_time_accumulate(self.h, C.c_int32(iters), C.byref(ms)))
        return ms.value

    def time_iteration(self, iters=5, radius=1e4):
        a, b, c, d = C.c_double(), C.c_double(), C.c_double(), C.c_double()
        _check(self.L.rcvd_time_iteration(self.h, C.c_int32(iters), C.c_double(radius), C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return {"iter_ms": a.value, "accumulate_ms": b.value, "linear_ms": c.value, "cost_ms": d.value}

    def last_iteration(self):
        """Bench hook: what the last time_iteration step computed -- gradient, candidate state (both [N, stride]), cost, candidate cost."""
        g, xc, out = np.empty(self.U, np.float64), np.empty(self.U, np.float64), (C.c_double * 2)()
        _check(self.L.rcvd_debug_last_iteration(self.h, _p(g, C.c_double), _p(xc, C.c_double), out))
        return {"gradient": g.reshape(self.N, self.stride), "candidate_state": xc.reshape(self.N, self.stride), "cost": out[0], "candidate_cost": out[1]}

    def structure_info(self):
        out = (C.c_int32 * 8)()
        _check(self.L.rcvd_structure_info(self.h, out))
        keys = ["frames", "offdiag_factor_blocks", "levels", "h_blocks", "npad", "stride", "tiles", "update_tasks"]
        return dict(zip(keys, list(out)))

    def linear_residual(self, radius=1e4):
        """Bench / test hook: one damped LM step at the current state; device-side residual of the linear system and checksums."""
        out = (C.c_double * 6)()
        _check(self.L.rcvd_debug_linear_residual(self.h, C.c_double(radius), out))
        keys = ["rel_residual", "rhs_norm", "cost", "grad_norm", "step_norm", "pivot_fail"]
        return dict(zip(keys, list(out)))

    def profile_linear(self, reps=3):
        """Bench hook: per-kernel-class device time of one factorisation + solve (serialised on one stream, CUDA events per launch)."""
        out = (C.c_double * 8)()
        _check(self.L.rcvd_debug_profile_linear(self.h, C.c_int32(reps), out))
        keys = ["load_ms", "potrf_ms", "trinv_ms", "trsm_ms", "gemm_ms", "solve_ms", "gemm_launches", "gemm_flops"]
        return dict(zip(keys, list(out)))

    def set_fast_path(self, on=True):
        """Test hook: False forces the generic accumulate kernel (the tests' reference); True (default) allows the specialised ones;
        2 selects k_accumulate_fast even on bilinear grids, where the run path would serve."""
        _check(self.L.rcvd_debug_set_fast_path(self.h, C.c_int32(int(on))))

    def set_update_kernel(self, tma=True, side_items_per_cta=0):
        """Test / bench hook: side_items_per_cta > 0 caps the work items per CTA of the one-team update launches.  tma must be True:
        the persistent TMA-fed kernel is the only update kernel (False raises)."""
        _check(self.L.rcvd_debug_set_update_kernel(self.h, C.c_int32(1 if tma else 0), C.c_int32(side_items_per_cta)))

    def set_update_order(self, order=1):
        """Test / bench hook: the order of the update kernel's work items within each launch, 1 (default) locality order, 0 sorted by
        cost.  Both run the same items: the factor is the same bit for bit."""
        _check(self.L.rcvd_debug_set_update_order(self.h, C.c_int32(order)))

    def set_eval_only(self, on=True):
        """Test / bench hook: the handle only evaluates cost / gradient; no matrix storage is allocated."""
        _check(self.L.rcvd_debug_set_eval_only(self.h, C.c_int32(1 if on else 0)))

    def set_distributed(self, on=True):
        """Test / bench hook (nranks > 1): distributed factorisation (default) or the replicated scheme."""
        _check(self.L.rcvd_debug_set_distributed(self.h, C.c_int32(1 if on else 0)))

    def distribution_info(self):
        out = (C.c_int32 * 4)()
        _check(self.L.rcvd_distribution_info(self.h, out))
        return dict(zip(["distributed", "first_replicated_level", "levels", "frames_owned"], list(out)))

    def set_order_slack(self, slack):
        _check(self.L.rcvd_debug_set_order_slack(self.h, C.c_int32(slack)))

    def set_overlap(self, on=True):
        _check(self.L.rcvd_debug_set_overlap(self.h, C.c_int32(1 if on else 0)))

    def launch_count(self):
        return int(self.L.rcvd_launch_count(self.h))


def nccl_unique_id():
    out = np.zeros(128, np.uint8)
    _check(lib().rcvd_nccl_unique_id(_p(out, C.c_uint8)))
    return out


def depth_apply(cfg, depth_params, src, device=0):
    """DepthXform::apply (reference lib/DepthMapTransform.cpp:394-415) on the GPU."""
    src = np.ascontiguousarray(src, np.float32); h, w = src.shape
    dp = np.ascontiguousarray(depth_params, np.float64); dst = np.empty_like(src)
    _check(lib().rcvd_depth_apply(C.byref(cfg), C.c_int32(device), _p(dp, C.c_double), _p(src, C.c_float), _p(dst, C.c_float), C.c_int32(h), C.c_int32(w)))
    return dst


def depth_param_map(cfg, depth_params, h, w, device=0):
    """GridDepthXform::paramMap (reference lib/DepthMapTransform.cpp:950-994) on the GPU."""
    k = 2 if cfg.value_xform == abi.VALUE_SCALESHIFT else 1
    dp = np.ascontiguousarray(depth_params, np.float64); out = np.empty((h, w, k), np.float64)
    _check(lib().rcvd_depth_param_map(C.byref(cfg), C.c_int32(device), _p(dp, C.c_double), _p(out, C.c_double), C.c_int32(h), C.c_int32(w)))
    return out[:, :, 0] if k == 1 else out


def spatial_warp(cfg, spatial_params, h, w, device=0):
    """SpatialXform::warp (reference lib/DepthMapTransform.cpp:428-449) on the GPU."""
    sp = np.ascontiguousarray(spatial_params, np.float64); out = np.empty((h, w, 2), np.float32)
    _check(lib().rcvd_spatial_warp(C.byref(cfg), C.c_int32(device), _p(sp, C.c_double), _p(out, C.c_float), C.c_int32(h), C.c_int32(w)))
    return out


def flow_guided_filter(depth, cams, fwd_flow, fwd_mask, bwd_flow, bwd_mask, first_out, num_out, frame_radius, spatial_radius=0, median=False,
                       inv_aspect=1.0, far_pairs=None, far_flow=None, far_mask=None, device=0):
    """rcvd_flow_guided_filter (DepthVideoProcessor::flowGuidedFilter, reference lib/Processor.cpp:315-590) on the GPU.
    depth [F,hd,wd] f32, cams [F,9] f32, flows [F,h,w,2] f32, masks [F,h,w] u8 -> filtered depth [num_out,h,w] f32."""
    depth = np.ascontiguousarray(depth, np.float32); cams = np.ascontiguousarray(cams, np.float32)
    F, hd, wd = depth.shape
    arrs = []
    for a, dt in ((fwd_flow, np.float32), (fwd_mask, np.uint8), (bwd_flow, np.float32), (bwd_mask, np.uint8), (far_flow, np.float32), (far_mask, np.uint8)):
        arrs.append(None if a is None else np.ascontiguousarray(a, dt))
    ff, fm, bf, bm, rf, rm = arrs
    ref_mask = fm if fm is not None else rm
    if ref_mask is None:
        raise ValueError("flow masks are needed to define the output resolution")
    h, w = ref_mask.shape[1:3]
    nfar = 0 if far_pairs is None else len(far_pairs)
    fp = None if nfar == 0 else np.ascontiguousarray(far_pairs, np.int32).reshape(-1, 2)
    prm = abi.FilterParams(num_frames=F, first_out=first_out, num_out=num_out, width=w, height=h, depth_width=wd, depth_height=hd,
                           frame_radius=frame_radius, spatial_radius=spatial_radius, median=1 if median else 0, num_far=nfar, inv_aspect=inv_aspect)
    out = np.zeros((num_out, h, w), np.float32)
    _check(lib().rcvd_flow_guided_filter(C.byref(prm), C.c_int32(device), _p(depth, C.c_float), _p(cams, C.c_float),
                                         _p(ff, C.c_float), _p(fm, C.c_uint8), _p(bf, C.c_float), _p(bm, C.c_uint8),
                                         _p(fp, C.c_int32), _p(rf, C.c_float), _p(rm, C.c_uint8), _p(out, C.c_float)))
    return out


def bilateral_filter(depth, out_frames, color_bgr=None, frame_radius=2, spatial_radius=0, depth_sigma=0.3, color_sigma=0.0, median=False,
                     in_place=False, xform_cfg=None, xform_params=None, device=0):
    """rcvd_bilateral_filter (DepthVideoProcessor::bilateralFilter, reference lib/Processor.cpp:183-313) on the GPU.
    depth [F,h,w] f32, out_frames ascending local indices, color_bgr [F,h,w,3] f32 (needed when color_sigma > 0) -> [num_out,h,w] f32.
    in_place with frame_radius > 0 feeds each filtered frame, through its depth transform (xform_cfg, xform_params [F,k] f64), to the
    windows of the frames after it, as the reference does when it filters stream 0 into itself."""
    depth = np.ascontiguousarray(depth, np.float32)
    F, h, w = depth.shape
    of = np.ascontiguousarray(out_frames, np.int32).reshape(-1)
    col = None if color_bgr is None else np.ascontiguousarray(color_bgr, np.float32)
    if col is not None and col.shape != (F, h, w, 3):
        raise ValueError(f"colour stack has shape {col.shape}, expected {(F, h, w, 3)}")
    xp = None if xform_params is None else np.ascontiguousarray(xform_params, np.float64)
    prm = abi.BilateralParams(num_frames=F, width=w, height=h, num_out=len(of), frame_radius=frame_radius, spatial_radius=spatial_radius,
                              median=1 if median else 0, depth_sigma=depth_sigma, color_sigma=color_sigma, in_place=1 if in_place else 0)
    out = np.zeros((len(of), h, w), np.float32)
    _check(lib().rcvd_bilateral_filter(C.byref(prm), C.c_int32(device), _p(depth, C.c_float), _p(col, C.c_float), _p(of, C.c_int32),
                                       None if xform_cfg is None else C.byref(xform_cfg), _p(xp, C.c_double), _p(out, C.c_float)))
    return out


def build_constraints(color_bgr, pair_frames,pair_flow, pair_mask, match_separation, inv_aspect, dyn_dist=None, min_dynamic_distance=-1.0,
                      trip_frames=None, trip_flow=None, trip_mask=None, device=0):
    """rcvd_build_constraints (FlowConstraintsCollection::compute + sampleConstraints, reference lib/FlowConstraints.cpp:352-550) on the GPU.
    Returns (pair_offsets, pair_constraints [n,4], trip_offsets, trip_constraints [m,6])."""
    color = np.ascontiguousarray(color_bgr, np.float32)
    F, h, w = color.shape[:3]
    pf = np.ascontiguousarray(pair_frames, np.int32).reshape(-1, 2); P = len(pf)
    pfl = np.ascontiguousarray(pair_flow, np.float32) if P else None; pm = np.ascontiguousarray(pair_mask, np.uint8) if P else None
    T = 0 if trip_frames is None else len(trip_frames)
    tf = np.ascontiguousarray(trip_frames, np.int32) if T else None
    tfl = np.ascontiguousarray(trip_flow, np.float32) if T else None; tm = np.ascontiguousarray(trip_mask, np.uint8) if T else None
    dd = None if dyn_dist is None else np.ascontiguousarray(dyn_dist, np.float32)
    prm = abi.BuilderParams(num_frames=F, width=w, height=h, dyn_width=0 if dd is None else dd.shape[2], dyn_height=0 if dd is None else dd.shape[1],
                            match_separation=match_separation, num_pairs=P, num_triplets=T, min_dynamic_distance=min_dynamic_distance, inv_aspect=inv_aspect)
    poff = np.zeros(P + 1, np.int64); toff = np.zeros(T + 1, np.int64)
    pcap, tcap = 0, 0
    for attempt in range(2):
        pout = np.zeros((max(pcap, 1), 4), np.float32); tout = np.zeros((max(tcap, 1), 6), np.float32)
        rc = lib().rcvd_build_constraints(C.byref(prm), C.c_int32(device), _p(color, C.c_float), _p(dd, C.c_float), _p(pf if P else None, C.c_int32), _p(pfl, C.c_float), _p(pm, C.c_uint8),
                                          _p(tf, C.c_int32), _p(tfl, C.c_float), _p(tm, C.c_uint8), _p(poff, C.c_int64), _p(pout, C.c_float), C.c_int64(pcap),
                                          _p(toff, C.c_int64), _p(tout, C.c_float), C.c_int64(tcap))
        if rc == 0:
            break
        if attempt == 0 and (poff[P] > pcap or toff[T] > tcap):
            pcap, tcap = int(poff[P]), int(toff[T])      # the first call reports the sizes
            continue
        _check(rc)
    return poff, pout[:poff[P]], toff, tout[:toff[T]]


def compute_tracks(color_bgr, frame_flags, flow=None, flow_mask=None, dyn_masks=None, spawn_distance=20, prune_distance=5, min_dynamic_distance=3.0,
                   inv_aspect=1.0, device=0):
    """rcvd_compute_tracks (DepthVideoProcessor::computeTracks, reference lib/Processor.cpp:646-886) on the GPU, before the deletion of short
    tracks.  Local stacks over the frame range: color_bgr [F,h,w,3] f32, frame_flags [F] u8 (abi.TRACK_*), flow [F,h,w,2] f32 and
    flow_mask [F,h,w] u8 (slot f: pair f-1 -> f), dyn_masks [F,dh,dw] u8 or None.
    Returns (frame_offsets [F+1] i64, track ids [n] i32, locations [n,2] f32, number of ids created)."""
    color = np.ascontiguousarray(color_bgr, np.float32)
    F, h, w = color.shape[:3]
    fl = np.ascontiguousarray(frame_flags, np.uint8).reshape(-1)
    if fl.size != F:
        raise ValueError(f"{fl.size} frame flags for {F} frames")
    fw = None if flow is None else np.ascontiguousarray(flow, np.float32)
    fm = None if flow_mask is None else np.ascontiguousarray(flow_mask, np.uint8)
    dm = None if dyn_masks is None else np.ascontiguousarray(dyn_masks, np.uint8)
    prm = abi.TrackParams(num_frames=F, width=w, height=h, dyn_width=0 if dm is None else dm.shape[2], dyn_height=0 if dm is None else dm.shape[1],
                          spawn_distance=spawn_distance, prune_distance=prune_distance, min_dynamic_distance=min_dynamic_distance, inv_aspect=inv_aspect)
    off = np.zeros(F + 1, np.int64)
    n = C.c_int64(0)
    cap = F * h * w // 128 + 1024     # ample at the default spawn distance; a larger result is reported and the call repeated
    for attempt in range(2):
        ids = np.zeros(max(cap, 1), np.int32); locs = np.zeros((max(cap, 1), 2), np.float32)
        rc = lib().rcvd_compute_tracks(C.byref(prm), C.c_int32(device), _p(color, C.c_float), _p(dm, C.c_uint8), _p(fw, C.c_float), _p(fm, C.c_uint8),
                                       _p(fl, C.c_uint8), _p(off, C.c_int64), _p(ids, C.c_int32), _p(locs, C.c_float), C.c_int64(cap), C.byref(n))
        if rc == 0:
            break
        if attempt == 0 and off[F] > cap:
            cap = int(off[F])      # the first call reports the size
            continue
        _check(rc)
    return off, ids[:off[F]], locs[:off[F]], int(n.value)


def _flag_family(frames, offsets, locs, width, flags=None):
    """One constraint family of static_flags / prune_static_flags as C arguments (count, frames, offsets, locs, flags), and the flag
    array the call writes: a copy of `flags`, or zeros when it is None."""
    n = 0 if frames is None else len(frames)
    if n == 0:
        return (C.c_int32(0), None, None, None, None), np.zeros(0, np.uint8)
    fr = np.ascontiguousarray(frames, np.int32)
    off = np.ascontiguousarray(offsets, np.int64)
    loc = np.ascontiguousarray(locs, np.float32).reshape(-1, width)
    fl = np.zeros(int(off[-1]), np.uint8) if flags is None else np.array(flags, np.uint8).reshape(-1)
    return (C.c_int32(n), _p(fr, C.c_int32), _p(off, C.c_int64), _p(loc, C.c_float), _p(fl, C.c_uint8)), fl


def static_flags(masks, distance, pair_frames=None, pair_offsets=None, pair_locs=None, trip_frames=None, trip_offsets=None, trip_locs=None, want_distance=False, device=0):
    """rcvd_static_flags (FlowConstraintsCollection::setStaticFlagFromDynamicMask + dynamicDistance, reference lib/FlowConstraints.cpp:573-660,
    :257-286) on the GPU.  masks [F,h,w] u8.  Returns (pair_static u8[n], trip_static u8[m], distance images [F,h,w] f32 or None)."""
    m = np.ascontiguousarray(masks, np.uint8); F, h, w = m.shape
    pairs, ps = _flag_family(pair_frames, pair_offsets, pair_locs, 4)
    trips, ts = _flag_family(trip_frames, trip_offsets, trip_locs, 6)
    dist = np.zeros((F, h, w), np.float32) if want_distance else None
    _check(lib().rcvd_static_flags(C.c_int32(device), _p(m, C.c_uint8), C.c_int32(F), C.c_int32(h), C.c_int32(w), C.c_float(distance),
                                   *pairs, *trips, _p(dist, C.c_float)))
    return ps, ts, dist


def prune_static_flags(num_frames, height, width, distance, pair_frames, pair_offsets, pair_locs, pair_static,
                       trip_centres=None, trip_offsets=None, trip_locs=None, trip_static=None, device=0):
    """rcvd_prune_static_flags (FlowConstraintsCollection::pruneStaticFlag, reference lib/FlowConstraints.cpp:662-748) on the GPU.
    height x width: the "down" stream's size.  Arrays as in static_flags; pair_static / trip_static are the input flags (not modified).
    Returns the pruned (pair_static u8[n], trip_static u8[m])."""
    pairs, ps = _flag_family(pair_frames, pair_offsets, pair_locs, 4, pair_static)
    trips, ts = _flag_family(trip_centres, trip_offsets, trip_locs, 6, trip_static)
    _check(lib().rcvd_prune_static_flags(C.c_int32(device), C.c_int32(num_frames), C.c_int32(height), C.c_int32(width), C.c_int32(distance),
                                         *pairs, *trips))
    return ps, ts


FP64_MMA_SHAPES = ("m8n8k4", "m16n8k4", "m16n8k8", "m16n8k16")


def fp64_tensor_peaks(device=0):
    """Bench hook: live-measured fp64 tensor-core (DMMA) peak of `device` in TFLOP/s for every mma.sync f64 shape."""
    out = {}
    for i, name in enumerate(FP64_MMA_SHAPES):
        v = C.c_double()
        _check(lib().rcvd_debug_fp64_tensor_peak(C.c_int32(device), C.c_int32(i), C.byref(v)))
        out[name] = v.value
    return out
