"""The conjugate-gradient linear solver on the H100 (rcvd_cg.cuh), forced on small problems with a factor budget of 0: the solve of a
structured matrix (rcvd_debug_cg_solve_matrix) against the numpy restatement tests/cg_ref.py and the block Cholesky, whole LM solves
against a Cholesky handle on the same problem, and the storage rcvd_problem_linear_info reports.  Run with `pytest -m gpu`."""
import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import cg_ref, helpers
from tests import linalg_ref as R
from tests.test_gpu_linalg import _problem

pytestmark = pytest.mark.gpu


def _cg_problem(nf, n, pairs, eta=None):
    P = _problem(nf, n, pairs)
    P.set_factor_budget(0)
    if eta is not None:
        P.set_cg_tolerance(eta)
    return P


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(b))


# npad <= 224 (k_potrf_smem) and > 224 (k_potrf_panel + k_potrf_trail); chain, hierarchical and disconnected frame graphs
MATRIX_CASES = [(45, "chain", 8), (23, "hierarchical2", 60), (61, "disconnected", 9), (250, "chain", 4), (240, "disconnected", 5)]


@pytest.mark.parametrize("mode", ["well", "lm"])
@pytest.mark.parametrize("nf,graph,n", MATRIX_CASES, ids=[f"{g}{n}-nf{nf}" for nf, g, n in MATRIX_CASES])
def test_cg_solve_matrix_matches_the_restatement(nf, graph, n, mode):
    pairs = R.GRAPHS[graph](n)
    if mode == "well":
        H, D2, b, _ = R.well_conditioned(n, nf, pairs, seed=nf)
    else:
        H, D2, b = R.lm_like(n, nf, pairs, 1e4, seed=nf)
    A = H + np.diag(D2)
    P = _cg_problem(nf, n, pairs)
    y, it = P.cg_solve_matrix(H, D2, b)
    ref = cg_ref.pcg(A, b, nf)
    near = any(abs(z - cg_ref.ETA) <= 1e-8 for z in ref["zeta"])
    print(f"CG {graph}{n} nf={nf} {mode}: iterations {it} (reference {ref['iterations']}, zeta near eta: {near}) |y - ref| {_rel(y, ref['x']):.2e}")
    assert not ref["broke"] and not ref["capped"]
    if not near:
        assert it == ref["iterations"]
        assert _rel(y, ref["x"]) <= 1e-9
    # deterministic: the same iterates bit for bit
    y2, it2 = P.cg_solve_matrix(H, D2, b)
    assert it2 == it and np.array_equal(y2, y)
    # the preconditioner ran on the per-frame Cholesky kernels; nothing of the block factorisation's off-diagonal machinery did
    paths = P.linear_paths()
    assert paths["potrf_smem" if nf <= 224 else "potrf_panel"] > 0 and paths["trinv"] > 0
    for k in ("trsm_ll4", "trsm_ll2", "trsm_gemm", "update_tma1", "update_tma2", "substitution_levels", "substitution_fused"):
        assert paths[k] == 0, k


@pytest.mark.parametrize("nf,graph,n", MATRIX_CASES, ids=[f"{g}{n}-nf{nf}" for nf, g, n in MATRIX_CASES])
def test_cg_at_tiny_eta_equals_the_cholesky_solve(nf, graph, n):
    """eta = 1e-14: the CG runs until its quadratic model stops decreasing in floating point, ~1e-8 relative error in y (see
    tests/test_cg.py); the Cholesky solve of the same well-conditioned system is exact to 1e-12 (FORWARD_TOL)."""
    pairs = R.GRAPHS[graph](n)
    H, D2, b, x = R.well_conditioned(n, nf, pairs, seed=nf + 1)
    P = _cg_problem(nf, n, pairs, eta=1e-14)
    y, it = P.cg_solve_matrix(H, D2, b)
    yc = _problem(nf, n, pairs).solve_matrix(H, D2, b)
    print(f"CG-TIGHT {graph}{n} nf={nf}: iterations {it} |y - y_chol| {_rel(y, yc):.2e} |y_chol - x*| {_rel(yc, x):.2e}")
    assert R.forward_error(yc, x) <= R.FORWARD_TOL
    assert _rel(y, yc) <= 1e-7


def test_breakdown_and_zero_rhs():
    nf, n = 16, 2
    pairs = R.chain(n)
    P = _cg_problem(nf, n, pairs)
    H, D2, b, _ = R.well_conditioned(n, nf, pairs)
    y, it = P.cg_solve_matrix(H, D2, np.zeros_like(b))
    assert it == 0 and not np.any(y)
    # coupling far stronger than the diagonal blocks: indefinite, positive diagonal blocks; the restatement breaks down as well
    Hi = H.copy(); Hi[:nf, nf:] *= 50.0; Hi[nf:, :nf] *= 50.0
    assert cg_ref.pcg(Hi + np.diag(D2), b, nf)["broke"]
    with pytest.raises(RuntimeError, match="conjugate gradients broke down"):
        P.cg_solve_matrix(Hi, D2, b)
    y, it = P.cg_solve_matrix(H, D2, b)                  # the handle recovers
    assert np.linalg.norm(y - np.linalg.solve(H + np.diag(D2), b)) <= 0.5 * np.linalg.norm(y)


def test_cholesky_handle_refuses_the_cg_hook_and_cg_handle_has_no_factor():
    nf, n = 16, 3
    pairs = R.chain(n)
    H, D2, b, _ = R.well_conditioned(n, nf, pairs)
    with pytest.raises(RuntimeError, match="block Cholesky"):
        _problem(nf, n, pairs).cg_solve_matrix(H, D2, b)
    P = _cg_problem(nf, n, pairs)
    P.cg_solve_matrix(H, D2, b)
    with pytest.raises(RuntimeError, match="conjugate gradients"):
        P.factor_dense()
    with pytest.raises(RuntimeError, match="conjugate gradients"):
        P.profile_linear()


# ---------------------------------------------------------------------------------------------------------
# whole LM solves: the CG handle against a Cholesky handle on the same problem
# ---------------------------------------------------------------------------------------------------------
def _handles(build, budget_zero_eta):
    """Two handles on the problem build() sets up: the default (block Cholesky) and one forced to CG."""
    G, C = build(), build()
    C.set_factor_budget(0)
    if budget_zero_eta is not None:
        C.set_cg_tolerance(budget_zero_eta)
    assert G.linear_info()["solver"] == abi.LINEAR_CHOLESKY and C.linear_info()["solver"] == abi.LINEAR_CG
    return G, C


def _bench_case(name, frames=None):
    import bench

    def build():
        spec, sc, cfg, pairs, offs, rec, med = bench.build_case(name, frames=frames)
        P = solver.Problem(cfg)
        helpers.setup_problem(P, cfg, pairs, offs, rec, med, bench.initial_state(sc, cfg, solver.frame_stride(cfg)))
        return P
    return build


def _variant_case(kind):
    """8-frame problems with the other residual families and parameterisations."""
    def build():
        if kind == "triplets":
            sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=8, depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=4)
        elif kind == "depth_pairs_bounded":
            sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=8, sep=12, depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=3,
                                                               depth_lower_bound=1, scale_grid_x=5, scale_grid_y=4, depth_deform_reg=1.0)
        else:
            sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=8, **dict(helpers.VARIANTS)[kind])
        P = solver.Problem(cfg)
        off_d, nd = helpers.layout_numbers(cfg)
        x = helpers.initial_state(sc, cfg, P.stride, off_d, nd)
        if kind == "depth_pairs_bounded":       # normalizeDepth: the depth pairs alone, the lower bound on the scales
            P.set_frames(np.ones(cfg.num_frames, np.uint8), med)
            P.set_depth_pairs(pairs, offs, rec)
            P.set_state(x)
            return P
        helpers.setup_problem(P, cfg, pairs, offs, rec, med, x)
        if kind == "triplets":
            P.set_triplets(*sc.triplets(sep=14))
        return P
    return build


LM_CASES = [("config1", _bench_case("config1_8f_128x96_grid4x4_sep10")), ("config2", _bench_case("config2_300f_384x224_grid16x12_sep10")),
            ("triplets", _variant_case("triplets")), ("depth_pairs_bounded", _variant_case("depth_pairs_bounded")),
            ("fixed_poses", _variant_case("identitydepth_fixposes")), ("shared_intrinsics", _variant_case("bicubic_shared_ratio_bicubicwarp"))]


@pytest.mark.parametrize("name,build", LM_CASES, ids=[c[0] for c in LM_CASES])
def test_lm_trajectory_at_tiny_eta_matches_the_cholesky(name, build):
    """With eta = 1e-14 the CG steps are the Cholesky's to ~1e-8 (the floor of the quadratic-model test, tests/test_cg.py).  Solving
    from the same start with an LM iteration cap of k = 1, 2, ... gives the trajectory step by step: the same iterations and
    successful steps (the same accepted / rejected sequence) and the same cost of the best iterate at every k <= 6, within 1e-8
    relative: the step's 1e-8 moves the cost by up to a few 1e-9 where a step still decreases it a lot, and the nonlinear trajectory
    carries such differences on (triplets: 3.4e-9 at k = 7, 2.8e-8 at k = 8).  Worst gaps over k <= 12 measured on an H100 80GB
    HBM3: config1 2.4e-10, config2 3.0e-11 (k <= 6), depth_pairs_bounded 1.2e-10, fixed_poses 2.6e-16, shared_intrinsics 2.0e-9.
    (The candidate cost of a rejected step is not compared: at config 2 the first, weakly damped steps overshoot to ~1e16, where 1e-8
    of the step moves the candidate's cost by ~1e-4.)"""
    G, C = _handles(build, 1e-14)
    x0 = G.get_state()
    K = 6
    worst = 0.0
    for k in range(1, K + 1):
        opt = abi.default_solve_options(max_iterations=k)
        G.set_state(x0); C.set_state(x0)
        sg, sc = G.solve(opt), C.solve(opt)
        assert (sg.iterations, sg.num_successful_steps, sg.termination) == (sc.iterations, sc.num_successful_steps, sc.termination), k
        worst = max(worst, abs(sg.final_cost - sc.final_cost) / abs(sg.final_cost))
        assert abs(sg.final_cost - sc.final_cost) <= 1e-8 * abs(sg.final_cost), (k, sg.final_cost, sc.final_cost)
        info = C.linear_info()
        assert info["cg_solves"] == sc.iterations and info["cg_iterations"] > 0
        if sg.iterations < k:
            break
    print(f"LM-TIGHT {name}: {sc.iterations} iterations ({sc.num_successful_steps} successful), worst cost gap {worst:.2e}, CG iterations "
          f"{info['cg_iterations']} (max {info['cg_max_iterations']}, capped {info['cg_capped_steps']})")


@pytest.mark.parametrize("name,build", LM_CASES, ids=[c[0] for c in LM_CASES])
def test_lm_with_default_eta_converges_to_the_cholesky_cost(name, build):
    """Default eta = 0.1 (inexact Newton steps): the solve converges, to the Cholesky's final cost within 1e-3 relative.  Measured on an
    H100 80GB HBM3 (relative final-cost gap, LM iterations Cholesky / CG): config1 7.4e-8 (19 / 21), config2 1.3e-6 (43 / 61),
    triplets 7.0e-7 (16 / 19), depth_pairs_bounded 2.3e-7 (6 / 7), fixed_poses 1.8e-7 (4 / 5), shared_intrinsics 3.1e-7 (15 / 15)."""
    G, C = _handles(build, None)
    sg, sc = G.solve(), C.solve()
    info = C.linear_info()
    gap = abs(sc.final_cost - sg.final_cost) / abs(sg.final_cost)
    print(f"LM-DEFAULT {name}: cholesky {sg.iterations} it cost {sg.final_cost:.8e} ({sg.message.decode()}); cg {sc.iterations} it cost "
          f"{sc.final_cost:.8e} ({sc.message.decode()}) gap {gap:.2e}; CG iterations {info['cg_iterations']} max {info['cg_max_iterations']} capped {info['cg_capped_steps']}")
    assert sg.termination == abi.TERM_CONVERGENCE
    assert sc.termination == abi.TERM_CONVERGENCE, sc.message
    assert gap <= 1e-3


def test_linear_info_reports_the_cg_storage():
    n = 40
    import bench
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case("config2_300f_384x224_grid16x12_sep10", frames=n)
    host = solver.linear_storage(cfg, pairs)
    for budget, path in ((0, abi.LINEAR_CG), (-1, abi.LINEAR_CHOLESKY)):
        P = solver.Problem(cfg)
        helpers.setup_problem(P, cfg, pairs, offs, rec, med, bench.initial_state(sc, cfg, solver.frame_stride(cfg)))
        P.set_factor_budget(budget)
        info = P.linear_info()
        assert info["solver"] == path
        assert (info["cholesky_bytes"], info["cg_bytes"]) == (host["cholesky_bytes"], host["cg_bytes"])
        if path == abi.LINEAR_CG:
            assert info["device_bytes"] == host["cg_bytes"] and info["factor_blocks"] == n       # no fill, no off-diagonal factor blocks
            assert info["budget_bytes"] == 0
        else:
            st = P.structure_info()
            assert info["device_bytes"] == host["cholesky_bytes"] and info["factor_blocks"] == n + 2 * st["offdiag_factor_blocks"]
            assert info["budget_bytes"] > 0
        s = P.solve(abi.default_solve_options(max_iterations=3))
        info = P.linear_info()
        if path == abi.LINEAR_CG:
            assert info["cg_solves"] == s.iterations and 0 < info["cg_max_iterations"] <= 500
            assert info["cg_max_iterations"] <= info["cg_iterations"] <= 500 * info["cg_solves"]
        else:
            assert info["cg_solves"] == 0 and info["cg_iterations"] == 0
