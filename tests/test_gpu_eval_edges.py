"""The residual and Jacobian kernels on the H100 at the geometric edges of tests/eval_edges_cases.py, against the CPU oracle's literal
Jet autodiff (set_jacobian_mode(1): Ceres' DynamicAutoDiffCostFunction restated, not the hand derivation the kernels share with the
oracle's analytic mode).  tests/test_eval_edges_ref.py establishes the oracle at the same cases without a GPU.

Per case: the rows of rcvd_evaluate_rows (k_pairs, k_triplets, k_regularisers in the Rows mode), the cost and gradient of k_pairs, and the
normal matrix, cost and gradient of the CostGradH pair kernel each fast-path setting selects (k_pairs, k_accumulate_runs,
k_accumulate_fast; which one ran is read from the handle's launch counters).  Tolerances are those of tests/test_gpu_rows.py and
tests/test_gpu_parity.py.

Non-finite residuals (log depth of a point behind the receiving camera): the rows are NaN in the same slots as the oracle's, the cost is
NaN, and the gradient is NaN in exactly the oracle's entries -- every column the NaN row reaches.  The normal matrix stays finite: rho'
of a NaN s is fmax(DBL_MIN, NaN) = DBL_MIN (ceres::CauchyLoss computes std::max(min, NaN) = min alike), so the row enters H scaled by
sqrt(DBL_MIN).  That is accepted: an evaluation with a NaN cost never becomes an iterate -- the LM step acceptance reads a non-finite
candidate cost as an increase and rejects the step, as Ceres does -- so H is only ever factored at states whose rows are all finite.
test_nonfinite_steps_are_rejected_as_by_the_oracle pins that acceptance end to end."""
import numpy as np
import pytest

from robust_cvd_b200 import abi
from tests import depth_pairs_ref as R
from tests import eval_edges_cases as E
from tests import helpers

pytestmark = pytest.mark.gpu

FAST_PATHS = (0, 1, 2)


def _constant(cfg, stride):
    """Per global column: the parameter is held constant."""
    from robust_cvd_b200 import solver
    offS = solver.spatial_param_offset(cfg)
    c = np.zeros(stride, bool)
    c[:6] = bool(cfg.fix_poses); c[6] = cfg.intr_opt == abi.INTR_FIXED
    c[7:offS] = bool(cfg.fix_depth_xforms); c[offS:] = bool(cfg.fix_spatial_xforms)
    return np.tile(c, cfg.num_frames)


def _dense(cols, J, U):
    """(cols, J) [n, m, k] -> J [n * m, U]; checks the padding (-1 and 0, after the used slots) and that no column repeats in a row."""
    n, m, k = J.shape
    c = cols.reshape(n * m, k); v = J.reshape(n * m, k)
    used = c >= 0
    assert (v[~used] == 0).all()
    assert (used[:, 1:] <= used[:, :-1]).all()                 # the unused slots come last
    s = np.sort(np.where(used, c, -1 - np.arange(k)[None, :]), axis=1)
    assert (s[:, 1:] != s[:, :-1]).all()
    assert c.max(initial=-1) < U
    D = np.zeros((n * m, U))
    rr = np.repeat(np.arange(n * m), k).reshape(n * m, k)
    D[rr[used], c[used]] = v[used]
    return D


def _close(a, ref, rel, floor=0.0):
    """Non-finite entries in the same places; the finite ones within rel of max(floor, largest finite |ref|)."""
    a, ref = np.asarray(a, np.float64).reshape(-1), np.asarray(ref, np.float64).reshape(-1)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(a), fin), (np.nonzero(np.isfinite(a) != fin)[0][:10])
    err = np.abs(a - ref)[fin].max(initial=0)
    assert err <= rel * max(floor, np.abs(ref[fin]).max(initial=0)), (err, rel)
    return err


def _match(r, J, r_ref, J_ref, rho, rho_ref):
    """tests/test_gpu_rows.py's tolerances: r and rho to 1e-10 of the largest, J to 1e-9 of each row's largest entry.  Finite rows
    match; non-finite residuals sit in the same slots and their Jacobian rows are finite and match too."""
    assert r.size == r_ref.size and J.shape == J_ref.shape
    _close(r, r_ref, 1e-10)
    _close(rho, rho_ref, 1e-10)
    assert np.isfinite(J).all() and np.isfinite(J_ref).all()
    if J.size:
        assert (np.abs(J - J_ref).max(axis=1) <= 1e-9 * np.abs(J_ref).max(axis=1)).all()


def _problems(cfg, pairs, offs, rec, med, x, triplets=None):
    """The oracle in Jet mode and the CUDA problem on the same inputs."""
    from oracle import oracle
    from robust_cvd_b200 import solver
    O = oracle.OracleProblem(cfg); G = solver.Problem(cfg)
    assert O.stride == G.stride
    O.set_jacobian_mode(1)
    for P in (O, G):
        helpers.setup_problem(P, cfg, pairs, offs, rec, med, x)
        if triplets is not None:
            P.set_triplets(*triplets)
    return O, G


def _pair_kernels_run(G, fn):
    """The pair kernels that assembled a normal matrix during fn(), from G's launch counters (rcvd_debug_pair_kernel_launches)."""
    before = G.pair_kernel_launches()
    fn()
    after = G.pair_kernel_launches()
    return {k for k in after if after[k] > before[k]}


def _intended_kernel(cfg, fast_path):
    """The CostGradH pair kernel a fast-path setting selects (rcvd_api.cu enqueue_residuals): 0 the generic k_pairs; 1 the run path on
    bilinear depth grids, else k_accumulate_fast where it serves the configuration; 2 k_accumulate_fast wherever it serves."""
    tc = (cfg.value_xform == abi.VALUE_SCALE and cfg.spatial_type == abi.SPATIAL_IDENTITY and cfg.intr_opt != abi.INTR_SHARED and
          not (cfg.fix_poses or cfg.fix_depth_xforms or cfg.fix_spatial_xforms) and not (cfg.depth_type == abi.DEPTH_GRID and cfg.depth_cubic))
    if fast_path == 0 or not tc:
        return "k_pairs"
    if fast_path == 1 and cfg.depth_type == abi.DEPTH_GRID:
        return "k_accumulate_runs"
    return "k_accumulate_fast"


def _reference_rows(cfg, O, U, const, tr):
    """The oracle's rows per family: (r, J with constant columns zeroed, rho)."""
    ro, Jo = O.static_jacobian(1)
    ref = {"pairs": (ro, Jo, R.robust(cfg, (ro.reshape(-1, 3) ** 2).sum(1))[0])}
    rt, Jt = O.triplet_jacobian()
    ref["triplets"] = (rt, Jt, tr[:, 9].astype(np.float64) * (rt.reshape(-1, 3) ** 2).sum(1))
    rg, Jg = O.regulariser_jacobian(1)
    ref["regularisers"] = (rg, Jg, rg * rg)
    return {f: (r, np.where(const[None, :], 0.0, J), rho) for f, (r, J, rho) in ref.items()}


@pytest.mark.parametrize("name", E.CASES)
def test_rows_match_jet_autodiff(name):
    cfg, pairs, offs, rec, med, x, trip = E.build(name)
    O, G = _problems(cfg, pairs, offs, rec, med, x, trip)
    ref = _reference_rows(cfg, O, G.U, _constant(cfg, G.stride), trip[2])
    for f, (r_ref, J_ref, rho_ref) in ref.items():
        r, rho, cols, J = G.rows(f, jacobian=True)
        _match(r, _dense(cols, J, G.U), r_ref, J_ref, rho, rho_ref)
    assert np.isfinite(G.rows("pairs")[0]).all() == (name not in E.NONFINITE)


@pytest.mark.parametrize("name", E.CASES)
def test_cost_gradient_and_normal_matrix_on_every_fast_path(name):
    """Each fast-path setting: the pair kernel it selects ran (from the launch counters), its normal matrix and -- read back from one timed LM
    step, rcvd_debug_last_iteration -- its cost and gradient match the Jet oracle (tests/test_gpu_parity.py's tolerances: cost 1e-11,
    g 1e-9, H 1e-9 of the largest entry), and so do the cost and gradient of rcvd_evaluate (k_pairs in the CostGrad mode).  The three
    settings agree with each other to 1e-10 (tests/test_gpu_parity.py::test_fast_kernel_matches_generic)."""
    cfg, pairs, offs, rec, med, x, trip = E.build(name)
    O, G = _problems(cfg, pairs, offs, rec, med, x, trip)
    co, go = O.evaluate(True)
    Ho = O.normal_matrix_dense()
    assert np.isfinite(Ho).all()
    if name not in E.LOCATIONS or (cfg.depth_type == abi.DEPTH_GRID and not cfg.depth_cubic):
        assert _intended_kernel(cfg, 1) == "k_accumulate_runs" and _intended_kernel(cfg, 2) == "k_accumulate_fast"   # the cases meant for them
    out = {}
    for fp in FAST_PATHS:
        G.set_fast_path(fp)
        G.set_state(x)
        Hs = []
        ran = _pair_kernels_run(G, lambda: Hs.append(G.normal_matrix_dense()))
        assert ran == {_intended_kernel(cfg, fp)}, (fp, ran)
        Hg = Hs[0]
        assert np.isfinite(Hg).all()
        assert np.abs(Hg - Ho).max() <= 1e-9 * np.abs(Ho).max()
        cg, gg = G.evaluate(True)
        assert _pair_kernels_run(G, lambda: G.time_iteration(iters=1)) == {_intended_kernel(cfg, fp)}, fp
        it = G.last_iteration()
        ch, gh = it["cost"], it["gradient"].reshape(-1)
        for c in (cg, ch):
            if np.isfinite(co):
                assert abs(c - co) <= 1e-11 * abs(co), (fp, c, co)
            else:
                assert not np.isfinite(c), (fp, c)
        for g in (gg, gh):
            _close(g, go, 1e-9, floor=1.0)
        out[fp] = (Hg, ch, gh)
    H0, c0, g0 = out[0]
    for fp in (1, 2):
        Hf, cf, gf = out[fp]
        assert np.abs(Hf - H0).max() <= 1e-10 * np.abs(H0).max()
        _close(gf, g0, 1e-10, floor=1.0)
        if np.isfinite(c0):
            assert abs(cf - c0) <= 1e-12 * abs(c0)


RUN_PATH_CASES = [n for n in E.LOCATIONS if "depth_bilinear" in n] + E.GROUPS


@pytest.mark.parametrize("name", RUN_PATH_CASES)
def test_run_path_keys_at_grid_lines_and_borders(name):
    """Records on grid lines and borders of a bilinear depth grid, each pair's records shuffled: the run path sorts them on the device
    by the cells of k_record_keys and gathers them in k_accumulate_runs.  Its normal matrix equals the generic kernel's and the Jet
    oracle's, and the rows come back in the caller's (shuffled) order."""
    cfg, pairs, offs, rec, med, x, trip = E.build(name)
    rng = np.random.default_rng(11)
    rec = np.concatenate([rec[offs[i]:offs[i + 1]][rng.permutation(offs[i + 1] - offs[i])] for i in range(len(pairs))])
    O, G = _problems(cfg, pairs, offs, rec, med, x)
    Ho = O.normal_matrix_dense()
    G.set_fast_path(1)
    Hr = []
    assert _pair_kernels_run(G, lambda: Hr.append(G.normal_matrix_dense())) == {"k_accumulate_runs"}
    G.set_fast_path(0)
    Hg = G.normal_matrix_dense()
    assert np.abs(Hr[0] - Hg).max() <= 1e-10 * np.abs(Hg).max()
    assert np.abs(Hr[0] - Ho).max() <= 1e-9 * np.abs(Ho).max()
    ro, Jo = O.static_jacobian(1)
    r, rho, cols, J = G.rows("pairs", jacobian=True)
    _match(r, _dense(cols, J, G.U), ro, Jo, rho, R.robust(cfg, (ro.reshape(-1, 3) ** 2).sum(1))[0])


@pytest.mark.parametrize("fast_path", FAST_PATHS)
def test_nonfinite_steps_are_rejected_as_by_the_oracle(fast_path):
    """eval_edges_cases.log_step_behind: a finite log-depth state whose first full LM steps put points behind the receiving camera.
    The GPU's first candidate cost is non-finite as the oracle's (test_eval_edges_ref.py restates that step); its solve rejects those
    steps and ends where the oracle's does: same termination, iterations within 2, final cost to 1e-6."""
    cfg, pairs, offs, rec, med, x = E.log_step_behind()
    O, G = _problems(cfg, pairs, offs, rec, med, x)
    G.set_fast_path(fast_path)
    assert np.isfinite(G.evaluate())
    G.time_iteration(iters=1)
    it = G.last_iteration()
    assert np.isfinite(it["cost"]) and not np.isfinite(it["candidate_cost"])
    G.set_state(x)
    opt = abi.default_solve_options(max_iterations=60)
    so, sg = O.solve(opt), G.solve(opt)
    assert sg.num_unsuccessful_steps >= 4
    assert so.termination == sg.termination, (so.message, sg.message)
    assert abs(so.iterations - sg.iterations) <= 2, (so.iterations, sg.iterations)
    assert abs(so.final_cost - sg.final_cost) <= 1e-6 * abs(so.final_cost), (so.final_cost, sg.final_cost)


@pytest.mark.parametrize("name", E.NONFINITE)
def test_nonfinite_cost_on_every_fast_path(name):
    cfg, pairs, offs, rec, med, x, trip = E.build(name)
    O, G = _problems(cfg, pairs, offs, rec, med, x, trip)
    assert not np.isfinite(O.evaluate())
    for fp in FAST_PATHS:
        G.set_fast_path(fp)
        assert not np.isfinite(G.evaluate())


def test_identity_start_solve_matches_oracle():
    """One solve from the reference's starting point (every rotation exactly 0, so every rotation of the first evaluation takes the
    small-angle branch) on an 8-frame bilinear-grid disparity problem; tests/test_gpu_parity.py::test_lm_solve_matches_oracle's
    tolerances."""
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=8, depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=4)
    off_d, nd = helpers.layout_numbers(cfg)
    x = sc.identity_state(E.frame_stride(cfg), off_d, nd)
    assert (x[:, 3:6] == 0).all()
    O, G = _problems(cfg, pairs, offs, rec, med, x)
    opt = abi.default_solve_options(max_iterations=60)
    so, sg = O.solve(opt), G.solve(opt)
    assert sg.gpu_launches > 0
    assert so.termination == sg.termination, (so.message, sg.message)
    assert abs(so.final_cost - sg.final_cost) <= 1e-6 * abs(so.final_cost), (so.final_cost, sg.final_cost)
    assert abs(so.iterations - sg.iterations) <= 2
    xo, xg = O.get_state(), G.get_state()
    assert np.linalg.norm(xo - xg) / np.linalg.norm(xo) < 1e-4
