"""The CPU oracle at the geometric edges of tests/eval_edges_cases.py: its analytic Jacobian against its literal Jet autodiff (the
restatement of Ceres' DynamicAutoDiffCostFunction that tests/test_gpu_eval_edges.py holds the CUDA kernels to), and the Jet Jacobian
against central finite differences of the residuals.  Establishes that the reference itself is right where the GPU tests use it."""
import numpy as np
import pytest

from robust_cvd_b200 import abi
from tests import eval_edges_cases as E
from tests import helpers

DBL_EPS = np.finfo(np.float64).eps


def _oracle(name):
    from oracle import oracle
    cfg, pairs, offs, rec, med, x, (ce, to, tr) = E.build(name)
    O = oracle.OracleProblem(cfg)
    helpers.setup_problem(O, cfg, pairs, offs, rec, med, x)
    O.set_triplets(ce, to, tr)
    return cfg, O, x.reshape(-1).copy(), rec


def _rows_match(r0, J0, r1, J1):
    """Residuals to 1e-13 of the largest, Jacobian rows to 1e-12 of each row's largest entry; non-finite residuals in the same slots."""
    fin = np.isfinite(r1)
    assert np.array_equal(fin, np.isfinite(r0))
    assert np.isfinite(J0).all() and np.isfinite(J1).all()
    assert np.abs(r0 - r1)[fin].max(initial=0) <= 1e-13 * np.abs(r1[fin]).max(initial=0)
    if J1.size:
        assert (np.abs(J0 - J1).max(axis=1) <= 1e-12 * np.abs(J1).max(axis=1)).all()


@pytest.mark.parametrize("name", E.CASES)
def test_analytic_jacobian_matches_jet(name):
    cfg, O, x, rec = _oracle(name)
    _rows_match(*O.static_jacobian(0), *O.static_jacobian(1))
    _rows_match(*O.regulariser_jacobian(0), *O.regulariser_jacobian(1))


def _finite_differences(residuals, x):
    """Central differences of residuals() over every state column, step h_j = 1e-6 max(1, |x_j|).  (r, F [rows, columns], h)."""
    steps = 1e-6 * np.maximum(1.0, np.abs(x))
    cols = []
    for j in range(x.size):
        xp, xm = x.copy(), x.copy(); xp[j] += steps[j]; xm[j] -= steps[j]
        cols.append((residuals(xp) - residuals(xm)) / (xp[j] - xm[j]))
    return residuals(x), np.stack(cols, 1), steps


def _check_fd(r, J, F, steps, skip_rows):
    """|F - J| per row within 1e-7 of the row's largest |J| plus the rounding of the difference quotient, 4 eps |r| / h.
    1e-7 covers the truncation of the central difference (h^2 |r'''| / 6, about 1e-12 here) and the small-angle branch of
    ceres::AngleAxisRotatePoint: below theta^2 = DBL_EPSILON it is first order, exact to O(theta) ~ 1.5e-8 of the rotated point."""
    keep = np.isfinite(r) & ~skip_rows
    tol = 1e-7 * np.abs(J).max(axis=1, keepdims=True) + 4 * DBL_EPS * np.abs(r)[:, None] / steps[None, :]
    bad = (np.abs(F - J) > tol) & keep[:, None]
    assert not bad.any(), (np.argwhere(bad)[:5], F[bad][:5], J[bad][:5])


def _switch_rows(r, J, loss_is_ratio_or_log, steps):
    """Depth rows (every third) of the max / min losses whose switch A = B (where the residual is 0) lies within the step of some column:
    |r| below the largest change a step can make, 10 |dr/dx| h."""
    skip = np.zeros(r.shape, bool)
    if loss_is_ratio_or_log:
        reach = 10 * (np.abs(J) * steps[None, :]).max(axis=1)
        skip[2::3] = (np.abs(r) <= reach)[2::3]
    return skip


@pytest.mark.parametrize("name", E.CASES)
def test_jet_jacobian_matches_finite_differences(name):
    """Every column, every row of the static pairs, smoothness triplets and regularisers.  Skipped: the depth rows of the depth-ratio
    and log-depth losses within a step of their max / min switch (none at these states; _switch_rows finds them).  The other kinks stay
    out of reach of the 1e-6 steps: clamped target depths are 1e-8 times their scale, 100 x under the 1e-6 clamp of the disparity
    loss, negated depths are far below it, and the deformation regulariser's min(|a|, |b|) switch needs two nodes within a step of
    each other in magnitude (the state's nodes differ by the 0.01 noise)."""
    cfg, O, x, rec = _oracle(name)
    O.set_jacobian_mode(1)
    ratio_log = cfg.static_loss_type in (abi.LOSS_REPRO_DEPTH_RATIO, abi.LOSS_REPRO_LOG_DEPTH)
    smooth_ratio_log = cfg.smooth_loss_type in (2, 3)

    def at(fn):
        def residuals(v):
            O.set_state(v)
            return fn()
        return residuals
    for fn, jac, ratio in ((lambda: O.static_jacobian(1, jac=False)[0], lambda: O.static_jacobian(1), ratio_log),
                           (lambda: O.triplet_jacobian()[0], O.triplet_jacobian, smooth_ratio_log),
                           (lambda: O.regulariser_jacobian(1)[0], lambda: O.regulariser_jacobian(1), False)):
        O.set_state(x)
        r, J = jac()
        r_fd, F, steps = _finite_differences(at(fn), x)
        O.set_state(x)
        assert np.array_equal(r_fd, r, equal_nan=True)
        skip = _switch_rows(r, J, ratio, steps)
        assert skip.sum() <= 0.01 * max(r.size, 1)
        _check_fd(r, J, F, steps, skip)


def test_the_cases_reach_their_edges():
    """Each case takes the branch it is named for, in the oracle: Huber on both sides of its threshold, Cauchy in its tail (rho' << 1),
    non-finite residuals exactly in the log-depth case with points behind the camera."""
    for name in E.CASES:
        cfg, O, x, rec = _oracle(name)
        r, _ = O.static_jacobian(1, jac=False)
        s = (r.reshape(-1, 3) ** 2).sum(1)
        assert np.isfinite(r).all() == (name not in E.NONFINITE), name
        if name == "huber_both_sides":
            b = cfg.robustness ** 2
            assert cfg.robust_type == abi.ROBUST_HUBER and (s > b).sum() > 100 and (s <= b).sum() > 100
        if name == "cauchy_tail":
            assert (1.0 / (1.0 + s / cfg.robustness ** 2) < 0.01).mean() > 0.5
        if name == "groups_sizes":
            cfg, pairs, offs, rec, med, x, _ = E.build(name)
            assert sorted(np.diff(offs).tolist()) == sorted(E.GROUP_COUNTS)
    # the transformed target depth of the clamped records is below 1e-6: the disparity residual is 1 / eps - 1 / A
    cfg, O, x, rec = _oracle("disparity_clamp")
    r, _ = O.static_jacobian(1, jac=False)
    assert (r[2::3][::11] < -0.99e6).all()


@pytest.mark.parametrize("name", E.NONFINITE)
def test_nonfinite_rows_agree_between_modes(name):
    """log(min / max) of a negative depth ratio: the same rows are NaN under the analytic and the Jet Jacobian (only the depth row of
    each such record), their Jacobians stay finite, and the cost is NaN."""
    cfg, O, x, rec = _oracle(name)
    r0, J0 = O.static_jacobian(0)
    r1, J1 = O.static_jacobian(1)
    bad = ~np.isfinite(r1)
    assert bad.any() and np.array_equal(bad, ~np.isfinite(r0))
    assert not bad[0::3].any() and not bad[1::3].any()
    assert np.array_equal(np.nonzero(bad[2::3])[0], np.nonzero(rec[:, 2] < 0)[0])
    assert np.isfinite(J0).all() and np.isfinite(J1).all()
    for mode in (0, 1):
        O.set_jacobian_mode(mode)
        assert np.isnan(O.evaluate())


def first_step_candidate_cost(O, x, radius):
    """The candidate cost of the first Levenberg-Marquardt step of the oracle's solve at x (Jacobi scaling S, LM diagonal clamped to
    [min_lm_diagonal, max_lm_diagonal] over the radius, step -S (S H S + D)^-1 S g), restated with numpy."""
    opt = abi.default_solve_options()
    O.set_state(x)
    c, g = O.evaluate(True)
    Hm = O.normal_matrix_dense()
    d = np.diag(Hm)
    S = 1.0 / (1.0 + np.sqrt(d))
    D = np.clip(S * S * d, opt.min_lm_diagonal, opt.max_lm_diagonal) / radius
    act = O.active_mask()
    y = np.zeros_like(g)
    y[act] = np.linalg.solve((Hm * S[:, None] * S[None, :] + np.diag(D))[np.ix_(act, act)], (S * g)[act])
    O.set_state(x - S * y)
    cand = O.evaluate()
    O.set_state(x)
    return c, cand


def test_log_step_behind_takes_nonfinite_steps():
    """The state of eval_edges_cases.log_step_behind is finite, its first full steps at radius 1e4, 1e3 and 1e2 are not; the oracle's
    solve rejects them (a non-finite candidate counts as an increase) and converges."""
    from oracle import oracle
    cfg, pairs, offs, rec, med, x = E.log_step_behind()
    O = oracle.OracleProblem(cfg)
    helpers.setup_problem(O, cfg, pairs, offs, rec, med, x)
    for radius in (1e4, 1e3, 1e2):
        c, cand = first_step_candidate_cost(O, x.reshape(-1), radius)
        assert np.isfinite(c) and not np.isfinite(cand), radius
    s = O.solve(abi.default_solve_options(max_iterations=60))
    assert s.termination == abi.TERM_CONVERGENCE and s.num_unsuccessful_steps >= 4 and s.final_cost < 0.1 * s.initial_cost
