"""CPU checks of rcvd_covariance's mathematics (no GPU): the numpy restatement of the selected inversion (tests/covariance_ref.py)
against a dense inverse, the rank test on a gauge-deficient matrix, and the measured premise behind the default min_pivot = 1e-10:
at the LM solution of the seeded synthetic problems the Jacobi-scaled normal matrix has exactly the six null directions of the
similarity gauge, which the pivot test catches, and holding frame 0's pose removes them with pivots far above the threshold."""
import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import covariance_ref as CR
from tests import helpers
from tests import linalg_ref as R

GRAPHS = [("chain", 6), ("star", 6), ("complete", 5), ("hierarchical2", 40)]


def _hold(n, nf, seed):
    """Random held parameters in a third of the frames."""
    rng = np.random.default_rng(seed)
    hold = np.zeros(n * nf, bool)
    for f in rng.choice(n, max(1, n // 3), replace=False):
        hold[f * nf + rng.choice(nf, rng.integers(1, nf // 2 + 1), replace=False)] = True
    return hold


@pytest.mark.parametrize("graph,n", GRAPHS)
def test_recurrence_matches_dense_inverse(graph, n):
    nf = 16
    pairs = R.GRAPHS[graph](n)
    # the restatement runs in the solver's elimination order and levels
    plan = solver.factor_plan(abi.default_config(n, 1.5, depth_type=abi.DEPTH_IDENTITY), np.array(pairs, np.int32).reshape(-1, 2))
    order, cs = R.elimination_order(n, pairs)
    lvl = R.levels(order, cs)
    assert list(plan["order"]) == order and [lvl[f] for f in range(n)] == list(plan["level"])
    H, _, _, _ = R.well_conditioned(n, nf, pairs, seed=n)
    hold = _hold(n, nf, seed=n)
    cov, products = CR.covariance(H, n, nf, pairs, hold)
    ref = CR.reduced_inverse(H, hold)
    assert products == sum(len(cs[k]) ** 2 + len(cs[k]) for k in range(n))
    fill = {(r, k) for k in range(n) for r in cs[k]}
    assert set(cov) == fill | {(k, k) for k in range(n)}
    scale = np.abs(ref).max()
    for (r, c), B in cov.items():
        E = ref[r * nf:(r + 1) * nf, c * nf:(c + 1) * nf]
        assert np.abs(B - E).max() <= 1e-12 * scale, (r, c)
        held_r, held_c = hold[r * nf:(r + 1) * nf], hold[c * nf:(c + 1) * nf]
        assert np.all(B[held_r] == 0) and np.all(B[:, held_c] == 0)


def test_gauge_direction_trips_the_pivot_test():
    n, nf = 6, 16
    pairs = R.chain(n)
    H = R.normal_matrix(n, nf, pairs, np.random.default_rng(3), gauge=True)
    order, _ = R.elimination_order(n, pairs)
    none = np.zeros(n * nf, bool)
    _, A = CR.scaled(H, none)
    hit = CR.first_failing_pivot(A, none, order, nf)
    assert hit is not None and abs(hit[2]) <= 1e-10
    # the gauge is column 0 of every frame together: holding one of them restores full rank
    hold = none.copy(); hold[0] = True
    _, A = CR.scaled(H, hold)
    assert CR.first_failing_pivot(A, hold, order, nf) is None


# the cases the default min_pivot was measured on: the default (Global) configuration and the first four variants at 8 frames, and
# the bilinear 4 x 4 grid at 40 frames
PREMISE = [("default", 8, {})] + [(name, 8, ov) for name, ov in helpers.VARIANTS[:4]] + [("bilinear_perframe_disp", 40, helpers.VARIANTS[0][1])]


@pytest.mark.parametrize("name,n,overrides", PREMISE, ids=[f"{c[0]}-{c[1]}" for c in PREMISE])
def test_min_pivot_premise(name, n, overrides):
    from oracle import oracle
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=n, **overrides)
    off_d, nd = helpers.layout_numbers(cfg)
    stride = solver.frame_stride(cfg)
    O = oracle.OracleProblem(cfg)
    helpers.setup_problem(O, cfg, pairs, offs, rec, med, helpers.initial_state(sc, cfg, stride, off_d, nd))
    O.solve(abi.default_solve_options(max_iterations=100))
    H = O.normal_matrix_dense()
    free = O.active_mask()
    order = list(range(n))               # the premise is about the matrix; any frame order shows the same null space
    _, A = CR.scaled(H, ~free)
    ev = np.linalg.eigvalsh(A[np.ix_(free, free)])
    assert int((ev < 1e-10 * ev.max()).sum()) == 6, ev[:8]
    assert CR.first_failing_pivot(A, ~free, order, stride) is not None
    hold = ~free
    hold[:6] = True                      # frame 0's position and rotation
    _, A = CR.scaled(H, hold)
    d = CR.pivots(A, order, stride)
    print(f"PREMISE {name} n={n}: smallest eigenvalue {ev[6]:.2e} (null {ev[5]:.1e}), smallest held pivot {d[~hold].min():.2e}")
    assert d[~hold].min() >= 1e-5
