"""tests/linalg_ref.py on its own (no GPU): LAPACK and the defect-free block Cholesky meet the thresholds of tests/test_gpu_linalg.py on
every generator mode, and every injected kernel defect misses them by at least 100x -- the evidence that the GPU tests can tell a
correct factorisation from a subtly wrong one."""
import numpy as np
import pytest
import scipy.linalg

from tests import linalg_ref as R

NF = 24          # neff = 24 = 8 (mod 16): the half last K stage exists
MODES = [("well", None), ("lm", 1e4), ("lm", 1e9), ("lm", 1e12)]


def _system(mode, radius, n, pairs, seed=0):
    if mode == "well":
        A, D2, b, x = R.well_conditioned(n, NF, pairs, seed)
        return A + np.diag(D2), b, x
    H, D2, b = R.lm_like(n, NF, pairs, radius, seed)
    return H + np.diag(D2), b, None


@pytest.mark.parametrize("graph", ["chain", "star", "complete", "disconnected"])
@pytest.mark.parametrize("mode,radius", MODES, ids=[f"{m}{'' if r is None else f'-{r:g}'}" for m, r in MODES])
def test_lapack_and_block_cholesky_meet_the_thresholds(graph, mode, radius):
    n = 7
    pairs = R.GRAPHS[graph](n)
    A, b, x = _system(mode, radius, n, pairs)
    order, cs = R.elimination_order(n, pairs)
    M, idx = R.permute(A, order, NF)
    lvl = R.levels(order, cs)
    for L in (np.linalg.cholesky(M), R.block_cholesky(A, n, NF, pairs)[1]):
        err, where = R.factor_error(L, M, NF, order, lvl)
        assert err <= R.FACTOR_TOL, (err, where)
        yp = scipy.linalg.cho_solve((L, True), b[idx])
        y = np.empty_like(yp); y[idx] = yp
        assert R.solve_error(A, y, b) <= R.SOLVE_TOL
        if x is not None:
            assert R.forward_error(y, x) <= R.FORWARD_TOL
        for q in range(n):
            Lkk = L[q * NF:(q + 1) * NF, q * NF:(q + 1) * NF]
            X = scipy.linalg.solve_triangular(Lkk, np.eye(NF), lower=True)
            assert R.linv_error(X, Lkk) <= R.LINV_TOL_PER_NF * NF


def test_block_cholesky_follows_the_elimination_order():
    pairs = R.hierarchical2(40)
    A, D2, b, x = R.well_conditioned(40, 8, pairs, seed=2)
    order, L = R.block_cholesky(A, 40, 8, pairs)
    M, _ = R.permute(A, order, 8)
    np.testing.assert_allclose(L, np.linalg.cholesky(M), rtol=0, atol=1e-12 * np.abs(L).max())
    # fill stays inside the symbolic pattern: blocks outside it are exactly zero
    _, cs = R.elimination_order(40, pairs)
    pos = {k: q for q, k in enumerate(order)}
    pattern = {(pos[r], pos[k]) for k in range(40) for r in cs[k]} | {(q, q) for q in range(40)}
    for bi in range(40):
        for bj in range(bi + 1):
            if (bi, bj) not in pattern:
                assert not L[bi * 8:(bi + 1) * 8, bj * 8:(bj + 1) * 8].any()


@pytest.mark.parametrize("defect", R.DEFECTS)
@pytest.mark.parametrize("mode,radius", MODES, ids=[f"{m}{'' if r is None else f'-{r:g}'}" for m, r in MODES])
def test_every_injected_defect_fails_by_100x(defect, mode, radius):
    n = 7
    pairs = R.complete(n)          # every frame couples to every later one: U2 targets, diagonal and off-diagonal targets
    A, b, x = _system(mode, radius, n, pairs, seed=1)
    order, cs = R.elimination_order(n, pairs)
    M, _ = R.permute(A, order, NF)
    Lgood, Lbad = R.block_cholesky(A, n, NF, pairs)[1], R.block_cholesky(A, n, NF, pairs, defect=defect)[1]
    for tile in (None, 16):          # the plain metric and the one loosened for explicit 16x16 tile inverses (GPU tests)
        good = R.factor_error(Lgood, M, NF, inverse_tile=tile)[0]
        bad, where = R.factor_error(Lbad, M, NF, order, R.levels(order, cs), inverse_tile=tile)
        assert good <= R.FACTOR_TOL
        assert bad >= 100 * R.FACTOR_TOL, (defect, tile, bad, where)


def test_negated_pivot_changes_only_that_pivot():
    n = 5
    pairs = R.chain(n)
    A, D2, b, x = R.well_conditioned(n, NF, pairs)
    order, _ = R.elimination_order(n, pairs)
    for j in (0, 1, 2, 3, NF + 5, n * NF - 1):
        An = R.negate_pivot(A, order, NF, j)
        M, _ = R.permute(An, order, NF)
        with pytest.raises(np.linalg.LinAlgError):
            np.linalg.cholesky(M)
        if j > 0:          # the leading j x j block is untouched and still positive definite
            np.linalg.cholesky(M[:j, :j])
        # the Schur complement at j is -0.5 d_j
        Mg, _ = R.permute(A, order, NF)
        Lg = np.linalg.cholesky(Mg)
        s = M[j, j] - Lg[j, :j] @ Lg[j, :j]
        assert s == pytest.approx(-0.5 * Lg[j, j] ** 2, rel=1e-9)


def test_metrics_are_exact_on_exact_data():
    L = np.tril(np.arange(1.0, 17.0).reshape(4, 4)) + 4 * np.eye(4)
    assert R.factor_error(L, L @ L.T, 4)[0] == 0.0
    A = L @ L.T; y = np.array([1.0, -2.0, 0.5, 3.0]); b = A @ y
    assert R.solve_error(A, y, b) == 0.0
    assert R.linv_error(np.linalg.inv(np.diag(np.diag(L))), np.diag(np.diag(L))) == 0.0
