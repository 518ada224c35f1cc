"""The conjugate-gradient linear solver without a GPU: the numpy restatement (tests/cg_ref.py) against dense solves and an independent
evaluation of its quadratic-model test, and the solver choice (rcvd_debug_linear_storage) against the block counts of
tests/linalg_ref.py at the benchmark sizes."""
import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import cg_ref
from tests import linalg_ref as R

# cudaDeviceProp::totalGlobalMem of an H100 80GB HBM3 (SXM; nvidia-smi reports 81559 MiB)
H100_80GB_TOTAL = 85017493504

GRAPH_CASES = [("chain", 8, 12), ("complete", 5, 9), ("disconnected", 9, 7), ("hierarchical2", 40, 6)]


@pytest.mark.parametrize("graph,n,nf", GRAPH_CASES, ids=[c[0] for c in GRAPH_CASES])
def test_pcg_converges_to_the_dense_solution(graph, n, nf):
    """eta -> 0.  The quadratic-model test sees the error through Q(x) - Q(x*) = |x - x*|_A^2, and Q itself is only known to ~1e-16
    relative: the decrease of Q drops into its rounding at a relative error of ~1e-8 in x, where the test stops any eta <= 1e-14 (the
    ratio turns negative or zero).  So the restatement reaches the dense solution to ~1e-8 (observed 1e-9 .. 1.4e-8)."""
    pairs = R.GRAPHS[graph](n)
    A, _, b, _ = R.well_conditioned(n, nf, pairs, seed=n)
    out = cg_ref.pcg(A, b, nf, eta=1e-14)
    x = np.linalg.solve(A, b)
    assert not out["broke"] and not out["capped"]
    assert np.linalg.norm(out["x"] - x) <= 1e-7 * np.linalg.norm(x), np.linalg.norm(out["x"] - x) / np.linalg.norm(x)
    assert out["iterations"] < 4 * n * nf


def _plain_pcg_iterates(A, b, nf, k):
    """x_1 .. x_k of textbook PCG with the frames' diagonal blocks as preconditioner (explicit inverses, recursive residual)."""
    n = A.shape[0] // nf
    Minv = np.zeros_like(A)
    for f in range(n):
        s = slice(f * nf, (f + 1) * nf)
        Minv[s, s] = np.linalg.inv(A[s, s])
    x, r = np.zeros_like(b), b.copy()
    z = Minv @ r; p = z.copy(); rz = r @ z; xs = []
    for _ in range(k):
        q = A @ p; alpha = rz / (p @ q)
        x = x + alpha * p; r = r - alpha * q
        xs.append(x.copy())
        z = Minv @ r; rz2 = r @ z; p = z + rz2 / rz * p; rz = rz2
    return xs


@pytest.mark.parametrize("graph,n,nf", GRAPH_CASES, ids=[c[0] for c in GRAPH_CASES])
@pytest.mark.parametrize("eta", [0.1, 1e-3])
def test_iteration_count_follows_the_quadratic_model(graph, n, nf, eta):
    """The iterates equal textbook PCG's, and the solve stops at the first iteration i with i (Q_i - Q_i-1) / Q_i < eta, Q evaluated
    from the iterates directly (Q(x) = x'Ax - 2b'x)."""
    pairs = R.GRAPHS[graph](n)
    A, b = cg_ref.spd_system(n, nf, pairs, cond_spread=6, seed=3 * n)
    out = cg_ref.pcg(A, b, nf, eta=eta)
    assert not out["broke"] and not out["capped"] and out["iterations"] >= 2
    xs = _plain_pcg_iterates(A, b, nf, out["iterations"])
    np.testing.assert_allclose(out["x"], xs[-1], rtol=0, atol=1e-9 * np.abs(xs[-1]).max())
    Q = [0.0] + [x @ A @ x - 2 * b @ x for x in xs]
    zeta = [i * (Q[i] - Q[i - 1]) / Q[i] for i in range(1, len(Q))]
    np.testing.assert_allclose(out["zeta"], zeta, rtol=1e-6, atol=1e-12)
    stop = next(i for i, z in enumerate(zeta, 1) if z < eta)
    assert out["iterations"] == stop


def test_iteration_cap_zero_rhs_and_breakdown():
    A, b = cg_ref.spd_system(6, 5, R.complete(6), cond_spread=8, seed=1)
    capped = cg_ref.pcg(A, b, 5, eta=1e-30, max_iterations=3)
    assert capped["capped"] and capped["iterations"] == 3 and not capped["broke"]
    assert np.array_equal(capped["x"], cg_ref.pcg(A, b, 5, eta=1e-30, max_iterations=3)["x"])
    zero = cg_ref.pcg(A, np.zeros_like(b), 5)
    assert zero["iterations"] == 0 and not np.any(zero["x"])
    # an indefinite matrix with positive 1 x 1 diagonal blocks: p'q = -12 at iteration 2
    broke = cg_ref.pcg(np.array([[1.0, 2.0], [2.0, 1.0]]), np.array([1.0, 0.0]), 1)
    assert broke["broke"] and broke["iterations"] == 2


def _config(n, gx, gy):
    return abi.default_config(n, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=gx, depth_grid_y=gy)


def _reference_storage(n, pairs, npad):
    """Both solvers' bytes from linalg_ref's elimination: H = N + coupled pairs blocks, N + fill + off-diagonal factor blocks, T, the
    diagonal inverses and tile inverses; CG: H, 2 N blocks, tile inverses, 2 slots per H block, 4 vectors, partials, slot lists, state."""
    order, cs = R.elimination_order(n, pairs, 4)
    nL = sum(len(cs[k]) for k in order)
    nH = n + len({(min(a, b), max(a, b)) for a, b in pairs if a != b})
    bs, tiles = 8 * npad * npad, 8 * n * npad * 16
    chol = bs * (nH + n + nL + max(nL, 1) + n) + tiles
    cg = bs * (nH + 2 * n) + tiles + 8 * (2 * nH * npad + 4 * n * npad + max(n, 264)) + 4 * (n + 1 + 2 * nH + n) + 56
    return chol, cg


SIZES = [(300, 16, 12, 208, abi.LINEAR_CHOLESKY), (600, 32, 24, 784, abi.LINEAR_CHOLESKY), (1000, 32, 24, 784, abi.LINEAR_CG)]


@pytest.mark.parametrize("n,gx,gy,npad,expect", SIZES, ids=["config2", "config4", "1000f_grid32x24"])
def test_solver_choice_at_benchmark_sizes(n, gx, gy, npad, expect):
    """Config 2 and config 4 (600 frames) keep the block Cholesky on an 80 GB H100; 1000 frames at a 32 x 24 grid (the factor alone
    ~107 GB) take conjugate gradients."""
    pairs = R.hierarchical2(n)
    got = solver.linear_storage(_config(n, gx, gy), pairs, device_total_bytes=H100_80GB_TOTAL)
    chol, cg = _reference_storage(n, pairs, npad)
    assert (got["cholesky_bytes"], got["cg_bytes"]) == (chol, cg)
    assert got["solver"] == expect
    print(f"STORAGE {n} frames grid {gx}x{gy}: cholesky {chol / 1e9:.1f} GB, cg {cg / 1e9:.1f} GB")


def test_zero_budget_device_selects_cg():
    pairs = R.chain(4)
    got = solver.linear_storage(_config(4, 4, 4), pairs, device_total_bytes=0)
    assert got["solver"] == abi.LINEAR_CG and got["cg_bytes"] < got["cholesky_bytes"]
