"""rcvd_covariance on the H100 (restated ceres::Covariance semantics): the selected inversion of the block-Cholesky factor
(robust_cvd_b200/csrc/rcvd_selinv.cuh) against dense inverses -- kernel by kernel at every block size the factorisation branches on,
and on whole problems at their LM solution -- and the call's refusals, rank test and freedom from side effects.  Run with `pytest -m gpu`."""
import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import covariance_ref as CR
from tests import helpers
from tests import linalg_ref as R
from tests.test_gpu_linalg import _problem

pytestmark = pytest.mark.gpu
U_ROUND = 2.0 ** -53
C_NORMWISE = 64.0           # normwise bound |Cov - inv| / |inv| <= C_NORMWISE * nf * kappa * u on every block


def _h_pairs(n, pairs):
    """Every diagonal block and both orientations of every coupled pair."""
    out = [(f, f) for f in range(n)]
    for a, b in pairs:
        out += [(a, b), (b, a)]
    return np.array(out, np.int32)


def _check_blocks(cov, ref, blocks, nf, bound, tag):
    worst = 0.0
    scale = np.abs(ref).max()
    for q, (a, b) in enumerate(blocks):
        E = ref[a * nf:(a + 1) * nf, b * nf:(b + 1) * nf]
        worst = max(worst, np.abs(cov[q] - E).max() / scale)
    print(f"COV {tag}: normwise error {worst:.2e} (bound {bound:.2e})")
    assert worst <= bound, (worst, bound)


def _kernel_case(nf, n, pairs, seed):
    P = _problem(nf, n, pairs)
    H, _, _, _ = R.well_conditioned(n, nf, pairs, seed=seed)
    rng = np.random.default_rng(seed)
    hold = np.zeros(n * nf, bool)
    for f in rng.choice(n, max(1, n // 3), replace=False):
        hold[f * nf + rng.choice(nf, rng.integers(1, max(2, nf // 4)), replace=False)] = True
    blocks = _h_pairs(n, pairs)
    cov = P.covariance_matrix(H, blocks, hold)
    ref = CR.reduced_inverse(H, hold)
    S, A = CR.scaled(H, hold)
    kappa = np.linalg.cond(A[np.ix_(~hold, ~hold)])
    _check_blocks(cov, ref, blocks, nf, C_NORMWISE * nf * kappa * U_ROUND, f"nf={nf} n={n}")
    for q, (a, b) in enumerate(blocks):
        assert np.all(cov[q][hold[a * nf:(a + 1) * nf]] == 0) and np.all(cov[q][:, hold[b * nf:(b + 1) * nf]] == 0)
    assert np.array_equal(P.covariance_matrix(H, blocks, hold), cov)          # same matrix: bitwise the same blocks
    launches = P.covariance_launches()
    assert launches["product"] > 0 and launches["trmm"] > 0 and launches["gather"] > 0 and launches["pivots"] > 0
    return P


# both k_potrf paths (smem up to npad 224, panel above) and the three TRSM paths (k_trsm_ll<4> to 272, <2> to 416, k_gemm_nt above)
@pytest.mark.parametrize("npad", [16, 32, 208, 224, 240, 416, 432, 784, 864])
def test_kernel_level_block_sizes(npad):
    n = 4
    P = _kernel_case(npad - 3, n, R.complete(n), seed=npad)
    assert P.structure_info()["npad"] == npad


@pytest.mark.parametrize("graph,n", [("chain", 7), ("star", 6), ("complete", 5), ("hierarchical2", 40)])
def test_kernel_level_graphs(graph, n):
    _kernel_case(24, n, R.GRAPHS[graph](n), seed=n)


def test_gauge_matrix_is_refused_through_the_hook():
    n, nf = 5, 16
    pairs = R.chain(n)
    P = _problem(nf, n, pairs)
    H = R.normal_matrix(n, nf, pairs, np.random.default_rng(3), gauge=True)
    with pytest.raises(RuntimeError, match=r"rcvd error 4: .*frame \d+, parameter \d+"):
        P.covariance_matrix(H, None, None)


# ---------------------------------------------------------------------------------------------------------
# problem level: at the LM solution, frame 0's pose held
# ---------------------------------------------------------------------------------------------------------
def _solved(name, overrides, extra=None, n=8):
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=n, **overrides)
    P = solver.Problem(cfg)
    off_d, nd = helpers.layout_numbers(cfg)
    helpers.setup_problem(P, cfg, pairs, offs, rec, med, helpers.initial_state(sc, cfg, P.stride, off_d, nd))
    if extra == "triplets":
        P.set_triplets(*sc.triplets(sep=14))
    elif extra == "depth_pairs":
        P.set_depth_pairs(pairs, offs, rec)
    P.solve(abi.default_solve_options(max_iterations=100))
    return P, pairs


CASES = [(name, ov, None) for name, ov in helpers.VARIANTS] + [
    ("triplets", helpers.VARIANTS[0][1], "triplets"), ("depth_pairs", helpers.VARIANTS[0][1], "depth_pairs"),
    ("fix_depth_xforms", dict(helpers.VARIANTS[0][1], fix_depth_xforms=1), None), ("fixed_intrinsics", dict(intr_opt=abi.INTR_FIXED), None)]


@pytest.mark.parametrize("name,overrides,extra", CASES, ids=[c[0] for c in CASES])
def test_problem_level(name, overrides, extra):
    P, pairs = _solved(name, overrides, extra)
    N, nf = P.N, P.stride
    H = P.normal_matrix_dense()
    hold = np.zeros(N * nf, bool); hold[:6] = True
    blocks = _h_pairs(N, {(min(a, b), max(a, b)) for a, b in np.asarray(pairs).reshape(-1, 2)})
    # the configuration's constant parameters and the parameters no residual touches have zero rows and columns of H
    zero = hold | (np.abs(H).sum(1) == 0)
    _, A = CR.scaled(H, zero)
    ev = np.linalg.eigvalsh(A[np.ix_(~zero, ~zero)])
    if ev[0] <= 1e-8 * ev[-1]:
        # The gauge of this variant is not frame 0's pose alone (fix_poses: the poses are constant, the depth scales are free;
        # the Euclidean loss measures world distances, so the scene scale is free too): the call must refuse, not invert.
        assert ev[0] <= 1e-12 * ev[-1], ("neither full rank nor a null direction", ev[:3])
        with pytest.raises(RuntimeError, match="rcvd error 4"):
            P.covariance(blocks, hold)
        return
    x0 = P.get_state().copy()
    cov = P.covariance(blocks, hold)
    ref = CR.reduced_inverse(H, zero)
    for q, (a, b) in enumerate(blocks):
        E = ref[a * nf:(a + 1) * nf, b * nf:(b + 1) * nf]
        err = np.abs(cov[q] - E).max() / max(np.abs(E).max(), 1e-300)
        assert err <= 1e-9, (name, a, b, err)
        zr, zc = zero[a * nf:(a + 1) * nf], zero[b * nf:(b + 1) * nf]
        assert np.all(cov[q][zr] == 0) and np.all(cov[q][:, zc] == 0)
    index = {(int(a), int(b)): q for q, (a, b) in enumerate(blocks)}
    for (a, b), q in index.items():
        assert np.array_equal(cov[q], cov[index[(b, a)]].T)
    # a second call re-evaluates H, whose accumulation order varies from run to run (atomics): equal within that spread; the
    # selected inversion itself is bitwise reproducible (test_kernel_level_*)
    again = P.covariance(blocks, hold)
    assert np.abs(again - cov).max() <= 1e-10 * np.abs(cov).max()
    assert np.array_equal(P.get_state(), x0)
    assert P.last_min_pivot > 1e-5


def test_rank_deficiency_is_refused_and_out_untouched():
    P, _ = _solved("default", {})
    out = np.full((P.N, P.stride, P.stride), 7.0)
    import ctypes as C
    rc = P.L.rcvd_covariance(P.h, None, C.c_double(1e-10), C.c_int32(P.N), solver._p(np.ascontiguousarray(np.repeat(np.arange(P.N, dtype=np.int32)[:, None], 2, 1)), C.c_int32),
                             solver._p(out, C.c_double), None)
    msg = P.L.rcvd_last_error().decode()
    assert rc == abi.ERR_NUMERIC and "frame" in msg and "parameter" in msg, msg
    assert np.all(out == 7.0)


def test_handle_state_and_next_solve_unchanged():
    opt = abi.default_solve_options(max_iterations=30)
    A, _ = _solved("default", {}, n=8)
    B, _ = _solved("default", {}, n=8)
    x, info = A.get_state().copy(), A.linear_info()
    hold = np.zeros(A.U, bool); hold[:6] = True
    A.covariance(None, hold)
    assert np.array_equal(A.get_state(), x) and A.linear_info() == info
    # perturb both identically, then solve: the handle that made the call must behave as the one that did not
    x1 = x + np.random.default_rng(1).normal(0, 0.01, x.shape)
    A.set_state(x1); B.set_state(x1)
    sa, sb = A.solve(opt), B.solve(opt)
    assert sa.termination == sb.termination and sa.iterations == sb.iterations
    assert sa.final_cost == pytest.approx(sb.final_cost, rel=1e-10)


def test_refusals_leave_the_handle_usable():
    P, pairs = _solved("default", {})
    N = P.N
    coupled = {(min(a, b), max(a, b)) for a, b in np.asarray(pairs).reshape(-1, 2)}
    far = next((a, b) for a in range(N) for b in range(a + 1, N) if (a, b) not in coupled)
    for blocks, match in [([far], "share no residual"), ([(0, N)], "out of range")]:
        with pytest.raises(RuntimeError, match=match):
            P.covariance(np.array(blocks), None)
    import ctypes as C
    assert P.L.rcvd_covariance(P.h, None, C.c_double(1e-10), C.c_int32(1), solver._p(np.zeros(2, np.int32), C.c_int32), None, None) == abi.ERR_INVALID
    P.set_factor_budget(0)
    with pytest.raises(RuntimeError, match="conjugate gradients"):
        P.covariance(None, None)
    assert P.covariance_launches()["product"] == 0
    s = P.solve(abi.default_solve_options(max_iterations=5))
    assert s.termination != abi.TERM_FAILURE


def test_config2_against_the_substitution_path():
    """Cov e_i through rcvd_debug_linear_solve (factorisation + substitution, not the selected inversion) at config 2."""
    import bench
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case("config2_300f_384x224_grid16x12_sep10")
    P = solver.Problem(cfg)
    helpers.setup_problem(P, cfg, pairs, offs, rec, med, bench.initial_state(sc, cfg, solver.frame_stride(cfg)))
    P.solve(abi.default_solve_options(max_iterations=5))
    N, nf = P.N, P.stride
    hold = np.zeros(N * nf, bool); hold[:6] = True
    coupled = sorted({(min(a, b), max(a, b)) for a, b in np.asarray(pairs).reshape(-1, 2)})
    blocks = _h_pairs(N, coupled)
    cov = P.covariance(blocks, hold)
    # H^-1 e = S (S H S + D2)^-1 S e on the free parameters for any positive S; zeroed parameters: S = 0, D2 = 1
    dH = _diag_of_h(P)
    zero = hold | (dH == 0)
    S = np.where(zero, 0.0, 1.0 / np.sqrt(np.where(dH > 0, dH, 1.0)))
    D2 = zero.astype(np.float64)
    rng = np.random.default_rng(0)
    worst = 0.0
    for col in [int(c) for c in rng.choice(np.nonzero(~zero)[0], 8, replace=False)]:
        e = np.zeros(N * nf); e[col] = S[col]
        v = S * P.debug_linear_solve(S, D2, e)          # S (S H S + D2)^-1 S e_col
        f, i = divmod(col, nf)
        for q, (a, b) in enumerate(blocks):
            if b == f:
                ref = v[a * nf:(a + 1) * nf]
                worst = max(worst, np.abs(cov[q][:, i] - ref).max() / np.abs(v).max())
    print(f"COV config2: column error {worst:.2e} of the column's largest entry")
    assert worst <= 1e-8


def _diag_of_h(P):
    """A positive scaling for the check (the dense normal matrix is too large at config 2): the squared Jacobian columns of every
    family, without the robust loss.  Zero exactly where H has a zero row: constant and untouched parameters."""
    d = np.zeros(P.U)
    for fam in abi.ROW_FAMILIES:
        if P.row_layout()[fam]["blocks"] == 0:
            continue
        r, rho, cols, J = P.rows(fam, jacobian=True)
        m = cols >= 0
        np.add.at(d, cols[m], J[m] ** 2)
    return d
