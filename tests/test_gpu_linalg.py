"""Kernel-level tests of the block-sparse Cholesky: a matrix of known structure goes through the production factorisation graph
(rcvd_debug_solve_matrix), the factor comes back (rcvd_debug_factor_dense) and is checked against tests/linalg_ref.py at every block size
and launch shape the kernels branch on.  Every case also asserts, through the launch counters (rcvd_debug_linear_paths), that the kernel
path it targets really ran.  Run on an H100 with `pytest -m gpu`."""
import numpy as np
import pytest

from robust_cvd_b200 import abi
from tests import linalg_ref as R

pytestmark = pytest.mark.gpu


def _config(nf, n):
    """A problem configuration whose per-frame stride is nf: 7 + depth parameters + 2 x spatial parameters."""
    spatial = [(0, {}), (2, dict(spatial_type=abi.SPATIAL_VERTICAL_LINEAR)), (4, dict(spatial_type=abi.SPATIAL_CORNERS_BILINEAR))]
    for S, sp in spatial:
        d = nf - 7 - 2 * S
        if d == 0:
            return abi.default_config(n, 1.5, depth_type=abi.DEPTH_IDENTITY, **sp)
        if d == 1:
            return abi.default_config(n, 1.5, depth_type=abi.DEPTH_GLOBAL, **sp)
        for gx in range(2, d // 2 + 1):
            if d % gx == 0 and d // gx >= 2:
                return abi.default_config(n, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=gx, depth_grid_y=d // gx, **sp)
    raise ValueError(nf)


def _problem(nf, n, pairs):
    from robust_cvd_b200 import solver
    P = solver.Problem(_config(nf, n))
    assert P.stride == nf
    pf = np.array(pairs, np.int32).reshape(-1, 2)
    P.set_constraints(pf, np.zeros(len(pf) + 1, np.int64), np.zeros((0, 6), np.float32))      # the frame graph; no records
    return P


def _check(P, n, nf, pairs, H, D2, b, x=None, tag="", slack=4):
    """Factor + solve on the GPU, then every metric of linalg_ref against its threshold.  Returns (y, L).
    The factor bound is the componentwise one with the TRSM's explicit tile inverses accounted for (linalg_ref.tile_inverse_bound);
    the plain componentwise value is reported beside it."""
    A = H + np.diag(D2)
    y = P.solve_matrix(H, D2, b)
    order, L, Linv = P.factor_dense(inverses=True)
    ref_order, cs = R.elimination_order(n, pairs, slack=slack)
    assert list(order) == ref_order                      # linalg_ref models the solver's elimination order and levels
    lvl = R.levels(ref_order, cs)
    M, _ = R.permute(A, order, nf)
    npad = (nf + 15) // 16 * 16
    fe, where = R.factor_error(L, M, nf, ref_order, lvl, inverse_tile=R.trsm_inverse_tile(npad, nf))
    fp, where_p = R.factor_error(L, M, nf, ref_order, lvl)
    se = R.solve_error(A, y, b)
    le = max(R.linv_error(Linv[q], L[q * nf:(q + 1) * nf, q * nf:(q + 1) * nf]) for q in range(n))
    fw = R.forward_error(y, x) if x is not None else float("nan")
    print(f"LINALG {tag} nf={nf} npad={npad} U={n * nf} factor={fe:.2f}u at {where} plain={fp:.2f}u at {where_p} solve={se:.3f}u "
          f"linv={le:.1f}u fwd={fw:.2e} paths={ {k: v for k, v in P.linear_paths().items() if v} }")
    assert fe <= R.FACTOR_TOL, (fe, where)
    assert se <= R.SOLVE_TOL, se
    assert le <= R.LINV_TOL_PER_NF * nf, le
    if x is not None:
        assert fw <= R.FORWARD_TOL, fw
    return y, L


def _well(P, n, nf, pairs, seed=0, tag="", slack=4):
    A, D2, b, x = R.well_conditioned(n, nf, pairs, seed)
    return _check(P, n, nf, pairs, A, D2, b, x, tag, slack)


def _assert_potrf_path(P, npad):
    p = P.linear_paths()
    if npad <= 224:
        assert p["potrf_smem"] > 0 and p["potrf_panel"] == 0
    else:
        assert p["potrf_panel"] > 0 and p["potrf_smem"] == 0


# ---------------------------------------------------------------------------------------------------------
# block size: every tile count of the shared-memory potrf, then across the panel / TRSM path boundaries
# ---------------------------------------------------------------------------------------------------------
NPADS = [16 * k for k in range(1, 15)] + [240, 256, 272, 288, 416, 432, 864]


@pytest.mark.parametrize("trim", [0, 9], ids=["nf=npad", "nf=npad-9"])
@pytest.mark.parametrize("npad", NPADS)
def test_npad_sweep(npad, trim):
    nf, n = npad - trim, 4
    pairs = R.complete(n)
    P = _problem(nf, n, pairs)
    _well(P, n, nf, pairs, seed=npad + trim, tag=f"npad-sweep")
    p = P.linear_paths()
    assert P.structure_info()["npad"] == npad
    _assert_potrf_path(P, npad)
    if npad <= 272:
        assert p["trsm_ll4"] > 0 and p["trsm_gemm"] == 0       # K_4: at most 3 x npad/32 strips per level, one wave
    elif npad <= 416:
        assert p["trsm_ll2"] > 0 and p["trsm_ll4"] == 0 and p["trsm_gemm"] == 0
    else:
        assert p["trsm_gemm"] > 0 and p["trsm_ll4"] == 0 and p["trsm_ll2"] == 0


def test_npad_880_is_refused():
    P = _problem(880, 2, R.chain(2))
    A, D2, b, x = R.well_conditioned(2, 880, R.chain(2))
    with pytest.raises(RuntimeError, match="too large"):
        P.solve_matrix(A, D2, b)


def test_entry_outside_the_frame_graph_is_refused():
    nf, n = 16, 4
    P = _problem(nf, n, R.chain(n))
    A, D2, b, x = R.well_conditioned(n, nf, R.chain(n))
    A[0, 3 * nf + 2] = A[3 * nf + 2, 0] = 1e-3            # frames 0 and 3 are not coupled
    with pytest.raises(RuntimeError, match="frames 0 and 3"):
        P.solve_matrix(A, D2, b)
    with pytest.raises(RuntimeError, match="no factorisation"):
        P.factor_dense()


# ---------------------------------------------------------------------------------------------------------
# update kernel shapes: neff 40, 104, 136 reach all 19 reachable warp tiles of k_update_tma; 48 = 0 (mod 16) has no half K stage
# ---------------------------------------------------------------------------------------------------------
UPDATE_NF = {40: 37, 104: 104, 136: 133, 48: 48}


UPDATE_CASES = [("chain", "tma"), ("complete", "tma"), ("complete", "items_per_cta_1")]


@pytest.mark.parametrize("graph,variant", UPDATE_CASES, ids=[f"{g}-{v}" for g, v in UPDATE_CASES])
@pytest.mark.parametrize("neff", sorted(UPDATE_NF))
def test_update_shapes(neff, graph, variant):
    """A chain has a few update items per level (k_update_tma<2>).  A complete graph puts every pair of the remaining frames into level
    0's side-stream launch: K_25 at one 80-row tile per block (neff <= 80) has 276 items, K_14 at 2 x 2 tiles 300, more than the
    2 x 132 CTAs of a k_update_tma<1> launch on an H100, so CTAs walk several items; capping at one item per CTA widens the grid
    instead."""
    nf = UPDATE_NF[neff]
    n = 6 if graph == "chain" else (14 if neff > 80 else 25)
    pairs = R.GRAPHS[graph](n)
    P = _problem(nf, n, pairs)
    with pytest.raises(RuntimeError, match="cp.async update path was removed"):
        P.set_update_kernel(False)
    if variant == "items_per_cta_1":
        P.set_update_kernel(True, 1)
    _well(P, n, nf, pairs, seed=neff, tag=f"update-{graph}-{variant}")
    p = P.linear_paths()
    if graph == "chain":
        assert p["update_tma2"] > 0 and p["update_tma1"] == 0
    elif variant == "tma":
        assert p["update_tma1_multi_item"] > 0
    else:
        assert p["update_tma1"] > 0 and p["update_tma1_multi_item"] == 0


# ---------------------------------------------------------------------------------------------------------
# graph shapes: the 300-frame hierarchical schedule (wide levels: level-launched substitution, then k_substitution), other
# elimination orders and the single-stream graph
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["default", "slack-1", "slack0", "no_overlap"])
@pytest.mark.parametrize("nf", [16, 23], ids=["npad16", "npad32"])
def test_hierarchical_graph(nf, variant):
    n = 300
    pairs = R.hierarchical2(n)
    P = _problem(nf, n, pairs)
    if variant.startswith("slack"):
        P.set_order_slack(int(variant[5:]))
    elif variant == "no_overlap":
        P.set_overlap(False)
    _well(P, n, nf, pairs, seed=nf, tag=f"hierarchical2-{variant}", slack=int(variant[5:]) if variant.startswith("slack") else 4)
    p = P.linear_paths()
    # at npad <= 64 every level has at most 4 substitution tasks per SM: all of them run in k_substitution
    assert p["substitution_fused"] > 0 and p["update_tma1"] > 0 and p["update_tma2"] > 0


@pytest.mark.parametrize("nf", [16, 23], ids=["npad16", "npad32"])
def test_wide_level_substitution_launches(nf):
    """A 300-frame star: level 0 has 299 frames and 299 forward tasks (more than 4 per SM), so it is substituted by level launches
    (k_fwd_* / k_bwd_*, partial 64-row chunk at npad 16 and 32) and the hub's level by k_substitution."""
    n = 300
    pairs = R.star(n)
    P = _problem(nf, n, pairs)
    _well(P, n, nf, pairs, seed=nf, tag="star300")
    p = P.linear_paths()
    assert p["substitution_levels"] > 0 and p["substitution_fused"] > 0


# ---------------------------------------------------------------------------------------------------------
# conditioning: the three generator modes on a shared-memory and a panel block size
# ---------------------------------------------------------------------------------------------------------
MODES = [("well", None), ("lm", 1e4), ("lm", 1e9), ("lm", 1e12)]


@pytest.mark.parametrize("mode,radius", MODES, ids=[f"{m}{'' if r is None else f'-{r:g}'}" for m, r in MODES])
@pytest.mark.parametrize("nf,graph,n", [(45, "disconnected", 8), (256, "star", 4)], ids=["npad48", "npad256"])
def test_conditioning(nf, graph, n, mode, radius):
    pairs = R.GRAPHS[graph](n)
    P = _problem(nf, n, pairs)
    if mode == "well":
        _well(P, n, nf, pairs, seed=7, tag=f"cond-{graph}-well")
    else:
        H, D2, b = R.lm_like(n, nf, pairs, radius, seed=7)
        _check(P, n, nf, pairs, H, D2, b, tag=f"cond-{graph}-lm-{radius:g}")
    _assert_potrf_path(P, (nf + 15) // 16 * 16)
    assert P.linear_paths()["trsm_ll4"] > 0


# ---------------------------------------------------------------------------------------------------------
# non-positive pivots: positions 0..3 (mod 4) of the 4x4-blocked pivot tile (a00, det01, b22, det23 in warp_chol16_blocked) and of
# k_potrf_panel, in the first, a middle and the last 16-tile of a level-0 frame and of the last-eliminated frame
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["level0", "last"])
@pytest.mark.parametrize("nf", [48, 256], ids=["smem", "panel"])
def test_pivot_failure_is_flagged(nf, which):
    n = 3
    pairs = R.chain(n)
    P = _problem(nf, n, pairs)
    A, D2, b, x = R.well_conditioned(n, nf, pairs, seed=3)
    _check(P, n, nf, pairs, A, D2, b, x, tag="pivot-before")
    order = list(P.factor_dense()[0])
    q = 0 if which == "level0" else n - 1
    nt = nf // 16
    for tile in sorted({0, nt // 2, nt - 1}):
        for p in range(4):
            j = q * nf + tile * 16 + p
            with pytest.raises(RuntimeError, match="non-positive pivot"):
                P.solve_matrix(R.negate_pivot(A, order, nf, j), D2, b)
    # the same handle still factors a valid matrix correctly
    A2, D22, b2, x2 = R.well_conditioned(n, nf, pairs, seed=4)
    _check(P, n, nf, pairs, A2, D22, b2, x2, tag="pivot-after")
    _assert_potrf_path(P, nf)


# ---------------------------------------------------------------------------------------------------------
# reuse and determinism: each target's update order is fixed and U2(l) is joined before U1(l+1), so the factor is bitwise
# reproducible across repeats, the single-stream graph and the un-captured profiling run
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nf,n", [(48, 18), (256, 4)], ids=["npad48-K18", "npad256-K4"])
def test_reuse_and_determinism(nf, n):
    pairs = R.complete(n)
    P = _problem(nf, n, pairs)
    _well(P, n, nf, pairs, seed=1, tag="reuse-1")
    A, D2, b, x = R.well_conditioned(n, nf, pairs, seed=2)
    y, L = _check(P, n, nf, pairs, A, D2, b, x, tag="reuse-2")
    y2 = P.solve_matrix(A, D2, b)
    assert np.array_equal(P.factor_dense()[1], L), "repeated factorisation differs"
    np.testing.assert_allclose(y2, y, rtol=0, atol=64 * R.U_ROUND * np.abs(y).max())      # the substitution sums with red_add
    P.set_overlap(False)
    P.solve_matrix(A, D2, b)
    assert np.array_equal(P.factor_dense()[1], L), "single-stream graph differs"
    P.set_overlap(True)
    P.profile_linear(reps=1)
    assert np.array_equal(P.factor_dense()[1], L), "un-captured profiling run differs"
    _assert_potrf_path(P, nf)
    p = P.linear_paths()
    assert p["update_tma1"] > 0 if n > 4 else (p["update_tma2"] > 0 and p["update_tma1"] == 0)      # K_18: 136 items in level 0's U2
