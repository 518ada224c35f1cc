"""The streamed TRSM: a k_trsm_ll launch that fits in one wave starts as a programmatic dependent of its level's k_potrf_smem and
reads each row panel of L_kk as soon as the Cholesky publishes it.  A panel read before its publication would carry the pre-factor
block into X and miss the factor bound by orders of magnitude, and would make the factor depend on timing.  Run on an H100 with
`pytest -m gpu`."""
import numpy as np
import pytest

from tests import linalg_ref as R
from tests.test_gpu_linalg import _check, _problem

pytestmark = pytest.mark.gpu


N_K5 = 5
PAIRS = [pr for c in range(N_K5) for pr in R.complete_range(5 * c, 5 * c + 5)]


def test_streamed_trsm_at_npad208():
    """Five disjoint K_5 at npad 208 (7 strips of 32 rows per TRSM task).  Level 0 factors five frames at once, each with four TRSM
    tasks: 140 CTAs, more than an H100's 132 SMs, so k_trsm_ll<2> at two CTAs per SM.  Level 1: 15 tasks, 105 CTAs, k_trsm_ll<4>.
    Both launches are a single wave and run streamed."""
    nf, n, pairs = 208, 5 * N_K5, PAIRS
    order, cs = R.elimination_order(n, pairs)
    lvl = R.levels(order, cs)
    level0 = [k for k in order if lvl[k] == 0]
    assert len(level0) == N_K5 and all(len(cs[k]) == 4 for k in level0)
    P = _problem(nf, n, pairs)
    A, D2, b, x = R.well_conditioned(n, nf, pairs, seed=11)
    y, L = _check(P, n, nf, pairs, A, D2, b, x, tag="trsm-stream")
    p = P.linear_paths()
    assert p["potrf_smem"] > 0 and p["trsm_ll4"] > 0 and p["trsm_ll2"] > 0
    assert p["trsm_ll_streamed"] == p["trsm_ll4"] + p["trsm_ll2"]      # every TRSM launch of this graph is a single wave
    assert P.structure_info()["npad"] == 208
    # the factor is bitwise the same whatever overlapped: a graph replay, the single-stream graph (the TRSM follows k_trinv there) and
    # the un-captured profiling run
    P.solve_matrix(A, D2, b)
    assert np.array_equal(P.factor_dense()[1], L), "repeated factorisation differs"
    P.set_overlap(False)
    P.solve_matrix(A, D2, b)
    assert np.array_equal(P.factor_dense()[1], L), "single-stream graph differs"
    P.set_overlap(True)
    P.profile_linear(reps=1)
    assert np.array_equal(P.factor_dense()[1], L), "un-captured profiling run differs"


def test_streamed_trsm_after_pivot_failure():
    """A non-positive pivot still runs every step of k_potrf_smem, so every progress counter is complete and the streamed TRSM
    finishes; the error is reported and the handle then factors a valid matrix."""
    nf, n, pairs = 208, 5 * N_K5, PAIRS
    P = _problem(nf, n, pairs)
    A, D2, b, x = R.well_conditioned(n, nf, pairs, seed=12)
    _check(P, n, nf, pairs, A, D2, b, x, tag="trsm-stream-pivot-before")
    order = list(P.factor_dense()[0])
    for j in (5, nf + 7 * 16 + 2):                       # first tile of the first frame, a middle tile of the second (both level 0)
        with pytest.raises(RuntimeError, match="non-positive pivot"):
            P.solve_matrix(R.negate_pivot(A, order, nf, j), D2, b)
    A2, D22, b2, x2 = R.well_conditioned(n, nf, pairs, seed=13)
    _check(P, n, nf, pairs, A2, D22, b2, x2, tag="trsm-stream-pivot-after")
    assert P.linear_paths()["trsm_ll_streamed"] > 0
