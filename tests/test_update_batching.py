"""The Schur-update passes of the block-Cholesky plan (robust_cvd_b200/csrc/rcvd_plan.h), read through rcvd_debug_update_passes and
checked against a numpy restatement: every block product in exactly one pass, the late pass of each target on the main stream, the
deferred passes grouped in level windows that do not cross the tail boundary and split into a level's two side launches, and a replay
of the stream and join order in which every two passes on one target, and every pass and its column's potrf / TRSM, are ordered.  The
GPU tests at the end (`pytest -m gpu`) factor graphs with multi-level passes against the dense reference."""
from collections import defaultdict

import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import linalg_ref as R


def _window(cfg):
    """rcvd_plan.h kUpdWindow / kUpdWindowMaxNf: below the tail, deferred passes group their source levels in aligned windows of 2
    levels when a frame block has at most 256 unknowns, else one pass per source level (always in the tail)."""
    return 2 if solver.frame_stride(cfg) <= 256 else 1


def _config(n, gx=4, gy=4):
    return abi.default_config(n, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=gx, depth_grid_y=gy)


def _tail(order, lvl):
    """First level of the trailing run of levels with fewer than 3 frames."""
    nl = max(lvl.values()) + 1
    sizes = [sum(1 for k in order if lvl[k] == l) for l in range(nl)]
    tb = nl
    while tb > 0 and sizes[tb - 1] < 3:
        tb -= 1
    return tb


def _expected_passes(n, pairs, nranks, rank, window_levels, slack=4):
    """{(r, c, apply level, stream, sorted source frames)} of one rank, restated from the elimination structure."""
    order, cs = R.elimination_order(n, pairs, slack)
    lvl = R.levels(order, cs)
    LB, owner = R.owners(order, cs, lvl, nranks)
    tb = _tail(order, lvl)
    nl = max(lvl.values()) + 1
    prods = defaultdict(list)
    for k in order:
        for a in range(len(cs[k])):
            for b in range(a + 1):
                r, c = cs[k][a], cs[k][b]
                if LB > 0 and lvl[k] < LB and owner[c] != rank:
                    continue
                prods[(r, c)].append(k)
    window = lambda l: l // window_levels if l < tb else nl + l
    out = set()
    for (r, c), ks in prods.items():
        lc = lvl[c]
        groups = defaultdict(list)
        for k in ks:
            groups["late" if lvl[k] == lc - 1 else window(lvl[k])].append(k)
        for key, g in groups.items():
            apply = max(lvl[k] for k in g)
            # a batched level's first side launch holds the passes into the columns of the level after next, the second the rest
            stream = 0 if key == "late" else (1 if window_levels == 1 or apply >= tb or lc == apply + 2 else 2)
            out.add((r, c, apply, stream, tuple(sorted(g))))
    return out, order, cs, lvl, LB, owner, tb


def _check(n, pairs, nranks=1, rank=0, cfg=None):
    cfg = cfg or _config(n)
    up = solver.update_passes(cfg, pairs, nranks=nranks, rank=rank)
    plan = solver.factor_plan(cfg, pairs, nranks=nranks, rank=rank)
    assert up["window"] == _window(cfg)
    exp, order, cs, lvl, LB, owner, tb = _expected_passes(n, pairs, nranks, rank, up["window"])
    passes, sources, join = up["passes"], up["sources"], up["join"]
    assert up["tail"] == tb and (LB == 0 or LB == tb)
    assert plan["update_passes"] == len(passes)
    got, off = [], 0
    for r, c, apply, stream, cnt in passes:
        got.append((int(r), int(c), int(apply), int(stream), tuple(sorted(int(k) for k in sources[off:off + cnt]))))
        off += cnt
    assert off == len(sources)
    # every product in exactly one pass, grouped as restated
    assert len(got) == len(set(got)) and set(got) == exp
    products = [(k, r, c) for r, c, _, _, ks in got for k in ks]
    assert len(products) == len(set(products))
    # launch order: by apply level, the late passes of a level, then its first and its second side launch
    keys = [(a, s) for _, _, a, s, _ in got]
    assert keys == sorted(keys)
    side_launches = {(a, s) for _, _, a, s, _ in got if s > 0}

    def side_done_before_u1(launch, m):
        """Side launch (level, 1 or 2) has finished before the main stream's late passes of level m: some side launch at or after it,
        enqueued before them (at a level < m), is waited for there or earlier (the side stream runs in order)."""
        return any(join[l2][s2 - 1] <= m for l2, s2 in side_launches if launch <= (l2, s2) and l2 < m)

    by_target = defaultdict(list)
    for r, c, apply, stream, ks in got:
        lc = lvl[c]
        src = [lvl[k] for k in ks]
        assert max(src) == apply < lc                                   # applied at its latest source, before its column
        assert (min(src) < tb) == (max(src) < tb)                       # never across the tail boundary (LB when distributed)
        if stream == 0:
            assert set(src) == {lc - 1}                                 # the late pass: level Lc - 1, main stream
        else:
            assert max(src) <= lc - 2
            assert side_done_before_u1((apply, stream), lc - 1)        # before the late pass and the potrf / TRSM of column c
        by_target[(r, c)].append((apply, stream))
    for lst in by_target.values():
        side = [a for a, s in lst if s > 0]
        assert len(side) == len(set(side))                              # one side pass per target per launch: ordered in the stream
        assert sum(1 for _, s in lst if s == 0) <= 1
    return plan


CASES = [(g, n) for g in R.GRAPHS for n in (17, 40) if g != "hierarchical2"] + [("hierarchical2", 40), ("hierarchical2", 300)]


@pytest.mark.parametrize("graph,n", CASES, ids=[f"{g}{n}" for g, n in CASES])
def test_passes_against_restatement(graph, n):
    _check(n, R.GRAPHS[graph](n))


def test_one_pass_per_source_level_at_large_blocks():
    """Frame blocks of 775 unknowns (config 4): one deferred pass per source level."""
    cfg = _config(40, 32, 24)
    assert solver.frame_stride(cfg) == 775
    _check(40, R.hierarchical2(40), cfg=cfg)


@pytest.mark.parametrize("nranks", [2, 4])
def test_distributed_passes(nranks):
    """Passes into column c are computed on owner[c] only, and none crosses the replicated tail (LB)."""
    for q in range(nranks):
        plan = _check(300, R.hierarchical2(300), nranks=nranks, rank=q)
        assert plan["distributed"] == 1


def test_pass_count_at_benchmark_size():
    """Config 2 (300 frames, hierarchical2 pairs): 9796 block products into 8557 (level, target) pairs, applied in 6925 passes."""
    plan = solver.factor_plan(_config(300, 16, 12), R.hierarchical2(300), order_slack=4, num_sms=132)
    assert plan["update_targets"] == 8557 and plan["update_passes"] == 6925
    up = solver.update_passes(_config(300, 16, 12), R.hierarchical2(300))
    assert len(up["sources"]) == 9796 and up["tail"] == 11


# --------------------------------------------------------------------------------------------------------------------------------------
# GPU: factorisations with passes that span several source levels
# --------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nf", [208, 240], ids=["npad208", "npad240-panel"])
def test_multi_level_passes_factor(nf):
    """hierarchical2(40) has targets whose sources lie three and more levels apart: deferred passes of two source levels.  The factor
    matches the dense reference, and is bitwise the same on a graph replay, the single-stream graph and the un-captured profiling run."""
    from tests.test_gpu_linalg import _check as check_factor, _problem
    n, pairs = 40, R.hierarchical2(40)
    P = _problem(nf, n, pairs)
    up = solver.update_passes(P.cfg, pairs)
    order, cs = R.elimination_order(n, pairs)
    lvl = R.levels(order, cs)
    off, multi, spread = 0, 0, 0
    for r, c, apply, stream, cnt in up["passes"]:
        src = {lvl[int(k)] for k in up["sources"][off:off + cnt]}
        off += cnt
        multi += len(src) > 1
        spread = max(spread, lvl[int(c)] - min(src))
    assert up["window"] == 2 and multi > 0 and spread >= 3
    A, D2, b, x = R.well_conditioned(n, nf, pairs, seed=nf)
    _, L = check_factor(P, n, nf, pairs, A, D2, b, x, tag="update-batching")
    P.solve_matrix(A, D2, b)
    assert np.array_equal(P.factor_dense()[1], L), "repeated factorisation differs"
    P.set_overlap(False)
    P.solve_matrix(A, D2, b)
    assert np.array_equal(P.factor_dense()[1], L), "single-stream graph differs"
    P.set_overlap(True)
    P.profile_linear(reps=1)
    assert np.array_equal(P.factor_dense()[1], L), "un-captured profiling run differs"
