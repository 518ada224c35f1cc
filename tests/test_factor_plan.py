"""The block-Cholesky plan (robust_cvd_b200/csrc/rcvd_plan.h) computed on the host through rcvd_debug_factor_plan and checked against the
numpy restatement in tests/linalg_ref.py: elimination order, levels, block counts, the extra frame-graph edges of shared intrinsics, the
position regulariser and triplets, and the multi-GPU distribution (owners, owner-major numbering, per-rank block counts).  No GPU."""
import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import linalg_ref as R


def _config(n, gx=4, gy=4, **kw):
    return abi.default_config(n, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=gx, depth_grid_y=gy, **kw)


def _undirected(pairs):
    return {(min(a, b), max(a, b)) for a, b in pairs if a != b}


def _check_against_reference(plan, n, edges, slack):
    """order and levels equal the numpy restatement over the frame graph `edges`, and so do the counts that follow from its fill."""
    order, cs = R.elimination_order(n, edges, slack)
    lvl = R.levels(order, cs)
    assert list(plan["order"]) == order
    assert list(plan["level"]) == [lvl[f] for f in range(n)]
    assert plan["levels"] == max(lvl.values()) + 1
    assert plan["offdiag_factor_blocks"] == sum(len(cs[k]) for k in order)
    # one update target per (level, target block) pair: the targets (r, c) of every source frame k of the level
    assert plan["update_targets"] == len({(lvl[k], cs[k][a], cs[k][b]) for k in order for a in range(len(cs[k])) for b in range(a + 1)})
    assert plan["h_blocks"] == n + len(_undirected(edges))
    return order, cs, lvl


# disconnected() couples frames up to 3 and needs at least 5
CASES = [(g, n) for g in R.GRAPHS for n in (2, 3, 17, 40) if g != "disconnected" or n >= 5] + [("hierarchical2", 300)]


@pytest.mark.parametrize("slack", [-1, 0, 1, 4])
@pytest.mark.parametrize("graph,n", CASES, ids=[f"{g}{n}" for g, n in CASES])
def test_order_and_levels(graph, n, slack):
    pairs = R.GRAPHS[graph](n)
    plan = solver.factor_plan(_config(n), pairs, order_slack=slack)
    _check_against_reference(plan, n, pairs, slack)
    assert plan["distributed"] == 0 and list(plan["perm"]) == list(range(n)) and not plan["owner"].any()


EXTRA = ["shared_intrinsics", "position_reg", "triplets", "triplets_shared_intrinsics"]


@pytest.mark.parametrize("slack", [-1, 4])
@pytest.mark.parametrize("extra", EXTRA)
@pytest.mark.parametrize("graph,n", [("chain", 17), ("disconnected", 40)], ids=["chain17", "disconnected40"])
def test_extra_edges(graph, n, extra, slack):
    """Shared intrinsics couple every frame of a pair or triplet to frame 0, the position regulariser every (f, f+1, f+2), a triplet
    its (c-1, c, c+1): the plan orders the graph with those edges added."""
    pairs = R.GRAPHS[graph](n)
    kw, centers, edges = {}, [], list(pairs)
    if extra == "position_reg":
        kw["position_reg"] = 0.5
        edges += [e for f in range(n - 2) for e in ((f, f + 1), (f, f + 2), (f + 1, f + 2))]
    if extra.startswith("triplets"):
        centers = list(range(1, n - 1, 3))
        edges += [e for c in centers for e in ((c - 1, c), (c - 1, c + 1), (c, c + 1))]
    if extra.endswith("shared_intrinsics"):
        kw["intr_opt"] = abi.INTR_SHARED
        edges += [(f, 0) for a, b in pairs for f in (a, b)] + [(f, 0) for c in centers for f in (c - 1, c, c + 1)]
    assert _undirected(edges) != _undirected(pairs)          # the case adds edges
    plan = solver.factor_plan(_config(n, **kw), pairs, centers, order_slack=slack)
    _check_against_reference(plan, n, edges, slack)


@pytest.mark.parametrize("pairs,centers,message", [
    ([(0, 1), (2, 5)], [], "pair frame index out of range"),
    ([(-1, 2)], [], "pair frame index out of range"),
    ([(0, 1)], [0], "triplet centre frame out of range"),
    ([(0, 1)], [2, 4], "triplet centre frame out of range"),
])
def test_out_of_range_frames_are_refused(pairs, centers, message):
    with pytest.raises(RuntimeError, match=message):
        solver.factor_plan(_config(5), pairs, centers)


def test_counts_at_benchmark_size():
    """BASELINE config 2 (300 frames, stride 199, npad 208) and config 4 (600 frames, stride 775, npad 784) on an H100's 132 SMs."""
    pairs = R.hierarchical2(300)
    cfg = _config(300, 16, 12)
    plan = solver.factor_plan(cfg, pairs, order_slack=4, num_sms=132)
    got = [plan[k] for k in ("levels", "offdiag_factor_blocks", "h_blocks", "update_targets", "first_substitution_level")]
    assert got == [43, 2138, 1183, 8557, 5]
    assert solver.factor_plan(cfg, pairs, nranks=2)["first_replicated_level"] == 11
    big = solver.factor_plan(_config(600, 32, 24), R.hierarchical2(600), nranks=2)
    assert [big["levels"], big["offdiag_factor_blocks"], big["first_replicated_level"]] == [58, 4558, 19]


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_distributed_plan(nranks):
    n = 300
    pairs = R.hierarchical2(n)
    cfg = _config(n, 16, 12)
    single = solver.factor_plan(cfg, pairs)
    plans = [solver.factor_plan(cfg, pairs, nranks=nranks, rank=q) for q in range(nranks)]
    order, cs = R.elimination_order(n, pairs)
    lvl = R.levels(order, cs)
    LB, owner = R.owners(order, cs, lvl, nranks)
    for p in plans:
        assert p["distributed"] == 1 and p["first_replicated_level"] == LB
        for k in ("order", "level"):                          # the distribution renumbers frames internally, not the schedule
            np.testing.assert_array_equal(p[k], single[k])
        for k in ("levels", "offdiag_factor_blocks", "h_blocks"):
            assert p[k] == single[k]
        np.testing.assert_array_equal(p["owner"], owner)      # every rank computes the same owners
        np.testing.assert_array_equal(p["perm"], plans[0]["perm"])
    assert sum(p["rank_frames"] for p in plans) == n
    assert sum(p["rank_l_blocks"] for p in plans) == n + single["offdiag_factor_blocks"]
    assert sum(p["rank_h_blocks"] for p in plans) == single["h_blocks"]
    # per rank: its frames, their diagonal blocks and the factor blocks of their columns, the H blocks of their columns
    pos = {k: i for i, k in enumerate(order)}
    for q, p in enumerate(plans):
        mine = [f for f in range(n) if owner[f] == q]
        assert p["rank_frames"] == len(mine)
        assert p["rank_l_blocks"] == sum(1 + len(cs[f]) for f in mine)
        assert p["rank_h_blocks"] == len(mine) + sum(1 for a, b in pairs if owner[a if pos[a] < pos[b] else b] == q)
    # internal numbering: owner-major, phase-A frames before phase-B frames within each owner, ascending frame ids inside those
    key = [(owner[f], lvl[f] >= LB, f) for f in plans[0]["perm"]]
    assert key == sorted(key) and sorted(plans[0]["perm"]) == list(range(n))


@pytest.mark.parametrize("extra", ["shared_intrinsics", "position_reg", "triplets"])
def test_replicated_scheme_is_forced(extra):
    """Shared intrinsics, the position regulariser and triplets couple frames by temporal index: the plan stays replicated."""
    n = 300
    kw = {"shared_intrinsics": dict(intr_opt=abi.INTR_SHARED), "position_reg": dict(position_reg=0.5), "triplets": {}}[extra]
    plan = solver.factor_plan(_config(n, **kw), R.hierarchical2(n), [150] if extra == "triplets" else [], nranks=2)
    assert plan["distributed"] == 0 and plan["rank_frames"] == n and not plan["owner"].any()
