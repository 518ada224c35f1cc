"""The first update pass into each fill block of the block-Cholesky factor (an L block that the normal matrix H does not have), read
through rcvd_debug_update_passes: k_load_factor leaves the interior of a fill block alone and that pass writes the block without reading
it (k_update_tma, kUpdFirstFill).  Checked against the elimination structure restated in tests/linalg_ref.py, single-GPU and for every
rank of the distributed factorisation, without a GPU; the last test (`pytest -m gpu`) factors a graph whose first passes run on both
launch shapes of k_update_tma."""
from collections import defaultdict

import pytest

from robust_cvd_b200 import abi, solver
from tests import linalg_ref as R

SYM, FIRST_FILL = 1, 2


def _config(n, gx=4, gy=4):
    return abi.default_config(n, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=gx, depth_grid_y=gy)


def _structure(n, pairs, nranks=1):
    """(fill blocks, earliest source level of every off-diagonal target, levels, LB, owners): the fill blocks are the (r, c) factor
    blocks, c eliminated first, whose frames H does not couple."""
    order, cs = R.elimination_order(n, pairs)
    lvl = R.levels(order, cs)
    LB, owner = R.owners(order, cs, lvl, nranks)
    edges = {(min(a, b), max(a, b)) for a, b in pairs if a != b}
    fill = {(r, k) for k in order for r in cs[k] if (min(r, k), max(r, k)) not in edges}
    first = {}
    for k in order:
        for a in range(len(cs[k])):
            for b in range(a):
                t = (cs[k][a], cs[k][b])
                first[t] = min(first.get(t, lvl[k]), lvl[k])
    return fill, first, lvl, LB, owner


def _passes(cfg, pairs, nranks=1, rank=0):
    """[(r, c, source frames, flags)] of one rank's update passes, in launch order."""
    up = solver.update_passes(cfg, pairs, nranks=nranks, rank=rank)
    out, off = [], 0
    for (r, c, _, _, cnt), fl in zip(up["passes"], up["flags"]):
        out.append((int(r), int(c), [int(k) for k in up["sources"][off:off + cnt]], int(fl)))
        off += cnt
    return out


def _check_rank(passes, fill, first, lvl):
    """Only fill blocks are flagged, at most once each, and a flagged pass is the rank's first pass into its block; a rank's first pass
    into a fill block is flagged exactly when it holds the block's earliest product.  Returns the flagged blocks."""
    flagged, seen = set(), set()
    for r, c, ks, fl in passes:
        assert bool(fl & SYM) == (r == c)
        is_first = (r, c) not in seen
        if fl & FIRST_FILL:
            assert (r, c) in fill, (r, c)                       # never a diagonal block or a block of H's structure
            assert is_first, (r, c)                             # the block's first pass in launch order, so flagged once
            flagged.add((r, c))
        if (r, c) in fill and is_first:
            assert bool(fl & FIRST_FILL) == (min(lvl[k] for k in ks) == first[(r, c)]), (r, c)
        seen.add((r, c))
    return flagged


CASES = [(g, n) for g in R.GRAPHS for n in (17, 40) if g != "hierarchical2"] + [("hierarchical2", 40), ("hierarchical2", 300)]


@pytest.mark.parametrize("graph,n", CASES, ids=[f"{g}{n}" for g, n in CASES])
def test_every_fill_block_has_one_first_pass(graph, n):
    pairs = R.GRAPHS[graph](n)
    fill, first, lvl, _, _ = _structure(n, pairs)
    flagged = _check_rank(_passes(_config(n), pairs), fill, first, lvl)
    assert flagged == fill


def test_first_passes_at_benchmark_size():
    """Config 2 (300 frames, hierarchical2 pairs, 16 x 12 grid): 2138 off-diagonal factor blocks, 1183 - 300 of them in H, so 1255 fill
    blocks, each written by its first pass without being read."""
    n, pairs = 300, R.hierarchical2(300)
    fill, first, lvl, _, _ = _structure(n, pairs)
    assert len(fill) == 2138 - (1183 - 300) == 1255
    flagged = _check_rank(_passes(_config(n, 16, 12), pairs), fill, first, lvl)
    assert flagged == fill


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_first_passes_distributed(nranks):
    """Every fill block is flagged on the owner of its column, which applies all of its phase-A products; another rank flags it only
    when the block has no phase-A product (its copy of the block comes from the owner's broadcast at the phase boundary and the first
    replicated pass overwrites it)."""
    n, pairs = 300, R.hierarchical2(300)
    cfg = _config(n)
    fill, first, lvl, LB, owner = _structure(n, pairs, nranks)
    assert LB > 0
    flagged = [_check_rank(_passes(cfg, pairs, nranks, q), fill, first, lvl) for q in range(nranks)]
    for q in range(nranks):
        for r, c in fill:
            if owner[c] == q:
                assert (r, c) in flagged[q]
            else:
                assert ((r, c) in flagged[q]) == (first[(r, c)] >= LB)
    counts = defaultdict(int)
    for f in flagged:
        for t in f:
            counts[t] += 1
    assert set(counts) == fill


@pytest.mark.gpu
def test_first_passes_on_both_launch_shapes_factor():
    """hierarchical2(300) at nf = 23 (npad 32, neff 24: fill blocks with padding rows and columns) puts first passes into fill blocks in
    launches of at most one item per SM (k_update_tma<2>) and in larger ones (k_update_tma<1>).  The factor matches the dense
    reference, and the launch counters show both shapes ran."""
    import torch
    from tests.test_gpu_linalg import _problem, _well
    n, nf, pairs = 300, 23, R.hierarchical2(300)
    P = _problem(nf, n, pairs)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    up = solver.update_passes(P.cfg, pairs, num_sms=sms)
    items, first_fill = defaultdict(int), defaultdict(int)          # one 24 x 24 tile per target: one item per pass
    for (r, c, apply, stream, _), fl in zip(up["passes"], up["flags"]):
        items[(apply, stream)] += 1
        first_fill[(apply, stream)] += bool(fl & FIRST_FILL)
    assert any(v and items[k] <= sms for k, v in first_fill.items())
    assert any(v and items[k] > sms for k, v in first_fill.items())
    _well(P, n, nf, pairs, seed=5, tag="fill-first-pass")
    p = P.linear_paths()
    assert p["update_tma2"] > 0 and p["update_tma1"] > 0
