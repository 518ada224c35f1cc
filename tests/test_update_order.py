"""The order of the Schur-update work items within each k_update_tma launch (rcvd_plan.h, order_update_items), read through
rcvd_debug_update_items: the locality order is a permutation of the cost-sorted items of every launch, no two items of a launch write
the same target tile, the single-wave (two-team) launches keep the cost order, and the traffic model (tools/update_traffic.py) sees
fewer distinct operand bytes per wave at the benchmark size.  The GPU tests at the end (`pytest -m gpu`) factor with both orders and
compare the factors bit for bit."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import linalg_ref as R

H100_SMS = 132


def _config(n, gx=4, gy=4):
    return abi.default_config(n, 1.5, depth_type=abi.DEPTH_GRID, depth_grid_x=gx, depth_grid_y=gy)


def _traffic_model():
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "update_traffic.py")
    spec = importlib.util.spec_from_file_location("update_traffic", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


CASES = {"config2": (300, 16, 12), "config4": (600, 32, 24), "hierarchical2_40": (40, 4, 4)}


def _check_orders(n, gx, gy, nranks=1, rank=0):
    cfg, pairs = _config(n, gx, gy), R.hierarchical2(n)
    by_cost = solver.update_items(cfg, pairs, nranks=nranks, rank=rank, num_sms=H100_SMS, order=0)
    local = solver.update_items(cfg, pairs, nranks=nranks, rank=rank, num_sms=H100_SMS, order=1)
    assert np.array_equal(by_cost["launches"], local["launches"]) and np.array_equal(by_cost["products"], local["products"])
    multi = 0
    for off, cnt in local["launches"].reshape(-1, 2):
        a, b = by_cost["items"][off:off + cnt], local["items"][off:off + cnt]
        # the same multiset of items
        assert np.array_equal(a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])])
        # pairwise disjoint target tiles (dst, m0, n0)
        assert len({(int(d), int(m), int(c)) for d, m, c in b[:, [0, 3, 4]]}) == cnt
        if cnt <= H100_SMS:
            assert np.array_equal(a, b), "a single-wave launch keeps the cost order"
        else:
            multi += 1
            cost = a[:, 2] * (a[:, 5] // 8) * (a[:, 6] // 8) * np.where(a[:, 7] & 1, 3, 4)
            assert np.all(np.diff(cost) <= 0), "order 0 is sorted by cost, heaviest first"
    return local, multi


@pytest.mark.parametrize("case", sorted(CASES))
def test_orders_are_permutations_per_launch(case):
    _, multi = _check_orders(*CASES[case])
    assert multi > 0 or case == "hierarchical2_40"


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_orders_distributed(nranks):
    for rank in range(nranks):
        _check_orders(300, 16, 12, nranks, rank)


def test_per_wave_operand_bytes_fall_at_config2():
    """The model's distinct operand bytes per wave and its HBM estimate fall with the locality order; the bytes streamed and the
    target read-modify-write, which the order does not change, stay."""
    UT = _traffic_model()
    old, new = UT.model(2, 0), UT.model(2, 1)
    multi = [i for i, r in enumerate(old) if r["waves"] > 1]
    assert multi
    mean = lambda rows: sum(rows[i]["wave_unique_mean"] * rows[i]["waves"] for i in multi) / sum(rows[i]["waves"] for i in multi)
    assert mean(new) < 0.6 * mean(old)
    assert max(new[i]["wave_unique_max"] for i in multi) < max(old[i]["wave_unique_max"] for i in multi)
    assert sum(r["hbm"] for r in new) < 0.7 * sum(r["hbm"] for r in old)
    for k in ("items", "streamed", "unique", "rmw"):
        assert sum(r[k] for r in new) == sum(r[k] for r in old), k


def test_bad_order_is_refused():
    L = solver.lib()
    L.rcvd_debug_set_update_order.argtypes = [C.c_void_p, C.c_int32]
    assert L.rcvd_debug_set_update_order(None, C.c_int32(1)) == abi.ERR_INVALID
    assert L.rcvd_last_error().decode() == "null problem"
    with pytest.raises(RuntimeError, match="update order must be 0 or 1"):
        solver.update_items(_config(40), R.hierarchical2(40), order=2)


# --------------------------------------------------------------------------------------------------------------------------------------
# GPU: both orders factor bit for bit alike
# --------------------------------------------------------------------------------------------------------------------------------------
def _five_k5():
    return [p for g in range(5) for p in R.complete_range(5 * g, 5 * g + 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("graph,n,nf", [("hierarchical2", 40, 208), ("hierarchical2", 40, 240), ("five_k5", 25, 208)],
                         ids=["hierarchical2-npad208", "hierarchical2-npad240", "five_k5-npad208"])
def test_orders_factor_bitwise(graph, n, nf):
    from tests.test_gpu_linalg import _check as check_factor, _problem
    pairs = R.hierarchical2(n) if graph == "hierarchical2" else _five_k5()
    P = _problem(nf, n, pairs)
    items = [solver.update_items(P.cfg, pairs, order=o)["items"] for o in (0, 1)]
    assert not np.array_equal(*items), "both orders are the same: the test would compare a factorisation with itself"
    A, D2, b, x = R.well_conditioned(n, nf, pairs, seed=nf)
    P.set_update_order(0)
    y0 = P.solve_matrix(A, D2, b)
    order0, L0, Li0 = P.factor_dense(inverses=True)
    P.set_update_order(1)
    y1, L1 = check_factor(P, n, nf, pairs, A, D2, b, x, tag=f"update-order {graph}")
    order1, _, Li1 = P.factor_dense(inverses=True)
    assert np.array_equal(order0, order1)
    assert np.array_equal(L0, L1), "the factor depends on the item order"
    assert np.array_equal(Li0, Li1), "the diagonal-block inverses depend on the item order"
    # the substitution's sums are not ordered (y may differ in the last bits between any two runs): y0 is held to the solve bound
    assert R.solve_error(A + np.diag(D2), y0, b) <= R.SOLVE_TOL
    with pytest.raises(RuntimeError, match="update order must be 0 or 1"):
        P.set_update_order(2)
