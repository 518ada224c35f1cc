"""The caller's state survives every setter of a built handle.  It is the later of the last set_state and the last solve's result:

(a) solve -> setter -> get_state returns the solved state bit for bit, and evaluate() the cost at it;
(b) solve -> set_state(x1) -> setter -> get_state returns x1 bit for bit, and evaluate() the cost of a fresh handle at x1.

Every setter is called with the inputs the handle already has, so only the state handling can change the results.  Before the handle
kept its invalidation rule in one place (drop_structure in rcvd_api.cu), each setter failed one of the two: (a) set_structure,
set_order_slack and set_eval_only, which did not save the solved state; (b) set_frames, the record setters and set_distributed,
which saved the solver's state over the newer x1."""
import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import helpers

pytestmark = pytest.mark.gpu
N = 8
OVERRIDES = helpers.VARIANTS[0][1]      # bilinear depth grid


def _case():
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=N, **OVERRIDES)
    off_d, nd = helpers.layout_numbers(cfg)
    x0 = helpers.initial_state(sc, cfg, solver.frame_stride(cfg), off_d, nd)
    x1 = helpers.initial_state(sc, cfg, solver.frame_stride(cfg), off_d, nd, seed=1)
    return cfg, pairs, offs, rec, med, x0, x1


SETTERS = {
    "set_frames": lambda P, c: P.set_frames(np.ones(N, np.uint8), c["med"]),
    "set_constraints": lambda P, c: P.set_constraints(c["pairs"], c["offs"], c["rec"]),
    "set_triplets": lambda P, c: P.set_triplets(np.zeros(0, np.int32), np.zeros(1, np.int64), np.zeros((0, 10), np.float32)),
    "set_depth_pairs": lambda P, c: P.set_depth_pairs(np.zeros((0, 2), np.int32), np.zeros(1, np.int64), np.zeros((0, 6), np.float32)),
    "set_structure": lambda P, c: P.set_structure(c["pairs"]),
    "set_order_slack": lambda P, c: P.set_order_slack(4),
    "set_eval_only": lambda P, c: P.set_eval_only(False),
    "set_distributed": lambda P, c: P.set_distributed(True),
}


def _solved_handle():
    cfg, pairs, offs, rec, med, x0, x1 = _case()
    P = helpers.setup_problem(solver.Problem(cfg, device=0), cfg, pairs, offs, rec, med, x0)
    P.solve(abi.default_solve_options(max_iterations=30))   # the first few steps can all be rejected
    xs = P.get_state()
    assert not np.array_equal(xs, x0.reshape(xs.shape))
    return P, cfg, dict(pairs=pairs, offs=offs, rec=rec, med=med), x1


@pytest.mark.parametrize("setter", SETTERS)
def test_solved_state_survives(setter):
    P, _, c, _ = _solved_handle()
    xs, cost = P.get_state(), P.evaluate()
    SETTERS[setter](P, c)
    assert np.array_equal(P.get_state(), xs)
    assert P.evaluate() == pytest.approx(cost, rel=1e-12, abs=0)


@pytest.mark.parametrize("setter", SETTERS)
def test_set_state_survives(setter):
    P, cfg, c, x1 = _solved_handle()
    P.set_state(x1)
    SETTERS[setter](P, c)
    assert np.array_equal(P.get_state(), x1.reshape(N, -1))
    fresh = helpers.setup_problem(solver.Problem(cfg, device=0), cfg, c["pairs"], c["offs"], c["rec"], c["med"], x1)
    assert P.evaluate() == pytest.approx(fresh.evaluate(), rel=1e-12, abs=0)
