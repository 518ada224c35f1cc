"""The constraint-family setters of the C ABI (rcvd_problem_set_constraints, _set_triplets, _set_depth_pairs, _set_structure) refuse
malformed arrays with RCVD_ERR_INVALID before they keep anything: after a refused call the handle evaluates the problem it had, also
once a later call has rebuilt the structure from the kept arrays."""
import ctypes as C

import numpy as np
import pytest

from robust_cvd_b200 import abi, solver
from tests import helpers

pytestmark = pytest.mark.gpu
N = 8


def _families():
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=N, depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=4)
    ce, to, tr = sc.triplets(sep=14)
    dp = (pairs[::2], np.concatenate([[0], np.cumsum(np.diff(offs)[::2])]), np.concatenate([rec[offs[i]:offs[i + 1]] for i in range(0, len(pairs), 2)]))
    fam = {"set_constraints": (pairs, offs, rec), "set_triplets": (ce, to, tr), "set_depth_pairs": dp}
    return sc, cfg, med, {k: tuple(np.array(a) for a in v) for k, v in fam.items()}


def _call(P, setter, n, frames, offsets=None, records=None):
    a = lambda v, t: None if v is None else np.ascontiguousarray(v, t)
    fr, off, rec = a(frames, np.int32), a(offsets, np.int64), a(records, np.float32)
    fn = getattr(P.L, "rcvd_problem_" + setter)
    if setter == "set_structure":
        return fn(P.h, C.c_int32(n), solver._p(fr, C.c_int32))
    return fn(P.h, C.c_int32(n), solver._p(fr, C.c_int32), solver._p(off, C.c_int64), solver._p(rec, C.c_float))


def _set(a, idx, v):
    a = a.copy(); a[idx] = v
    return a


def _bad_inputs(setter, fr, off=None, rec=None):
    """(name, n, frames, offsets, records): each breaks one rule of the valid input (fr, off, rec)"""
    n = len(fr)
    if setter == "set_structure":
        return [("negative count", -1, fr, None, None), ("null frames", n, None, None, None)]
    assert n >= 2 and off[1] >= 5
    out = [("negative count", -1, fr, off, rec), ("null frames", n, None, off, rec), ("null offsets", n, fr, None, rec)]
    out += [("first offset -128", n, fr, _set(off, 0, -128), rec), ("first offset 5", n, fr, _set(off, 0, 5), rec),
            ("decreasing offsets", n, fr, _set(off, 1, off[2] + 1), rec), ("missing records", n, fr, off, None)]
    if setter == "set_triplets":
        out += [("centre 0", n, _set(fr, 0, 0), off, rec), ("centre N-1", n, _set(fr, 0, N - 1), off, rec)]
    else:
        out += [("frame out of range", n, _set(fr, (0, 1), N), off, rec), ("negative frame", n, _set(fr, (0, 0), -1), off, rec),
                ("equal frames", n, _set(fr, (0, 1), fr[0, 0]), off, rec)]
    return out


SETTERS = ["set_constraints", "set_triplets", "set_depth_pairs", "set_structure"]
CASES = [(s, name) for s in SETTERS
         for name, *_ in _bad_inputs(s, np.zeros((2, 2), np.int32), np.array([0, 5, 10]), np.zeros((10, 6), np.float32))]


@pytest.mark.parametrize("setter,case", CASES, ids=[f"{s}-{c.replace(' ', '_')}" for s, c in CASES])
def test_refused_call_changes_nothing(setter, case):
    sc, cfg, med, fam = _families()
    P = solver.Problem(cfg, device=0)
    P.set_frames(np.ones(N, np.uint8), med)
    for s, arrays in fam.items():
        getattr(P, s)(*arrays)
    off_d, nd = helpers.layout_numbers(cfg)
    P.set_state(helpers.initial_state(sc, cfg, P.stride, off_d, nd))
    c0, g0 = P.evaluate(True)

    def same():
        # the cost is reduced in a fixed order; the gradient is summed with atomics, so only the order of its additions may differ
        c, g = P.evaluate(True)
        assert c == c0
        np.testing.assert_allclose(g, g0, rtol=0, atol=1e-12 * np.abs(g0).max())

    valid = fam["set_constraints"][:1] if setter == "set_structure" else fam[setter]   # the global pair graph is the local one
    _, n, fr, off, rec = next(b for b in _bad_inputs(setter, *valid) if b[0] == case)
    with pytest.raises(RuntimeError, match=f"rcvd error {abi.ERR_INVALID}:"):
        solver._check(_call(P, setter, n, fr, off, rec))
    same()
    P.set_frames(np.ones(N, np.uint8), med)          # rebuilds the structure from the arrays the handle kept
    same()
    assert _call(P, setter, len(valid[0]), *valid) == abi.OK   # the same arrays without the defect are accepted
    same()
