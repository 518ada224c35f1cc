"""The constraint lists of rcvd_static_flags and rcvd_prune_static_flags are checked on the host, before any device is needed: a call
that breaks one list rule of include/rcvd.h returns RCVD_ERR_INVALID (on a machine without a GPU too) and leaves the caller's flags as
they were (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from robust_cvd_b200 import abi, solver

F, H, W = 4, 8, 8
SENTINEL = 7


def _lists():
    """Two pairs and two triplets, all valid; flags hold a sentinel that no call may write when it refuses."""
    return {"pair": {"frames": np.array([[0, 1], [2, 3]], np.int32), "offsets": np.array([0, 1, 3], np.int64),
                     "locs": np.full((3, 4), 0.5, np.float32), "flags": np.full(3, SENTINEL, np.uint8)},
            "triplet": {"frames": np.array([1, 2], np.int32), "offsets": np.array([0, 2, 3], np.int64),
                        "locs": np.full((3, 6), 0.5, np.float32), "flags": np.full(3, SENTINEL, np.uint8)}}


def _break(lists, family, rule):
    fam = lists[family]
    if rule == "negative first offset":
        fam["offsets"] = np.array([-4, 1, 3], np.int64)
    elif rule == "positive first offset":
        fam["offsets"] = np.array([1, 1, 3], np.int64)
    elif rule == "decreasing offsets":
        fam["offsets"] = np.array([0, 2, 1], np.int64)
    elif rule == "null locations":
        fam["locs"] = None
    elif rule == "frame out of range":     # a pair frame of F, or a triplet centre without a next frame
        fam["frames"] = np.array([[0, 1], [2, F]], np.int32) if family == "pair" else np.array([1, F - 1], np.int32)
    elif rule == "bad centre":              # a pair frame below 0, or a triplet centre without a previous frame
        fam["frames"] = np.array([[-1, 1], [2, 3]], np.int32) if family == "pair" else np.array([0, 2], np.int32)


def _args(fam):
    def ptr(a, t):
        return None if a is None else a.ctypes.data_as(C.POINTER(t))
    return (C.c_int32(len(fam["frames"])), ptr(fam["frames"], C.c_int32), ptr(fam["offsets"], C.c_int64), ptr(fam["locs"], C.c_float),
            ptr(fam["flags"], C.c_uint8))


def _static_flags(lists):
    masks = np.full((F, H, W), 255, np.uint8)
    return solver.lib().rcvd_static_flags(C.c_int32(0), masks.ctypes.data_as(C.POINTER(C.c_uint8)), C.c_int32(F), C.c_int32(H), C.c_int32(W),
                                          C.c_float(2.0), *_args(lists["pair"]), *_args(lists["triplet"]), None)


def _prune_static_flags(lists):
    lists["pair"]["flags"][0] = 0           # one non-static pair constraint: the call would stamp
    return solver.lib().rcvd_prune_static_flags(C.c_int32(0), C.c_int32(F), C.c_int32(H), C.c_int32(W), C.c_int32(2),
                                                *_args(lists["pair"]), *_args(lists["triplet"]))


RULES = ["negative first offset", "positive first offset", "decreasing offsets", "null locations", "frame out of range", "bad centre"]


@pytest.mark.parametrize("call", [_static_flags, _prune_static_flags], ids=["static_flags", "prune_static_flags"])
@pytest.mark.parametrize("family", ["pair", "triplet"])
@pytest.mark.parametrize("rule", RULES)
def test_a_broken_list_is_refused_before_the_device(call, family, rule):
    lists = _lists()
    _break(lists, family, rule)
    before = {k: v["flags"].copy() for k, v in lists.items()}
    if call is _prune_static_flags:
        before["pair"][0] = 0
    assert call(lists) == abi.ERR_INVALID, solver.lib().rcvd_last_error().decode()
    for k in lists:
        np.testing.assert_array_equal(lists[k]["flags"], before[k], err_msg=k)
