"""FlowConstraintsCollection.pruneStaticFlag without a GPU: the sequential host restatement (RCVD_CONSTRAINT_BUILDER=host) against the
numpy transcription of the reference (tests/prune_ref.py), flag for flag; and the C ABI's refusal without a device."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

lp = pytest.importorskip("lib_python")
from robust_cvd_b200 import abi, solver, synthetic, synthetic_files  # noqa: E402
from tests import prune_ref  # noqa: E402
from tests.helpers import write_masked_scene  # noqa: E402

CV_32FC3, CV_8UC1 = 21, 0


@pytest.fixture(autouse=True)
def _host_constraint_builder(monkeypatch):
    monkeypatch.setenv("RCVD_CONSTRAINT_BUILDER", "host")


@pytest.fixture(scope="module")
def masked_scene(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("prune8"))
    write_masked_scene(root)
    return root


@pytest.fixture(scope="module")
def aspect_scene(tmp_path_factory):
    """A 96x64 "down" stream in a video whose frames.txt says 64x64: constraint rows are y / 64 (inverse aspect 1), so the end pixel
    row int(loc.y * 96) runs up to 1.5 h.  The dynamic masks are square (64x64), so that setStaticFlagFromDynamicMask's own rows stay
    inside its masks."""
    root = str(tmp_path_factory.mktemp("prune_aspect"))
    sc = synthetic.Scene(6, 96, 64, seed=11)
    rng = np.random.default_rng(4)
    masks = []
    for _ in range(sc.N):
        m = np.full((64, 64), 255, np.uint8); cx, cy = rng.integers(12, 52, 2); m[cy - 9:cy + 9, cx - 9:cx + 9] = 0; masks.append(m)
    synthetic_files.write_scene(sc, root, full_size=(64, 64), dynamic_masks=masks)
    return root


def _collection(root):
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", CV_32FC3); v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True)
    fc = lp.FlowConstraintsCollection(v, fp)           # the first call computes the lists and caches them in the scene directory
    fc.setStaticFlagFromDynamicMask(8)
    ds = v.colorStream("down")
    return v, fc, ds.height(), ds.width()


def _state(fc):
    P = {k: (np.asarray(a[0]).copy(), np.asarray(a[1]).copy()) for k, a in fc._pairs().items()}
    T = {k: (np.asarray(a[0]).copy(), np.asarray(a[1]).copy()) for k, a in fc._triplets().items()}
    return P, T


def _check_against_reference(v, fc, h, w, distance):
    P0, T0 = _state(fc)
    fc.pruneStaticFlag(distance)
    P1, T1 = _state(fc)
    want_p, want_t = prune_ref.prune_static_flag(P0, T0, v.numFrames(), h, w, distance)
    assert P1.keys() == want_p.keys() and T1.keys() == want_t.keys()
    for k in P1:
        np.testing.assert_array_equal(P1[k][0], P0[k][0])
        np.testing.assert_array_equal(P1[k][1], want_p[k], err_msg=f"pair {k}")
    for k in T1:
        np.testing.assert_array_equal(T1[k][1], want_t[k], err_msg=f"triplet {k}")
    flipped = sum(int((P0[k][1] & ~P1[k][1]).sum()) for k in P1) + sum(int((T0[k][1] & ~T1[k][1]).sum()) for k in T1)
    return P0, T0, flipped


@pytest.mark.parametrize("distance", [0, 1, 5, 20])
def test_host_prune_matches_reference(masked_scene, distance):
    v, fc, h, w = _collection(masked_scene)
    P0, T0, flipped = _check_against_reference(v, fc, h, w, distance)
    assert sum(int((~s).sum()) for _, s in P0.values()) > 0                  # dynamic pair constraints stamp
    assert sum(len(s) for _, s in T0.values()) > 20                          # triplets are looked up
    if distance >= 5:
        assert flipped > 0                                                   # the discs reach static constraints


def test_host_prune_clamps_rows_beyond_the_image(aspect_scene):
    v, fc, h, w = _collection(aspect_scene)
    assert (w, h) == (96, 64) and v.invAspect() == 1.0
    P0, _ = _state(fc)
    rows = np.concatenate([(locs[:, [1, 3]] * np.float32(w)).astype(np.int64).ravel() for locs, _ in P0.values()])
    assert (rows >= h).sum() > 100                                          # lookups the reference makes past the frame
    _, _, flipped = _check_against_reference(v, fc, h, w, 5)
    assert flipped > 0


def test_negative_distance_changes_nothing(masked_scene):
    v, fc, h, w = _collection(masked_scene)
    P0, T0 = _state(fc)
    fc.pruneStaticFlag(-3)
    P1, T1 = _state(fc)
    for k in P0:
        np.testing.assert_array_equal(P1[k][1], P0[k][1])
    for k in T0:
        np.testing.assert_array_equal(T1[k][1], T0[k][1])


def test_missing_down_stream_raises(masked_scene):
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, masked_scene, False)
    v.createColorStream("down", "color_down", ".raw", CV_32FC3); v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True)
    fc = lp.FlowConstraintsCollection(v, fp)
    fc.setStaticFlagFromDynamicMask(8)
    v2 = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v2, masked_scene, False)
    fc2 = lp.FlowConstraintsCollection(v2, fp)                                # loads the cached lists; the video has no "down" stream
    with pytest.raises(RuntimeError, match="Color stream 'down' not found"):
        fc2.pruneStaticFlag(5)


def test_prune_reports_no_device():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is present")
    except ImportError:
        pass
    no_device = rf"^rcvd error {abi.ERR_NO_DEVICE}: no usable CUDA device \(.+\); this library has no CPU fallback$"
    locs = np.full((1, 4), 0.5, np.float32)
    with pytest.raises(RuntimeError, match=no_device):
        solver.prune_static_flags(2, 8, 8, 2, [(0, 1)], [0, 1], locs, [0])
