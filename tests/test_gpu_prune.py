"""Static-flag pruning on the device (rcvd_prune_static_flags, FlowConstraintsCollection::pruneStaticFlag, reference
lib/FlowConstraints.cpp:662-748): the C ABI against the numpy transcription (tests/prune_ref.py) bit for bit on random constraint
ends, and lib_python's default path against its RCVD_CONSTRAINT_BUILDER=host restatement, flags and the solve that reads them."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from robust_cvd_b200 import solver, synthetic, synthetic_files  # noqa: E402
from tests import prune_ref  # noqa: E402

pytestmark = pytest.mark.gpu
CV_32FC3, CV_8UC1 = 21, 0
F = 8          # frames 6 and 7 belong to no pair


def _locs(rng, n, ends, h, w, distance):
    """n constraints of `ends` ends: pixels over the image, its borders, rows at and beyond h (up to past the disc), as float32
    locations whose end pixel int(loc * w) is the drawn one or a neighbour."""
    xs = np.concatenate([rng.integers(-1, w + 1, n * ends), [0, w - 1, 0, w - 1, w // 2, w // 2, 0, w - 1]])
    ys = np.concatenate([rng.integers(-1, h + min(distance, 2 * h) + 3, n * ends), [0, 0, h - 1, h - 1, h, h + distance, h + 1, h + distance + 1]])
    k = rng.permutation(xs.size)[:n * ends]
    px = np.stack([xs[k], ys[k]], -1).astype(np.float64) + rng.uniform(0, 1, (n * ends, 2))
    return (px / w).astype(np.float32).reshape(n, 2 * ends)


def _case(rng, h, w, distance, p_static=0.7):
    pairs = [(0, 1), (1, 2), (2, 2), (0, 4), (3, 1), (4, 5), (5, 3), (1, 0)]
    P = {}
    for a, b in pairs:
        n = int(rng.integers(0, 40)) if (a, b) != (1, 0) else 0        # one pair without constraints
        P[(a, b)] = (_locs(rng, n, 2, h, w, distance), rng.uniform(size=n) < p_static)
    T = {}
    for t in (1, 3, 6):                                                # centre 6: frames 5, 6, 7 -- two of them with no pair
        n = int(rng.integers(5, 40))
        T[t] = (_locs(rng, n, 3, h, w, distance), rng.uniform(size=n) < p_static)
    return P, T


def _run(P, T, h, w, distance):
    keys, tkeys = sorted(P), sorted(T)
    po = np.concatenate([[0], np.cumsum([len(P[k][1]) for k in keys])]).astype(np.int64)
    to = np.concatenate([[0], np.cumsum([len(T[t][1]) for t in tkeys])]).astype(np.int64)
    pl = np.concatenate([P[k][0] for k in keys]); ps = np.concatenate([P[k][1] for k in keys]).astype(np.uint8)
    tl = np.concatenate([T[t][0] for t in tkeys]); ts = np.concatenate([T[t][1] for t in tkeys]).astype(np.uint8)
    gps, gts = solver.prune_static_flags(F, h, w, distance, keys, po, pl, ps, tkeys, to, tl, ts)
    return ({k: gps[po[i]:po[i + 1]].astype(bool) for i, k in enumerate(keys)},
            {t: gts[to[i]:to[i + 1]].astype(bool) for i, t in enumerate(tkeys)})


def _assert_equal(got, want):
    for k in want:
        np.testing.assert_array_equal(got[k], want[k], err_msg=str(k))


@pytest.mark.parametrize("h,w", [(20, 17), (24, 70), (33, 96)])
@pytest.mark.parametrize("distance", [0, 1, 31, 32, 33, 100, None])
def test_prune_kernels_match_reference(h, w, distance):
    distance = h + w + 9 if distance is None else distance               # a disc larger than the image
    rng = np.random.default_rng(h * 1000 + w + distance)
    P, T = _case(rng, h, w, distance)
    l0 = solver.lib().rcvd_static_flag_launch_count()
    gp, gt = _run(P, T, h, w, distance)
    assert solver.lib().rcvd_static_flag_launch_count() == l0 + 3
    wp, wt = prune_ref.prune_static_flag(P, T, F, h, w, distance)
    _assert_equal(gp, wp); _assert_equal(gt, wt)
    flipped = sum(int((P[k][1] & ~wp[k]).sum()) for k in P) + sum(int((T[t][1] & ~wt[t]).sum()) for t in T)
    assert flipped > 0


def test_all_static_launches_nothing_and_all_dynamic():
    h, w, distance = 24, 70, 5
    rng = np.random.default_rng(3)
    P, T = _case(rng, h, w, distance, p_static=1.0)
    l0 = solver.lib().rcvd_static_flag_launch_count()
    gp, gt = _run(P, T, h, w, distance)
    assert solver.lib().rcvd_static_flag_launch_count() == l0
    assert all(v.all() for v in gp.values()) and all(v.all() for v in gt.values())
    P = {k: (locs, np.zeros(len(s), bool)) for k, (locs, s) in P.items()}
    gp, gt = _run(P, T, h, w, distance)
    assert solver.lib().rcvd_static_flag_launch_count() == l0 + 3
    wp, wt = prune_ref.prune_static_flag(P, T, F, h, w, distance)
    _assert_equal(gp, wp); _assert_equal(gt, wt)
    assert not any(v.any() for v in gp.values()) and any((~v).any() for v in gt.values())
    # a negative distance changes nothing and launches nothing
    l1 = solver.lib().rcvd_static_flag_launch_count()
    gp, gt = _run(P, T, h, w, -1)
    assert solver.lib().rcvd_static_flag_launch_count() == l1
    _assert_equal(gt, {t: s for t, (_, s) in T.items()})


# ---- through lib_python: a 40-frame 384x224 scene with moving dynamic blobs ----
N, W, H = 40, 384, 224


@pytest.fixture(scope="module")
def scene40(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("prune40") / "scene")
    sc = synthetic.Scene(N, W, H, seed=6)
    rng = np.random.default_rng(2)
    yy, xx = np.mgrid[0:H, 0:W]
    c = rng.uniform([0, 0], [H, W], (4, 2)); vel = rng.normal(0, 2.0, (4, 2)); r = rng.uniform(12, 30, 4)
    masks = []
    for f in range(N):
        m = np.full((H, W), 255, np.uint8)
        for k in range(4):
            cy, cx = (c[k] + f * vel[k]) % [H, W]
            m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r[k] ** 2] = 0
        masks.append(m)
    synthetic_files.write_scene(sc, root, dynamic_masks=masks, workers=min(8, os.cpu_count() or 1))
    import lib_python as lp
    v = _open(lp, root)
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True)
    lp.FlowConstraintsCollection(v, fp)                                  # computes the lists on the device and caches them
    return root


def _open(lp, root):
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", CV_32FC3); v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    return v


def _pruned(lp, root, monkeypatch, which, distance):
    """setStaticFlagFromDynamicMask(8) on the default path, then pruneStaticFlag(distance) on `which`."""
    v = _open(lp, root)
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True)
    monkeypatch.delenv("RCVD_CONSTRAINT_BUILDER", raising=False)
    fc = lp.FlowConstraintsCollection(v, fp)
    fc.setStaticFlagFromDynamicMask(8)
    before = {k: np.asarray(a[1]).copy() for k, a in fc._pairs().items()}
    monkeypatch.setenv("RCVD_CONSTRAINT_BUILDER", which)
    l0 = solver.lib().rcvd_static_flag_launch_count()
    fc.pruneStaticFlag(distance)
    launched = solver.lib().rcvd_static_flag_launch_count() - l0
    monkeypatch.delenv("RCVD_CONSTRAINT_BUILDER", raising=False)
    return v, fc, before, launched


@pytest.mark.parametrize("distance", [5, 20])
def test_lib_python_device_prune_equals_host(scene40, monkeypatch, distance):
    import lib_python as lp
    _, gfc, before, glaunch = _pruned(lp, scene40, monkeypatch, "gpu", distance)
    _, hfc, _, hlaunch = _pruned(lp, scene40, monkeypatch, "host", distance)
    assert glaunch == 3 and hlaunch == 0
    gp, hp = gfc._pairs(), hfc._pairs()
    gt, ht = gfc._triplets(), hfc._triplets()
    assert gp.keys() == hp.keys() and gt.keys() == ht.keys() and len(gt) == N - 2
    for k in gp:
        np.testing.assert_array_equal(np.asarray(gp[k][1]), np.asarray(hp[k][1]), err_msg=f"pair {k}")
    for k in gt:
        np.testing.assert_array_equal(np.asarray(gt[k][1]), np.asarray(ht[k][1]), err_msg=f"triplet {k}")
    n_before = sum(int((~s).sum()) for s in before.values())
    n_after = sum(int((~np.asarray(a[1])).sum()) for a in gp.values())
    assert 0 < n_before < n_after                                        # the discs made static constraints non-static
    assert sum(int((~np.asarray(a[1])).sum()) for a in gt.values()) > 0


def test_lib_python_solve_after_device_prune_equals_host(scene40, monkeypatch):
    import lib_python as lp

    def run(which):
        v, fc, _, _ = _pruned(lp, scene40, monkeypatch, which, 5)
        proc = lp.DepthVideoProcessor(v)
        params = lp.DepthVideoProcessor.Params(); params.depthStream = 0
        params.poseOptimizer.frameRange.fromString(f"0-{N - 1}"); params.poseOptimizer.maxIterations = 20
        params.poseOptimizer.numSteps = 1; params.poseOptimizer.coarseToFine = False
        params.depthXformDesc.parse("Grid(Scale, Linear, 4, 3, 1)"); proc.resetDepthXforms(params)
        proc.normalizeDepth(params, fc)
        proc.optimizePoses(params, fc)
        ds = v.depthStream(0)
        flags = {k: np.asarray(a[1]).copy() for k, a in fc._pairs().items()}
        pos = np.stack([ds.frame(i).extrinsics.position for i in range(N)])
        rot = np.array([[ds.frame(i).extrinsics.orientation.x(), ds.frame(i).extrinsics.orientation.y(),
                         ds.frame(i).extrinsics.orientation.z(), ds.frame(i).extrinsics.orientation.w()] for i in range(N)])
        dp = np.stack([np.array(ds.frame(i).depthXform().params()) for i in range(N)])
        return flags, pos, rot, dp
    gf, gpos, grot, gdp = run("gpu")
    hf, hpos, hrot, hdp = run("host")
    for k in gf:
        np.testing.assert_array_equal(gf[k], hf[k], err_msg=f"pair {k}")
    assert np.abs(gpos).max() > 0 and gdp.shape == (N, 12)
    # equal flags give equal problems; the solver's atomic reductions may still reorder the last bits of a sum
    np.testing.assert_allclose(gpos, hpos, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(grot, hrot, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(gdp, hdp, rtol=1e-9, atol=1e-12)
