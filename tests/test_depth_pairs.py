"""Pairwise depth normalisation without a GPU: the CPU restatement of the DisparityDissimilarityCost rows (tests/depth_pairs_ref.py)
checked against itself, finite differences and a closed form; the depth-pair records lib_python assembles for
normalizeDepthFromFirstFrame = false; and what the mode does to the per-frame scales of a synthetic scene."""
import os
import sys

import numpy as np
import pytest

from oracle import host_ref
from robust_cvd_b200 import abi, synthetic, synthetic_files
from tests import depth_pairs_ref as R
from tests import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the depth transforms of the family: Global Scale / ScaleShift, bilinear grid (Scale), Catmull-Rom grid (Scale, ScaleShift)
TRANSFORMS = [
    ("global_scale", dict(depth_type=abi.DEPTH_GLOBAL)),
    ("global_scaleshift", dict(depth_type=abi.DEPTH_GLOBAL, value_xform=abi.VALUE_SCALESHIFT)),
    ("linear_grid_scale", dict(depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=3)),
    ("cubic_grid_scale", dict(depth_type=abi.DEPTH_GRID, depth_cubic=1, depth_grid_x=5, depth_grid_y=4)),
    ("cubic_grid_scaleshift", dict(depth_type=abi.DEPTH_GRID, depth_cubic=1, value_xform=abi.VALUE_SCALESHIFT, depth_grid_x=4, depth_grid_y=3)),
]


def _case(overrides, num_frames=4, sep=16):
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=num_frames, sep=sep, **overrides)
    ref = R.DepthPairs(cfg, pairs, offs, rec)
    off_d, nd = helpers.layout_numbers(cfg)
    x = helpers.initial_state(sc, cfg, ref.stride, off_d, nd, perturb=0.05)
    return sc, cfg, ref, x.reshape(-1)


@pytest.mark.parametrize("name,overrides", TRANSFORMS, ids=[t[0] for t in TRANSFORMS])
def test_jet_and_analytic_jacobians_agree_with_each_other_and_finite_differences(name, overrides):
    sc, cfg, ref, x = _case(overrides)
    ca, ga, Ha = ref.evaluate(x)
    cj, gj, Hj = ref.evaluate(x, jet=True)
    assert ref.rec.shape[0] > 50 and np.abs(ga).max() > 0
    assert abs(ca - cj) <= 1e-12 * abs(ca)
    assert np.abs(ga - gj).max() <= 1e-12 * np.abs(ga).max()
    assert np.abs(Ha - Hj).max() <= 1e-12 * np.abs(Ha).max()
    # central differences of the robustified cost over every depth parameter
    cols = np.flatnonzero(np.abs(ga) > 0)
    for i in cols[:: max(1, cols.size // 12)]:
        h = 1e-6 * max(1.0, abs(x[i]))
        xp, xm = x.copy(), x.copy(); xp[i] += h; xm[i] -= h
        fd = (ref.evaluate(xp)[0] - ref.evaluate(xm)[0]) / (2 * h)
        assert abs(fd - ga[i]) <= 1e-6 * np.abs(ga).max(), (i, fd, ga[i])
    # only depth-transform parameters are reached: no pose, focal or spatial column
    J = ref.rows(x)[1].reshape(ref.rec.shape[0], cfg.num_frames, ref.stride)
    assert not J[:, :, :7].any()


def test_cost_is_the_cauchy_sum_of_the_disparity_differences():
    sc, cfg, ref, x = _case(TRANSFORMS[0][1])
    s = x.reshape(cfg.num_frames, -1)[:, 7]
    f = ref.frames
    r = 1.0 / (s[f[:, 0]] * ref.rec[:, 2].astype(np.float64)) - 1.0 / (s[f[:, 1]] * ref.rec[:, 5].astype(np.float64))
    b = cfg.robustness ** 2
    assert abs(ref.evaluate(x)[0] - 0.5 * np.sum(b * np.log(1.0 + r * r / b))) <= 1e-12 * ref.evaluate(x)[0]
    assert abs(ref.evaluate(x, jet=True)[0] - 0.5 * np.sum(b * np.log(1.0 + r * r / b))) <= 1e-12 * ref.evaluate(x)[0]


@pytest.mark.parametrize("name,overrides", TRANSFORMS[:2] + TRANSFORMS[3:4], ids=["global_scale", "global_scaleshift", "cubic_grid_scale"])
def test_a_clamped_end_contributes_no_derivative(name, overrides):
    """max(D, 1e-6) is Jet max: where the transformed depth is below 1e-6 the constant branch is taken."""
    sc, cfg, ref, x = _case(overrides)
    X = x.reshape(cfg.num_frames, -1).copy()
    X[1, 7:] = 0.0                                       # every node of frame 1: D = 0 (scale and shift 0)
    for jet in (False, True):
        r, J = ref.rows(X.reshape(-1), jet)
        J = J.reshape(-1, cfg.num_frames, ref.stride)
        assert not J[:, 1].any()
        touches1 = (ref.frames == 1).any(axis=1)
        other = np.where(ref.frames[touches1, 0] == 1, ref.frames[touches1, 1], ref.frames[touches1, 0])
        assert np.abs(J[np.flatnonzero(touches1), other]).sum() > 0      # the other end keeps its derivative
        if name != "global_scale":
            continue
        end0 = ref.frames[touches1, 0] == 1                       # r = 1 / 1e-6 - 1 / (s_b d_b)
        np.testing.assert_allclose(np.abs(r[touches1][end0]), np.abs(1e6 - 1.0 / (X[ref.frames[touches1][end0, 1], 7] * ref.rec[touches1][end0, 5])), rtol=1e-12)


# ---------------------------------------------------------------------------------------------------------------------------------
# records assembled by lib_python
# ---------------------------------------------------------------------------------------------------------------------------------
CV_32FC3, CV_8UC1 = 21, 0


@pytest.fixture(autouse=True)
def _host_constraint_builder(monkeypatch):
    monkeypatch.setenv("RCVD_CONSTRAINT_BUILDER", "host")   # no GPU: the sequential host builder


def _lp():
    sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))
    return pytest.importorskip("lib_python")


def test_depth_pair_records_of_the_pairwise_normalisation(tmp_path):
    lp = _lp()
    root = str(tmp_path / "scene")
    sc, pairs, masks = helpers.write_masked_scene(root)
    # invalid source depth in frame 2: disparity 0 (depth inf) in one block, negative in another
    path = f"{root}/depth_midas2/depth/frame_000002.raw"
    disp = synthetic_files.read_raw(path).copy()
    disp[10:40, 10:60] = 0.0; disp[50:80, 60:120] = -1.0
    synthetic_files.write_raw(path, disp)
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("full", "color_full", ".png", CV_32FC3); v.createColorStream("down", "color_down", ".raw", CV_32FC3)
    v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True)
    fc = lp.FlowConstraintsCollection(v, fp); fc.setStaticFlagFromDynamicMask(8)
    sid = v.numDepthStreams() - 1
    opt = lp.DepthVideoPoseOptimizer(v, sid)
    params = lp.DepthVideoPoseOptimizer.Params(); params.frameRange.fromString("0-5")
    assert params.normalizeDepthFromFirstFrame is True
    d = opt._buildProblem(params, fc, 0.0, True)                   # default: first-frame mode, no pairs
    assert d["dpair_frames"].size == 0 and d["dpair_records"].size == 0 and d["dpair_offsets"].tolist() == [0]
    params.normalizeDepthFromFirstFrame = False
    d = opt._buildProblem(params, fc, 0.0, True)
    ds = v.depthStream(sid)
    recs, offs, pf, nonstatic, dropped = [], [0], [], 0, 0
    for (a, b), (loc, st) in sorted(fc._pairs().items()):          # std::map order
        if a > 5 or b > 5:
            continue
        r = host_ref.observation_records(loc, ds.frame(a).sourceDepth(), ds.frame(b).sourceDepth(), v.invAspect())
        nonstatic += int((~st).sum()); dropped += loc.shape[0] - r.shape[0]
        recs.append(r); offs.append(offs[-1] + len(r)); pf += [a, b]
    np.testing.assert_array_equal(d["dpair_records"].reshape(-1, 6), np.concatenate(recs))
    np.testing.assert_array_equal(d["dpair_offsets"], offs)
    np.testing.assert_array_equal(d["dpair_frames"], pf)
    assert nonstatic > 0 and dropped > 0                            # both rules were exercised
    rec = d["dpair_records"].reshape(-1, 6)
    assert np.all(np.isfinite(rec[:, [2, 5]])) and np.all(rec[:, [2, 5]] > 0)
    assert d["records"].size == 0 and d["pair_frames"].size == 0   # no static-scene rows in the normalisation
    assert set(map(tuple, d["dpair_frames"].reshape(-1, 2))) == {k for k in fc._pairs() if max(k) <= 5}


# ---------------------------------------------------------------------------------------------------------------------------------
# what the mode does to the scales (CPU oracle for the regularisers, the restatement for the pairs)
# ---------------------------------------------------------------------------------------------------------------------------------
def _normalise_both_ways(sc, pairs, offs, rec, med):
    cfg = abi.default_config(sc.N, sc.aspect, depth_type=abi.DEPTH_GLOBAL, depth_lower_bound=1, scale_grid_x=10, scale_grid_y=8)
    ir = np.ones(sc.N, np.uint8)
    O = R.regulariser_problem(cfg, ir, med)
    x0 = np.zeros((sc.N, R.frame_stride(cfg))); x0[:, 6] = sc.phi; x0[:, 7] = 1.0
    # first-frame mode: the scale regulariser alone, then frame 0's transform copied to all (lib/PoseOptimizer.cpp:1127-1138)
    O.set_state(x0)
    O.solve(abi.default_solve_options(max_iterations=100))
    first = np.full(sc.N, O.get_state()[0, 7])
    ref = R.DepthPairs(cfg, pairs, offs, rec)
    pairwise = R.solve(O, ref, x0, R.lower_bounded(cfg, ir)).reshape(sc.N, -1)[:, 7]
    return first, pairwise


def _disagreement(s, pairs, offs, rec):
    f = np.repeat(np.asarray(pairs).reshape(-1, 2), np.diff(offs), axis=0)
    da, db = s[f[:, 0]] * rec[:, 2].astype(np.float64), s[f[:, 1]] * rec[:, 5].astype(np.float64)
    return np.median(np.abs(1.0 / da - 1.0 / db) * da)


def test_pairwise_normalisation_gives_each_frame_its_scale():
    sc = synthetic.Scene(8, 128, 96, seed=4)
    pairs, offs, rec = sc.constraints(sep=12)
    med = sc.median_depths()
    first, pairwise = _normalise_both_ways(sc, pairs, offs, rec, med)
    assert np.ptp(pairwise) > 0.05 * pairwise.mean()
    assert _disagreement(pairwise, pairs, offs, rec) < 0.5 * _disagreement(first, pairs, offs, rec)


def test_pairwise_normalisation_survives_a_mostly_invalid_first_frame():
    """With frame 0's depth more than half invalid its median is 0: the scale row of frame 0 is clamped (zero Jacobian), the first-frame
    mode leaves scale 1 everywhere (reference behaviour, SURVEY A12); the pairs still tie frame 0 to its neighbours."""
    sc = synthetic.Scene(8, 128, 96, seed=4)
    pairs, offs, rec = sc.constraints(sep=12)
    med = sc.median_depths(); med[0] = 0.0
    first, pairwise = _normalise_both_ways(sc, pairs, offs, rec, med)
    np.testing.assert_array_equal(first, 1.0)
    assert np.all(np.isfinite(pairwise)) and np.all(np.abs(pairwise - 1.0) > 1e-3)
