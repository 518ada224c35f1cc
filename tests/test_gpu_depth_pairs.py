"""Pairwise depth normalisation on the H100: the depth-pair family of the C ABI (rcvd_problem_set_depth_pairs, k_depth_pairs) against
the CPU restatement of tests/depth_pairs_ref.py on the same records, and normalizeDepth with normalizeDepthFromFirstFrame = false
through lib_python, replayed on the CPU."""
import os
import sys

import numpy as np
import pytest

from robust_cvd_b200 import abi, solver, synthetic, synthetic_files
from tests import depth_pairs_ref as R
from tests import helpers
from tests.test_depth_pairs import TRANSFORMS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CV_32FC3 = 21
TIGHT = dict(function_tolerance=1e-16, gradient_tolerance=1e-13, parameter_tolerance=1e-13)   # run to the minimum


def _options(max_iterations, **kw):
    o = abi.default_solve_options(max_iterations)
    for f, v in kw.items():
        setattr(o, f, v)
    return o


def _problem(P, cfg, med, pairs, offs, rec, x, static=None):
    P.set_frames(np.ones(cfg.num_frames, np.uint8), med)
    if static is not None:
        P.set_constraints(*static)
    if hasattr(P, "set_depth_pairs"):
        P.set_depth_pairs(pairs, offs, rec)
    P.set_state(x)
    return P


def _reference(cfg, med, pairs, offs, rec, static=None):
    from oracle import oracle
    O = oracle.OracleProblem(cfg)
    O.set_frames(np.ones(cfg.num_frames, np.uint8), med)
    O.set_constraints(*(static if static is not None else (np.zeros((0, 2), np.int32), np.zeros(1, np.int64), np.zeros((0, 6), np.float32))))
    return O, R.DepthPairs(cfg, pairs, offs, rec)


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


@pytest.mark.parametrize("name,overrides", TRANSFORMS, ids=[t[0] for t in TRANSFORMS])
def test_cost_gradient_and_normal_matrix_match_the_restatement(name, overrides):
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=6, sep=12, scale_grid_x=5, scale_grid_y=4, **overrides)
    G = solver.Problem(cfg, device=0)
    off_d, nd = helpers.layout_numbers(cfg)
    x = helpers.initial_state(sc, cfg, G.stride, off_d, nd, perturb=0.05)
    O, ref = _reference(cfg, med, pairs, offs, rec)
    _problem(G, cfg, med, pairs, offs, rec, x)
    cg, gg = G.evaluate(True)
    ct, gt, Ht = R.total(O, ref, x.reshape(-1))
    assert abs(cg - ct) <= 1e-9 * abs(ct)
    assert _rel(gg, gt) <= 1e-9
    assert _rel(G.normal_matrix_dense(), Ht) <= 1e-9
    assert abs(G.evaluate() - ct) <= 1e-9 * abs(ct)              # the cost-only pass


def test_depth_pairs_add_to_the_static_scene_rows():
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=6, sep=12, depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=3)
    G = solver.Problem(cfg, device=0)
    off_d, nd = helpers.layout_numbers(cfg)
    x = helpers.initial_state(sc, cfg, G.stride, off_d, nd)
    dp = (pairs[::2], np.concatenate([[0], np.cumsum(np.diff(offs)[::2])]), np.concatenate([rec[offs[i]:offs[i + 1]] for i in range(0, len(pairs), 2)]))
    O, ref = _reference(cfg, med, *dp, static=(pairs, offs, rec))
    _problem(G, cfg, med, *dp, x, static=(pairs, offs, rec))
    cg, gg = G.evaluate(True)
    ct, gt, Ht = R.total(O, ref, x.reshape(-1))
    assert abs(cg - ct) <= 1e-9 * abs(ct) and _rel(gg, gt) <= 1e-9 and _rel(G.normal_matrix_dense(), Ht) <= 1e-9


@pytest.mark.parametrize("name,overrides", TRANSFORMS[:4], ids=[t[0] for t in TRANSFORMS[:4]])
def test_bounded_solve_reaches_the_reference_minimum(name, overrides):
    """depth_lower_bound = 1, the scale and deformation regularisers (depthDeformRegInitial), as normalizeDepth sets them; 16 frames on the hierarchical2 pair graph (off-diagonal
    factor blocks; Global transforms have npad 16).  (Global ScaleShift runs into the flat minimum scale 0, shift 1: every disparity 1.)"""
    sc = synthetic.Scene(16, 128, 96, seed=2)
    cfg = abi.default_config(16, sc.aspect, depth_lower_bound=1, scale_grid_x=5, scale_grid_y=4, depth_deform_reg=1.0, **overrides)
    pairs, offs, rec = sc.constraints(pairs=synthetic.hierarchical2_pairs(16), sep=24)
    med = sc.median_depths()
    G = solver.Problem(cfg, device=0)
    k = 2 if cfg.value_xform == abi.VALUE_SCALESHIFT else 1
    x0 = np.zeros((16, G.stride)); x0[:, 6] = sc.phi; x0[:, 7:G.stride:k] = 1.0
    O, ref = _reference(cfg, med, pairs, offs, rec)
    _problem(G, cfg, med, pairs, offs, rec, x0)
    s = G.solve(_options(500, **TIGHT))
    assert s.termination != abi.TERM_FAILURE and s.final_cost < s.initial_cost, s.message
    info = G.structure_info()
    xg = G.get_state()
    xr = R.solve(O, ref, x0, R.lower_bounded(cfg, np.ones(16, np.uint8))).reshape(16, -1)
    assert np.all(xg[:, 7:G.stride:k] >= 0.0)
    assert _rel(xg[:, 7:], xr[:, 7:]) <= 1e-6, (xg[:, 7:9], xr[:, 7:9])
    assert info["h_blocks"] > 16 and info["offdiag_factor_blocks"] > 0   # the pairs' cross blocks reached the factorisation
    if cfg.depth_type == abi.DEPTH_GLOBAL:
        assert info["npad"] == 16


def test_normalize_depth_pairwise_through_lib_python(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))
    import lib_python as lp
    root = str(tmp_path / "scene")
    sc = synthetic.Scene(8, 128, 96, seed=3)
    synthetic_files.write_scene(sc, root)
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("full", "color_full", ".png", CV_32FC3); v.createColorStream("down", "color_down", ".raw", CV_32FC3)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True)
    fc = lp.FlowConstraintsCollection(v, fp); fc.setStaticFlagFromDynamicMask(8)
    proc = lp.DepthVideoProcessor(v)
    params = lp.DepthVideoProcessor.Params()
    params.depthStream = v.numDepthStreams() - 1
    params.frameRange.fromString("0-7"); params.poseOptimizer.frameRange.fromString("0-7")
    params.poseOptimizer.maxIterations = 100
    params.op = lp.DepthVideoProcessor.Op.ResetDepthXforms
    params.depthXformDesc.type = lp.XformType.Depth; params.depthXformDesc.depthType = lp.DepthXformType.Global; params.depthXformDesc.valueXform = lp.ValueXformType.Scale
    proc.process(params)
    params.poseOptimizer.normalizeDepthFromFirstFrame = False
    opt = lp.DepthVideoPoseOptimizer(v, params.depthStream)
    d = opt._buildProblem(params.poseOptimizer, fc, 0.0, True)
    assert d["dpair_records"].size > 0
    cfg = abi.Config.from_buffer_copy(d["config"])
    O = R.regulariser_problem(cfg, d["in_range"], d["median"])
    ref = R.DepthPairs(cfg, d["dpair_frames"], d["dpair_offsets"], d["dpair_records"])
    proc.normalizeDepth(params, fc)
    ds = v.depthStream(params.depthStream)
    scales = np.array([ds.frame(f).depthXform().params()[0] for f in range(8)])
    # replay of the same arrays through the C ABI: with the solve options normalizeDepth uses, the same scales; with tight
    # tolerances, the reference minimum
    xr = R.solve(O, ref, d["state"], R.lower_bounded(cfg, d["in_range"])).reshape(8, -1)[:, 7]
    for opts, want, tol in ((_options(100), scales, 1e-6), (_options(100, **TIGHT), xr, 1e-6)):
        G = solver.Problem(cfg, device=0)
        G.set_frames(d["in_range"], d["median"]); G.set_depth_pairs(d["dpair_frames"], d["dpair_offsets"], d["dpair_records"]); G.set_state(d["state"])
        G.solve(opts)
        np.testing.assert_allclose(G.get_state()[:, 7], want, rtol=tol)
    np.testing.assert_allclose(scales, xr, rtol=1e-3)               # Ceres' default function_tolerance stops short of the minimum
    assert np.ptp(scales) > 1e-3 * scales.mean()                   # no copy from the first frame
    for f in range(8):
        assert ds.frame(f).depth() is not None
    # pose optimisation from that state to completion
    params.poseOptimizer.numSteps = 1; params.poseOptimizer.coarseToFine = False; params.poseOptimizer.maxIterations = 50
    proc.optimizePoses(params, fc)
    xs = lp.DepthVideoPoseOptimizer(v, params.depthStream)._buildProblem(params.poseOptimizer, fc, 0.1, False)["state"].reshape(8, -1)
    assert np.all(np.isfinite(xs)) and np.abs(xs[1:, :3]).max() > 0
