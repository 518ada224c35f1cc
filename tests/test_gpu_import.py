"""GPU test of the dataset layouts with ground truth and a COLMAP reconstruction: the reference's PoseOptimizer.__init__
(pose_optimization.py:98-175) imports them, and optimize_poses (:177-240) then starts from the COLMAP cameras. Restated through
lib_python on a synthetic scene whose ground truth and COLMAP reconstruction both hold the scene's true cameras."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from robust_cvd_b200 import solver, synthetic, synthetic_files  # noqa: E402

pytestmark = pytest.mark.gpu
CV_32FC3 = 21
N, W, H = 8, 128, 96
S = 2.5          # COLMAP's world is S times the scene's: its positions are S times larger and its depth maps hold S times the depth


def _write_dataset(root):
    from scipy.spatial.transform import Rotation
    sc = synthetic.Scene(N, W, H, seed=21, motion=0.05, rot_deg=1.0, flow_noise=0.0, depth_noise=0.0, scale_sigma=0.0)
    sc.global_scale[:] = 1.0     # the network depth is the true depth, so the true cameras are what the optimiser should find
    # Scale the world so that frame 0's median depth is 1: normalizeDepth scales the depth that way, and the true cameras then stay
    # true in the optimiser's units. Flow does not change with the world's scale.
    d0 = np.sort(sc.depth_image(0).ravel())
    c = 1.0 / float(d0[d0.size // 2])
    sc.planes = [(n, d * c) for n, d in sc.planes]
    sc.t = sc.t * c
    synthetic_files.write_scene(sc, root)
    vfov, hfov = 2 * np.arctan(sc.phi), 2 * np.arctan(sc.phi * sc.aspect)
    quats = Rotation.from_matrix(sc.R).as_quat()     # x y z w
    # ground truth: depth_gt/poses.txt (lib/Importer.cpp:438-479)
    os.makedirs(os.path.join(root, "depth_gt"))
    with open(os.path.join(root, "depth_gt", "poses.txt"), "w") as f:
        f.write(f"{N}\n" + "".join(" ".join(f"{x:.9g}" for x in (*sc.t[i], *quats[i], hfov, vfov)) + "\n" for i in range(N)))
    # COLMAP: camera-to-world [R | S t] with +x right, +y up, looking down -z (the scene's convention), focal lengths in pixels,
    # and disparity maps 1 / (S depth)
    os.makedirs(os.path.join(root, "colmap_dense"))
    extr = np.concatenate([sc.R, S * sc.t[:, :, None]], axis=2)
    fx, fy = W / (2 * sc.phi * sc.aspect), H / (2 * sc.phi)
    intr = np.tile([fx, fy, W / 2, H / 2], (N, 1))
    np.savez(os.path.join(root, "colmap_dense", "metadata.npz"), extrinsics=extr, intrinsics=intr)
    with open(os.path.join(root, "colmap_dense", "scales.csv"), "w") as f:
        f.write("frame_000000.png,2.0\nframe_000001.png,2.0\n")     # (1 + 2 + 2) / 2 = S, the reference's formula
    os.makedirs(os.path.join(root, "depth_colmap_dense", "depth"))
    py, px = np.mgrid[0:H, 0:W]
    true_depth = []
    for i in range(N):
        D = sc.ray_depth(i, -1.0 + 2.0 * px.ravel() / W, 1.0 - 2.0 * py.ravel() / H).reshape(H, W)
        true_depth.append(D)
        synthetic_files.write_raw(os.path.join(root, "depth_colmap_dense", "depth", f"frame_{i:06d}.raw"), (1.0 / (S * D)).astype(np.float32))
    return sc, np.stack(true_depth)


def _copy_poses(v, src_id, dst_id):   # PoseOptimizer.copy_poses (pose_optimization.py:242-260)
    src, dst = v.depthStream(src_id), v.depthStream(dst_id)
    dst.resetDepthXforms(src.depthXformDesc()); dst.resetSpatialXforms(src.spatialXformDesc())
    for i in range(v.numFrames()):
        s, d = src.frame(i), dst.frame(i)
        d.depthXform().copyFrom(s.depthXform()); d.spatialXform().copyFrom(s.spatialXform())
        d.extrinsics = s.extrinsics; d.intrinsics = s.intrinsics


def _rotation(e):
    from scipy.spatial.transform import Rotation
    return Rotation.from_quat([e.orientation.x(), e.orientation.y(), e.orientation.z(), e.orientation.w()]).as_matrix()


def _rotvec(R):
    from scipy.spatial.transform import Rotation
    return Rotation.from_matrix(R).as_rotvec()


def _cost(d, pose_state):
    from robust_cvd_b200 import abi
    G = solver.Problem(abi.Config.from_buffer_copy(d["config"]))
    try:
        G.set_frames(d["in_range"], d["median"], d["adaptive"] if d["adaptive"].size else None)
        G.set_constraints(d["pair_frames"].reshape(-1, 2), d["offsets"], d["records"].reshape(-1, 6))
        x = d["state"].reshape(N, -1).copy(); x[:, :6] = pose_state
        G.set_state(x)
        return G.evaluate()
    finally:
        G.close()


def test_optimize_poses_from_imported_ground_truth_and_colmap(tmp_path):
    import lib_python as lp
    root = str(tmp_path / "scene")
    sc, true_depth = _write_dataset(root)
    # --- PoseOptimizer.__init__ ---
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("full", "color_full", ".png", CV_32FC3); v.createColorStream("down", "color_down", ".raw", CV_32FC3)
    v.createDepthStream("depth_gt", "depth_gt", [-1, -1])
    gt_id = v.numDepthStreams() - 1
    lp.DepthVideoImporter.importPoses(v, f"{root}/depth_gt/poses.txt", gt_id)
    lp.DepthVideoImporter.importColmapDepth(v)
    v.createDepthStream("colmap_dense", "depth_colmap_dense_imported", [-1, -1])
    colmap_id = v.depthStreamIndex("colmap_dense")
    lp.DepthVideoImporter.importColmapRecon(v, f"{root}/colmap_dense/metadata.npz", colmap_id, False)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    opt_id = v.depthStreamIndex("depth_midas2")
    _copy_poses(v, colmap_id, opt_id)
    v.printInfo(); v.save()
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True)
    fc = lp.FlowConstraintsCollection(v, fp); fc.setStaticFlagFromDynamicMask(8); fc.save()

    # ground-truth stream: the file's values, parsed as float32
    want = np.array(open(f"{root}/depth_gt/poses.txt").read().split()[1:], np.float32).reshape(N, 9)
    gt = v.depthStream(gt_id)
    for i in range(N):
        e, intr = gt.frame(i).extrinsics, gt.frame(i).intrinsics
        got = [*e.position, e.orientation.x(), e.orientation.y(), e.orientation.z(), e.orientation.w(), intr.hFov, intr.vFov]
        np.testing.assert_array_equal(np.array(got, np.float32), want[i])
    # the imported COLMAP depth is the true depth, and the optimised stream starts from the true cameras
    assert lp.DepthVideoImporter.loadScale(root) == S
    disp = synthetic_files.read_raw(f"{root}/depth_colmap_dense_imported/depth/frame_000003.raw")
    np.testing.assert_allclose(disp, 1.0 / true_depth[3], rtol=1e-6)
    ds = v.depthStream(opt_id)
    for i in range(N):
        f = ds.frame(i)
        assert f._enabled and v.depthStream(colmap_id).frame(i)._enabled
        np.testing.assert_allclose(np.asarray(f.extrinsics.position), sc.t[i], atol=2e-7 * max(1.0, np.abs(sc.t).max()))
        np.testing.assert_allclose(_rotation(f.extrinsics), sc.R[i], atol=1e-6)
        assert abs(f.intrinsics.vFov - 2 * np.arctan(sc.phi)) < 1e-6 and abs(f.intrinsics.hFov - 2 * np.arctan(sc.phi * sc.aspect)) < 1e-6

    # --- optimize_poses ---
    v.clearDepthCaches()
    proc = lp.DepthVideoProcessor(v)
    params = lp.DepthVideoProcessor.Params()
    params.depthStream = v.numDepthStreams() - 1
    params.frameRange.fromString("0-7"); params.poseOptimizer.frameRange.fromString("0-7")
    # Two options (--opt.intr_opt, --opt.scale_regularization in the reference) make the true cameras the optimum. The scale
    # regulariser pulls every frame's median depth to 1, which the true depths of a moving camera do not quite satisfy; a weak one
    # still fixes the scale. Per-frame focal lengths let z-translation, focal length and depth scale trade against each other at this
    # narrow field of view; the COLMAP intrinsics are kept fixed instead. With the defaults the positions end ~0.015 from the truth.
    params.poseOptimizer.scaleReg = 1e-3
    params.poseOptimizer.intrOpt = lp.IntrinsicsOptimization.Fixed
    params.op = lp.DepthVideoProcessor.Op.ResetDepthXforms
    params.depthXformDesc.type = lp.XformType.Depth; params.depthXformDesc.depthType = lp.DepthXformType.Global; params.depthXformDesc.valueXform = lp.ValueXformType.Scale
    proc.process(params)
    params.op = lp.DepthVideoProcessor.Op.ResetSpatialXforms
    params.spatialXformDesc.type = lp.XformType.Spatial; params.spatialXformDesc.spatialType = lp.SpatialXformType.Identity; params.spatialXformDesc.valueXform = lp.ValueXformType.Scale
    proc.process(params)
    proc.normalizeDepth(params, fc)
    # The first step's starting state: the imported poses fit the constraints; identity poses, with everything else equal, do not.
    # A transposed rotation or a position multiplied instead of divided by the scale fails this.
    d = lp.DepthVideoPoseOptimizer(v, params.depthStream)._buildProblem(params.poseOptimizer, fc, params.poseOptimizer.depthDeformRegFinal, False)
    x0 = d["state"].reshape(N, -1)
    np.testing.assert_allclose(x0[:, :3], sc.t, atol=1e-6)
    np.testing.assert_allclose(x0[:, 3:6], sc.w_aa, atol=1e-5)
    cost_imported, cost_identity = _cost(d, x0[:, :6]), _cost(d, np.zeros((N, 6)))
    print(f"cost at the imported poses {cost_imported:.6g}, at identity poses {cost_identity:.6g}")
    assert cost_imported < 1e-3 * cost_identity, (cost_imported, cost_identity)
    proc.optimizePoses(params, fc)
    # gauge: express every camera in frame 0's camera and fit the one free scale
    R = np.stack([_rotation(ds.frame(i).extrinsics) for i in range(N)]); p = np.stack([np.asarray(ds.frame(i).extrinsics.position, np.float64) for i in range(N)])
    rel_R, rel_t = R[0].T @ R, (p - p[0]) @ R[0]
    true_R, true_t = sc.R[0].T @ sc.R, (sc.t - sc.t[0]) @ sc.R[0]
    scale = float((rel_t * true_t).sum() / (rel_t * rel_t).sum())
    rot_err = max(np.linalg.norm(_rotvec(true_R[i].T @ rel_R[i])) for i in range(N))
    pos_err = np.abs(scale * rel_t - true_t).max()
    print(f"final relative poses: rotation error {rot_err:.3g} rad, position error {pos_err:.3g} (gauge scale {scale:.6f}, "
          f"trajectory extent {np.abs(true_t).max():.3g})")
    assert rot_err < 1e-3 and pos_err < 1e-3, (rot_err, pos_err)
