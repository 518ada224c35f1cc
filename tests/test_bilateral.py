"""Joint depth / colour bilateral filter on the CPU: the vectorised float32 restatement (tests/bilateral_ref.py::bilateral_filter) against a
literal scalar transcription of the reference loop (lib/Processor.cpp:183-313), the committed golden outputs, and the host-side
argument checks of DepthVideoProcessor::bilateralFilter, which all happen before any device work."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import bilateral_ref  # noqa: E402
from robust_cvd_b200 import synthetic, synthetic_files  # noqa: E402

f32 = np.float32
CV_32FC3, CV_8UC3 = 21, 16


def scalar_bilateral(depth, out_frames, color=None, frame_radius=2, spatial_radius=0, depth_sigma=0.3, color_sigma=0.0, median=False,
                     retransform=None):
    """The reference loop transcribed statement by statement, one pixel and one sample at a time."""
    depth = np.array(depth, f32, copy=True)
    F, h, w = depth.shape
    ds2 = f32(f32(depth_sigma) * f32(depth_sigma)); cs2 = f32(f32(color_sigma) * f32(color_sigma))
    out = np.zeros((len(out_frames), h, w), f32)
    for o, frame in enumerate(out_frames):
        f0, f1 = max(0, frame - frame_radius), min(F - 1, frame + frame_radius)
        for y in range(h):
            y0, y1 = max(0, y - spatial_radius), min(h - 1, y + spatial_radius)
            for x in range(w):
                x0, x1 = max(0, x - spatial_radius), min(w - 1, x + spatial_radius)
                ref = depth[frame, y, x]
                sum_d = f32(0); sum_w = f32(0); samples = []
                for wf in range(f0, f1 + 1):
                    for wy in range(y0, y1 + 1):
                        for wx in range(x0, x1 + 1):
                            d = depth[wf, wy, wx]
                            e = f32(0)
                            if depth_sigma > 0:
                                t = f32(d - ref)
                                e = f32(e + f32(-f32(t * t) / ds2))
                            if color_sigma > 0:
                                c, rc = color[wf, wy, wx], color[frame, y, x]
                                t0, t1, t2 = f32(c[0] - rc[0]), f32(c[1] - rc[1]), f32(c[2] - rc[2])
                                d2 = f32(f32(f32(t0 * t0) + f32(t1 * t1)) + f32(t2 * t2))
                                e = f32(e + f32(-d2 / cs2))
                            wt = f32(np.exp(e)) if e != 0 else f32(1)
                            if median:
                                samples.append((d, wt))
                            else:
                                sum_d = f32(sum_d + f32(d * wt))
                            sum_w = f32(sum_w + wt)
                if median:
                    half = f32(sum_w / f32(2)); cum = f32(0)
                    for d, wt in sorted(samples):
                        cum = f32(cum + wt)
                        if cum >= half:
                            out[o, y, x] = d
                            break
                else:
                    out[o, y, x] = f32(sum_d / sum_w) if sum_w > 0 else f32(0)
        if retransform is not None and frame_radius > 0:
            depth[frame] = retransform(frame, out[o])
    return out


def small_case(F=5, w=5, h=4, seed=0):
    rng = np.random.default_rng(seed)
    depth = rng.uniform(0.5, 3.0, (F, h, w)).astype(f32)
    depth[1, 0, :3] = depth[2, 1, 1]            # exact depth ties across frames: the median breaks them by weight
    depth[3, 2, 2] = 0.0; depth[0, 3, 4] = -0.0
    color = rng.uniform(0, 1, (F, h, w, 3)).astype(f32)
    return depth, color


@pytest.mark.parametrize("median", [False, True])
@pytest.mark.parametrize("use_color", [False, True])
@pytest.mark.parametrize("radius", [0, 1, 3])
def test_restatement_equals_scalar_loop(median, use_color, radius):
    depth, color = small_case(seed=radius)
    kw = dict(frame_radius=2, spatial_radius=radius, depth_sigma=0.3, color_sigma=0.1 if use_color else 0.0, median=median)
    for out_frames in ([0, 1, 2, 3, 4], [1, 3, 4]):           # the full stack and a partial, non-consecutive range
        want = scalar_bilateral(depth, out_frames, color, **kw)
        got = bilateral_ref.bilateral_filter(depth, out_frames, color, **kw)
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("median", [False, True])
def test_restatement_in_place_recurrence_equals_scalar_loop(median):
    depth, color = small_case(F=6, seed=7)
    scale = np.array([1.3, 0.7, 1.1, 0.9, 1.6, 0.8], np.float64)
    retransform = lambda f, img: (img.astype(np.float64) * scale[f]).astype(f32)   # noqa: E731  (a Global Scale transform)
    kw = dict(frame_radius=2, spatial_radius=1, depth_sigma=0.3, color_sigma=0.2, median=median, retransform=retransform)
    want = scalar_bilateral(depth, [1, 2, 4], color, **kw)
    got = bilateral_ref.bilateral_filter(depth, [1, 2, 4], color, **kw)
    np.testing.assert_array_equal(got, want)
    # the recurrence changes the result: frame 2 reads frame 1's filtered depth
    plain = bilateral_ref.bilateral_filter(depth, [1, 2, 4], color, **{**kw, "retransform": None})
    np.testing.assert_array_equal(got[0], plain[0])
    if not median:
        assert not np.array_equal(got[1], plain[1])


def test_unit_weights_mean_is_window_average():
    """depthSigma = colorSigma = 0: every weight is 1, the mean is the plain float32 window sum / count."""
    depth, _ = small_case(seed=3)
    got = bilateral_ref.bilateral_filter(depth, [2], frame_radius=1, spatial_radius=1, depth_sigma=0.0)
    s = f32(0)
    for wf in (1, 2, 3):
        for wy in (0, 1):
            for wx in (0, 1):
                s = f32(s + depth[wf, wy, wx])
    assert got[0, 0, 0] == f32(s / f32(12))


def test_restatement_against_committed_golden():
    """tests/golden/bilateral_golden.npz (written by `python tests/bilateral_ref.py`) pins the restatement."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "bilateral_golden.npz"))
    depth, color, scale = g["depth"], g["color"], g["scale"]
    retransform = lambda f, img: (img.astype(np.float64) * scale[f]).astype(f32)   # noqa: E731
    for name, kw in bilateral_ref.golden_configs():
        if kw.pop("in_place", False):
            kw["retransform"] = retransform
        np.testing.assert_array_equal(bilateral_ref.bilateral_filter(depth, list(g["out_frames"]), color, **kw), g[name], err_msg=name)


# ---- the C ABI and lib_python without a device ----
def _no_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is present")
    except ImportError:
        pass


def test_solver_bilateral_filter_needs_a_device():
    from robust_cvd_b200 import solver
    _no_gpu()
    depth, color = small_case()
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        solver.bilateral_filter(depth, [1, 2], color, frame_radius=1, spatial_radius=1, color_sigma=0.1, median=True)


def test_solver_bilateral_filter_rejects_bad_arguments():
    """Argument errors are reported before the device is looked at (so also on a machine without one)."""
    from robust_cvd_b200 import solver
    depth, color = small_case()
    with pytest.raises(RuntimeError, match="ascending"):
        solver.bilateral_filter(depth, [2, 1])
    with pytest.raises(RuntimeError, match="ascending"):
        solver.bilateral_filter(depth, [5])
    with pytest.raises(RuntimeError, match="colour stack"):
        solver.bilateral_filter(depth, [1], color_sigma=0.1)
    with pytest.raises(RuntimeError, match="transform"):
        solver.bilateral_filter(depth, [1], in_place=True)
    big = np.ones((3, 64, 65), f32)              # 64 x 65 x 1 = 4160 samples per pixel
    with pytest.raises(RuntimeError, match="at most 4096 samples"):
        solver.bilateral_filter(big, [1], frame_radius=0, spatial_radius=64, median=True)


@pytest.fixture(scope="module")
def scene_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("bilateral_scene"))
    synthetic_files.write_scene(synthetic.Scene(5, 24, 16, seed=2), root)
    return root


def _open(root, down_type=CV_32FC3):
    lp = pytest.importorskip("lib_python")
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", down_type)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    v.createDepthStream("filtered", "depth_filtered", [24, 16])
    return lp, v


def test_lib_python_bilateral_filter_needs_a_device(scene_root):
    _no_gpu()
    lp, v = _open(scene_root)
    p = lp.DepthVideoProcessor.Params(); p.op = lp.DepthVideoProcessor.Op.BilateralFilter
    proc = lp.DepthVideoProcessor(v)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        proc.process(p)
    p.depthStream = 1; p.colorSigma = 0.1; p.median = True; p.frameRange.fromString("1,3")
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        proc.bilateralFilter(p)


def test_lib_python_bilateral_filter_argument_errors(scene_root, tmp_path):
    lp, v = _open(scene_root)
    proc = lp.DepthVideoProcessor(v)
    p = lp.DepthVideoProcessor.Params()
    p.depthStream = 2
    with pytest.raises(RuntimeError, match="Depth stream out of range"):
        proc.bilateralFilter(p)
    p.depthStream = 1; p.frameRange.fromString("2-7")
    with pytest.raises(RuntimeError, match="out-of-range frame"):
        proc.bilateralFilter(p)
    # a missing depth frame inside the windows of the range
    import shutil
    root = str(tmp_path / "scene")
    shutil.copytree(scene_root, root)
    os.remove(os.path.join(root, "depth_midas2", "depth", "frame_000004.raw"))
    lp, v2 = _open(root)
    p.frameRange.fromString("1-2")
    with pytest.raises(RuntimeError, match="Depth frame 4 of depth stream 0 has no depth image"):
        lp.DepthVideoProcessor(v2).bilateralFilter(p)
    p.frameRange.fromString("0-1")
    p.frameRadius = 2; p.colorSigma = 0.1
    # colour of a different size than the depth
    synthetic_files.write_raw(os.path.join(root, "color_down", "frame_000001.raw"), np.zeros((8, 12, 3), f32))
    lp, v3 = _open(root)
    with pytest.raises(RuntimeError, match="differ in size"):
        lp.DepthVideoProcessor(v3).bilateralFilter(p)
    # a colour stream that is not CV_32FC3
    lp, v4 = _open(scene_root, down_type=CV_8UC3)
    with pytest.raises(RuntimeError, match="CV_32FC3"):
        lp.DepthVideoProcessor(v4).bilateralFilter(p)
    # without a "down" colour stream
    v5 = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v5, scene_root, False)
    v5.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    p.colorSigma = 0.0; p.depthStream = 0
    with pytest.raises(RuntimeError, match="'down' not found"):
        lp.DepthVideoProcessor(v5).bilateralFilter(p)
