"""Joint depth / colour bilateral filter on the GPU (rcvd_bilateral_filter, csrc/rcvd_bilateral.cuh) against the float32 restatement of
the reference loop (tests/bilateral_ref.py::bilateral_filter, lib/Processor.cpp:183-313): through the C ABI and through lib_python."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import bilateral_ref  # noqa: E402
from robust_cvd_b200 import abi, solver, synthetic, synthetic_files  # noqa: E402

pytestmark = pytest.mark.gpu
f32 = np.float32
CV_32FC3 = 21


def scene_stacks(F=7, w=37, h=23, seed=4):
    sc = synthetic.Scene(F, w, h, seed=seed, motion=0.05, rot_deg=0.6)
    depth = np.stack([sc.depth_image(f) for f in range(F)]).astype(f32)
    color = np.stack([synthetic_files.texture(sc, f) for f in range(F)]).astype(f32)
    return depth, color


def launches():
    return solver.lib().rcvd_filter_launch_count()


def window_samples(depth, color, frame, y, x, frame_radius, spatial_radius, depth_sigma, color_sigma):
    """(depth, weight) pairs of one pixel's window, sorted like std::pair (the reference's median order)."""
    F, h, w = depth.shape
    ref = depth[frame, y, x]
    out = []
    for wf in range(max(0, frame - frame_radius), min(F - 1, frame + frame_radius) + 1):
        for wy in range(max(0, y - spatial_radius), min(h - 1, y + spatial_radius) + 1):
            for wx in range(max(0, x - spatial_radius), min(w - 1, x + spatial_radius) + 1):
                e = f32(0)
                d = depth[wf, wy, wx]
                if depth_sigma > 0:
                    t = f32(d - ref); e = f32(e + f32(-f32(t * t) / f32(f32(depth_sigma) * f32(depth_sigma))))
                if color_sigma > 0:
                    c, rc = color[wf, wy, wx], color[frame, y, x]
                    t0, t1, t2 = f32(c[0] - rc[0]), f32(c[1] - rc[1]), f32(c[2] - rc[2])
                    e = f32(e + f32(-f32(f32(f32(t0 * t0) + f32(t1 * t1)) + f32(t2 * t2)) / f32(f32(color_sigma) * f32(color_sigma))))
                out.append((d, f32(np.exp(e)) if e != 0 else f32(1)))
    return sorted(out)


def check_median(got, want, depth, color, out_frames, kw, min_equal=0.995):
    """At least min_equal of the pixels are bit-equal.  Every other one is a sample of its own window, and the running weight in sorted
    order stays within 1e-5 of half the total from the restatement's pick up to the sample before the GPU's (or the other way round):
    a last-ulp difference between CUDA expf and numpy's exp moves the point where the running weight reaches the half, by one rank,
    or by several when the samples in between weigh next to nothing (colour-far samples underflow to ~1e-20)."""
    eq = got == want
    assert eq.mean() >= min_equal, eq.mean()
    for o, y, x in zip(*np.nonzero(~eq)):
        s = window_samples(depth, color, out_frames[o], y, x, kw["frame_radius"], kw["spatial_radius"], kw["depth_sigma"], kw["color_sigma"])
        cum = np.cumsum([float(wt) for _, wt in s]); half = cum[-1] / 2
        gi = [i for i, (d, _) in enumerate(s) if d == got[o, y, x]]; wi = [i for i, (d, _) in enumerate(s) if d == want[o, y, x]]
        assert gi and wi, (o, y, x, got[o, y, x], want[o, y, x])
        lo, hi = min((abs(a - b), min(a, b), max(a, b)) for a in gi for b in wi)[1:]
        assert abs(cum[lo] - half) <= 1e-5 * half and abs(cum[hi - 1] - half) <= 1e-5 * half, (o, y, x, lo, hi, cum[lo], cum[hi - 1], half)


@pytest.mark.parametrize("out_frames", [[0, 1, 2, 3, 4, 5, 6], [1, 3, 4]])
@pytest.mark.parametrize("radius,frame_radius,color_sigma", [(0, 2, 0.0), (1, 2, 0.0), (2, 1, 0.1), (3, 3, 0.05)])
def test_mean_matches_restatement(out_frames, radius, frame_radius, color_sigma):
    depth, color = scene_stacks()
    kw = dict(frame_radius=frame_radius, spatial_radius=radius, depth_sigma=0.3, color_sigma=color_sigma)
    want = bilateral_ref.bilateral_filter(depth, out_frames, color, **kw)
    l0 = launches()
    got = solver.bilateral_filter(depth, out_frames, color if color_sigma > 0 else None, **kw)
    assert launches() == l0 + 1
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=0)
    assert np.abs(got - depth[out_frames]).max() > 1e-4


@pytest.mark.parametrize("median,radius,frame_radius", [(False, 1, 2), (False, 3, 1), (False, 60, 1), (False, 80, 1), (True, 1, 2), (True, 3, 1), (True, 12, 1)])
def test_unit_weights_are_bit_equal(median, radius, frame_radius):
    """depthSigma = colorSigma = 0: every weight is 1, so the sums carry no exp and GPU and restatement agree bit for bit.  The mean
    at radius 60 stages a 152 KB halo tile; at radius 80 the halo does not fit in shared memory and the kernel reads global memory."""
    depth, color = scene_stacks()
    kw = dict(frame_radius=frame_radius, spatial_radius=radius, depth_sigma=0.0, color_sigma=0.0, median=median)
    want = bilateral_ref.bilateral_filter(depth, [0, 2, 3, 6], **kw)
    got = solver.bilateral_filter(depth, [0, 2, 3, 6], **kw)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("radius,frame_radius,depth_sigma,color_sigma", [(1, 2, 0.3, 0.1), (2, 1, 0.3, 0.0), (0, 3, 0.3, 0.2)])
def test_median_matches_restatement(radius, frame_radius, depth_sigma, color_sigma):
    depth, color = scene_stacks()
    kw = dict(frame_radius=frame_radius, spatial_radius=radius, depth_sigma=depth_sigma, color_sigma=color_sigma)
    out_frames = [0, 1, 2, 3, 4, 5, 6]
    want = bilateral_ref.bilateral_filter(depth, out_frames, color, median=True, **kw)
    l0 = launches()
    got = solver.bilateral_filter(depth, out_frames, color, median=True, **kw)
    assert launches() == l0 + 1
    check_median(got, want, depth, color, out_frames, kw)


def test_in_place_recurrence_matches_restatement():
    """In place, frame g's window reads xform_f(filtered_f) for the output frames f before it: one filter launch per output frame, and
    the transform between them is the dense apply kernel (the restatement uses rcvd_depth_apply for it); both are counted."""
    depth, color = scene_stacks()
    cfg = abi.default_config(1, 1.5)                   # Global Scale, as DepthFrame::depth() applies it
    scale = np.array([0.8, 1.25, 1.1, 0.6, 1.4, 0.95, 1.05])
    xp = scale.reshape(-1, 1)
    retransform = lambda f, img: solver.depth_apply(cfg, [scale[f]], img)   # noqa: E731
    out_frames = [1, 2, 3, 5]
    for median in (False, True):
        kw = dict(frame_radius=2, spatial_radius=1, depth_sigma=0.3, color_sigma=0.1, median=median)
        want = bilateral_ref.bilateral_filter(depth, out_frames, color, retransform=retransform, **kw)
        l0 = launches()
        got = solver.bilateral_filter(depth, out_frames, color, in_place=True, xform_cfg=cfg, xform_params=xp, **kw)
        assert launches() == l0 + 2 * len(out_frames)
        if median:
            assert (got == want).mean() >= 0.995
        else:
            np.testing.assert_allclose(got, want, rtol=1e-5, atol=0)
            plain = solver.bilateral_filter(depth, out_frames, color, **kw)
            assert np.abs(plain[1:] - got[1:]).max() > 1e-3          # the recurrence is not the independent filter


def test_median_at_size_with_colour():
    """384 x 224 (the config-2 frame size) with 9 frames, r 2, frame radius 2, colour and median: the real tile grid."""
    sc = synthetic.Scene(9, 384, 224, seed=8, motion=0.03, rot_deg=0.4)
    depth = np.stack([sc.depth_image(f) for f in range(9)]).astype(f32)
    color = np.stack([synthetic_files.texture(sc, f) for f in range(9)]).astype(f32)
    out_frames = [0, 3, 4, 8]
    kw = dict(frame_radius=2, spatial_radius=2, depth_sigma=0.3, color_sigma=0.1)
    want = bilateral_ref.bilateral_filter(depth, out_frames, color, median=True, **kw)
    got = solver.bilateral_filter(depth, out_frames, color, median=True, **kw)
    check_median(got, want, depth, color, out_frames, kw)
    mean_want = bilateral_ref.bilateral_filter(depth, out_frames, color, **kw)
    np.testing.assert_allclose(solver.bilateral_filter(depth, out_frames, color, **kw), mean_want, rtol=1e-5, atol=0)


def test_median_sample_limit():
    """The largest window the median takes (4096 samples: 64 x 64 pixels of one frame) works; 4097 samples are refused."""
    assert abi.BILATERAL_MAX_MEDIAN_SAMPLES == 4096
    rng = np.random.default_rng(5)
    depth = rng.uniform(0.5, 2.0, (1, 64, 64)).astype(f32)
    depth[0, 10:20, 10:20] = 1.0                        # many exact depth ties
    kw = dict(frame_radius=0, spatial_radius=32, depth_sigma=0.0, median=True)
    np.testing.assert_array_equal(solver.bilateral_filter(depth, [0], **kw), bilateral_ref.bilateral_filter(depth, [0], **kw))
    kw["depth_sigma"] = 0.3
    got, want = solver.bilateral_filter(depth, [0], **kw), bilateral_ref.bilateral_filter(depth, [0], **kw)
    assert (got == want).mean() >= 0.995
    over = rng.uniform(0.5, 2.0, (1, 241, 17)).astype(f32)          # 17 x 241 = 4097
    with pytest.raises(RuntimeError, match="at most 4096 samples per pixel; this window has 4097"):
        solver.bilateral_filter(over, [0], frame_radius=0, spatial_radius=120, median=True)
    assert solver.bilateral_filter(over, [0], frame_radius=0, spatial_radius=120, median=False).shape == (1, 241, 17)


# ---- through lib_python ----
@pytest.fixture(scope="module")
def scene_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("bilateral_pipeline"))
    sc = synthetic.Scene(6, 40, 28, seed=13, motion=0.05, rot_deg=0.5)
    synthetic_files.write_scene(sc, root)
    return sc, root


def _open(sc, root):
    import lib_python as lp
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", CV_32FC3)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    v.createDepthStream("filtered", "depth_filtered", [40, 28])
    proc = lp.DepthVideoProcessor(v)
    rp = lp.DepthVideoProcessor.Params(); rp.depthStream = 0
    rp.depthXformDesc.type = lp.XformType.Depth; rp.depthXformDesc.depthType = lp.DepthXformType.Global; rp.depthXformDesc.valueXform = lp.ValueXformType.Scale
    proc.resetDepthXforms(rp)
    # lib_python, like the reference, exposes no setter for transform parameters: they arrive through video.dat (what a solve saves).
    # Write the video, put a distinct scale into every frame's Global transform of stream 0, and load it again.
    import struct
    v.save()
    scale = [1.0 / float(sc.global_scale[f]) for f in range(sc.N)]
    assert all(s != 1.0 for s in scale)
    dat = bytearray(open(os.path.join(root, "video.dat"), "rb").read())
    desc = rp.depthXformDesc.str().encode()
    one, pos, k = struct.pack("<d", 1.0), 0, 0
    while k < sc.N:
        pos = dat.index(desc, pos) + len(desc)
        if dat[pos:pos + 8] == one:                      # a frame's descriptor followed by its parameter (not the stream's)
            dat[pos:pos + 8] = struct.pack("<d", scale[k]); k += 1
    open(os.path.join(root, "video.dat"), "wb").write(bytes(dat))
    v = lp.DepthVideo(); v.load(root)
    assert [v.depthStream(0).frame(f).depthXform().params()[0] for f in range(sc.N)] == scale
    return lp, v, lp.DepthVideoProcessor(v), scale


def test_op_bilateral_filter_default_params_in_place(scene_root):
    """Default Params: stream 0 into itself over every frame, frame radius 2, depthSigma 0.3, mean -- the frame-sequential recurrence."""
    sc, root = scene_root
    lp, v, proc, scale = _open(sc, root)
    ds = v.depthStream(0)
    depth = np.stack([np.array(ds.frame(f).depth()) for f in range(sc.N)])
    color = np.stack([np.array(v.colorStream("down").frame(f).image()) for f in range(sc.N)])
    cfg = abi.default_config(1, 1.5)
    want = bilateral_ref.bilateral_filter(depth, list(range(sc.N)), color, retransform=lambda f, img: solver.depth_apply(cfg, [scale[f]], img))
    p = lp.DepthVideoProcessor.Params(); p.op = lp.DepthVideoProcessor.Op.BilateralFilter
    assert (p.depthStream, p.spatialRadius, p.frameRadius, p.median, p.colorSigma) == (0, 0, 2, False, 0.0) and abs(p.depthSigma - 0.3) < 1e-7
    l0 = launches()
    proc.process(p)
    assert launches() == l0 + 2 * sc.N
    got = np.stack([np.array(ds.frame(f).sourceDepth()) for f in range(sc.N)])
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=0)
    assert np.abs(got - depth).max() > 1e-4
    for f in range(sc.N):       # depth() of a filtered frame is its transform applied to the stored filtered image
        np.testing.assert_array_equal(np.array(ds.frame(f).depth()), solver.depth_apply(cfg, [scale[f]], got[f]))


def test_bilateral_filter_out_of_place_median_partial_range(scene_root):
    sc, root = scene_root
    lp, v, proc, scale = _open(sc, root)
    ds = v.depthStream(0)
    depth = np.stack([np.array(ds.frame(f).depth()) for f in range(sc.N)])
    color = np.stack([np.array(v.colorStream("down").frame(f).image()) for f in range(sc.N)])
    p = lp.DepthVideoProcessor.Params()
    p.depthStream = 1; p.median = True; p.spatialRadius = 1; p.colorSigma = 0.1
    p.frameRange.fromString("1,3-4")
    proc.bilateralFilter(p)
    kw = dict(frame_radius=2, spatial_radius=1, depth_sigma=float(f32(0.3)), color_sigma=float(f32(0.1)))
    want = bilateral_ref.bilateral_filter(depth, [1, 3, 4], color, median=True, **kw)
    got = np.stack([np.array(v.depthStream(1).frame(f).sourceDepth()) for f in (1, 3, 4)])
    check_median(got, want, depth, color, [1, 3, 4], kw)
    for f in (0, 2, 5):
        assert v.depthStream(1).frame(f).sourceDepth() is None
    np.testing.assert_array_equal(np.stack([np.array(ds.frame(f).depth()) for f in range(sc.N)]), depth)   # stream 0 untouched
