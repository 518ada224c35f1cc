"""GPU test of DepthFrame.warp(): the frame's spatial transform evaluated over its stream's size by the dense warp kernel, bit-equal
to spatialXform().warp(h, w), kept until the transform changes and dropped by setDepth, clearCache and clearXformedCache."""
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

pytestmark = pytest.mark.gpu
N, W, H = 3, 40, 24
SPATIAL = ["Identity", "VerticalLinear", "CornersBilinear", "BilinearGrid(4, 3)", "BicubicGrid(5, 4)"]


def _video(root, spec, seed=0):
    """A video whose depth stream "d" ([W, H], no depth files) has the spatial transform `spec` with seeded parameters. Python cannot
    set a transform's parameters, so they are written into the video.dat that DepthVideo.save() writes, right after each frame's
    transform descriptor, and the video is loaded back."""
    import lib_python as lp
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "frames.txt"), "w") as f:
        f.write(f"{N}\n{W}\n{H}\n" + "".join(f"{i / 30.0:.6f}\n" for i in range(N)))
    v = lp.DepthVideo()
    lp.DepthVideoImporter.importVideo(v, root, False)
    v.createDepthStream("d", "d", [W, H])
    desc = lp.XformDescriptor(); desc.reset(lp.XformType.Spatial); desc.parse(spec)
    v.depthStream(0).resetSpatialXforms(desc)
    n = v.depthStream(0).frame(0).spatialXform().numParams()
    v.save()
    fn = os.path.join(root, "video.dat")
    raw = bytearray(open(fn, "rb").read())
    tag = struct.pack("<iQ", 1, len(desc.str())) + desc.str().encode()
    at = [i for i in range(len(raw)) if raw.startswith(tag, i)]
    assert len(at) == N + 1           # the stream's descriptor, then each frame's
    params = np.random.default_rng(seed).normal(scale=0.05, size=(N, n))
    for f, p in enumerate(at[1:]):
        raw[p + len(tag):p + len(tag) + 8 * n] = params[f].tobytes()
    open(fn, "wb").write(bytes(raw))
    v = lp.DepthVideo(); v.load(root)
    for f in range(N):
        assert v.depthStream(0).frame(f).spatialXform().params() == list(params[f])
    return v


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("spec", SPATIAL)
def test_frame_warp_equals_the_transform_warp(tmp_path, spec):
    v = _video(str(tmp_path / "v"), spec)
    ds = v.depthStream(0)
    warps = []
    for f in range(N):
        fr = ds.frame(f)
        got = fr.warp()
        assert got.dtype == np.float32 and got.shape == (H, W, 2)
        np.testing.assert_array_equal(_bits(got), _bits(fr.spatialXform().warp(ds.height(), ds.width())))
        np.testing.assert_array_equal(_bits(fr.warp()), _bits(got))
        warps.append(got)
    if spec != "Identity":      # the seeded parameters differ per frame, so do the warps
        assert not np.array_equal(warps[0], warps[1])


def test_frame_warp_follows_the_transform(tmp_path):
    v = _video(str(tmp_path / "v"), "BicubicGrid(5, 4)")
    ds = v.depthStream(0)
    a, b = ds.frame(0), ds.frame(1)
    before = a.warp()
    a.spatialXform().copyFrom(b.spatialXform())                  # new parameters
    after = a.warp()
    assert not np.array_equal(after, before)
    np.testing.assert_array_equal(_bits(after), _bits(b.spatialXform().warp(H, W)))
    a.resetSpatialXform()                                         # zero parameters
    np.testing.assert_array_equal(_bits(a.warp()), _bits(a.spatialXform().warp(H, W)))
    import lib_python as lp
    desc = lp.XformDescriptor(); desc.reset(lp.XformType.Spatial); desc.parse("CornersBilinear")
    ds.resetSpatialXforms(desc)                                   # a new descriptor
    got = a.warp()
    np.testing.assert_array_equal(_bits(got), _bits(a.spatialXform().warp(H, W)))


def _device_events(fn):
    """Device activities (kernels, copies) of one call, from the CUDA profiler: whether the call recomputed the warp."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def test_frame_warp_cache_is_dropped_with_the_depth_caches(tmp_path):
    v = _video(str(tmp_path / "v"), "BilinearGrid(4, 3)", seed=3)
    fr = v.depthStream(0).frame(2)
    want = _bits(fr.spatialXform().warp(H, W))
    drops = [("setDepth", lambda: fr.setDepth(np.full((H, W), 2.0, np.float32))), ("clearXformedCache", fr.clearXformedCache),
             ("clearCache", fr.clearCache)]
    assert _device_events(fr.warp) > 0
    for name, drop in drops:
        assert _device_events(fr.warp) == 0, name                 # cached
        drop()
        got = []
        assert _device_events(lambda: got.append(fr.warp())) > 0, name
        np.testing.assert_array_equal(_bits(got[0]), want)
