"""Frame downscaling on the GPU (rcvd_resize_area, robust_cvd_b200.video): bit for bit against cv2.resize(INTER_AREA) and the float32
restatement tests/resize_ref.py on every path (integer factors, area tables, upscale and mixed) and at the production shapes, batches
beyond one launch's 65535 frames and beyond one host chunk, the .raw bytes against the reference's writer format, the PNG pixels against
the reference's own files (tests/golden/downscale_golden.npz), and end to end: downscale_all on a color_full directory, read back through
lib_python's "down" stream."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

from tests import resize_ref as ref
from tests.test_downscale import GOLDEN, PRODUCTION, bits_equal, golden_calls, sweep_cases, write_dir
from robust_cvd_b200 import solver, synthetic_files, video

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cv2_outputs(frames_bgr, h, w):
    """cv2's results for [F, H, W, 3] u8 B, G, R frames: float32 B, G, R, and the PNG pixels R, G, B."""
    import cv2
    raw = np.stack([cv2.resize(ref.to_float(f), (w, h), interpolation=cv2.INTER_AREA) for f in frames_bgr])
    return raw, ref.to_png_u8(raw)[..., ::-1]


def check_call(frames_bgr, sizes):
    """One rcvd_resize_area call with a raw and a png output per size, against cv2; returns the number of differing values."""
    outs = solver.resize_area(frames_bgr, [(h, w, kind) for h, w in sizes for kind in ("raw", "png")])
    bad = 0
    for k, (h, w) in enumerate(sizes):
        raw, pngpix = cv2_outputs(frames_bgr, h, w)
        bad += int((outs[2 * k].view(np.uint32) != raw.view(np.uint32)).sum()) + int((outs[2 * k + 1] != pngpix).sum())
    return bad


def test_sweep_bit_equal_to_cv2():
    rng = np.random.default_rng(11)
    bad, paths = 0, {}
    for W, H, w, h in sweep_cases():
        frames = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
        bad += check_call(frames, [(h, w)])
        paths[ref.resize_path(W, H, w, h)] = paths.get(ref.resize_path(W, H, w, h), 0) + 1
    print(f"sweep paths {paths}: {bad} values differ from cv2")
    assert bad == 0


def test_three_outputs_per_call_and_restatement():
    """Three sizes of one batch in one call (every path at once), against cv2 and the restatement."""
    rng = np.random.default_rng(12)
    frames = rng.integers(0, 256, (3, 45, 60, 3), dtype=np.uint8)
    sizes = [(15, 20), (31, 25), (50, 64)]                      # integer 3 x 3, area tables, upscale
    assert [ref.resize_path(60, 45, w, h) for h, w in sizes] == ["integer", "area", "linear"]
    outs = solver.resize_area(frames, [(15, 20, "raw"), (31, 25, "png"), (50, 64, "raw")])
    for (h, w), out in zip(sizes, outs):
        for f, o in zip(frames, out):
            want = ref.resize_area(ref.to_float(f), w, h)
            if o.dtype == np.uint8:
                np.testing.assert_array_equal(o, ref.to_png_u8(want)[..., ::-1])
            else:
                assert bits_equal(o, want)


def test_production_shapes():
    rng = np.random.default_rng(13)
    bad = 0
    by_source = {}
    for (W, H), (w, h) in PRODUCTION:
        by_source.setdefault((W, H), []).append((h, w))
    for (W, H), sizes in by_source.items():
        frames = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
        for hw in sizes:
            bad += check_call(frames, [hw])
        got = solver.resize_area(frames[:1], [(h, w, "raw") for h, w in sizes])   # up to three sizes in one call
        for (h, w), o in zip(sizes, got):
            assert bits_equal(o[0], ref.resize_area(ref.to_float(frames[0]), w, h)), (W, H, w, h)
    assert bad == 0


def test_more_frames_than_one_launch():
    """70000 tiny frames: grid.y takes at most 65535 frames per launch.  The restatement resizes every frame at once as channels of one
    image (each channel's arithmetic is the same)."""
    rng = np.random.default_rng(14)
    F = 70000
    frames = rng.integers(0, 256, (F, 3, 5, 3), dtype=np.uint8)
    L = solver.lib()
    L.rcvd_resize_launch_count.restype = C.c_int64
    n0 = L.rcvd_resize_launch_count()
    raw, pngpix = solver.resize_area(frames, [(2, 3, "raw"), (2, 3, "png")])
    assert L.rcvd_resize_launch_count() - n0 == 4
    stacked = ref.to_float(frames.transpose(1, 2, 0, 3).reshape(3, 5, F * 3))
    want = ref.resize_area(stacked, 3, 2).reshape(2, 3, F, 3).transpose(2, 0, 1, 3)
    assert bits_equal(raw, want)
    np.testing.assert_array_equal(pngpix, ref.to_png_u8(want)[..., ::-1])


def _golden_dir(g, name, root):
    frames = g[f"{name}/frames"]
    write_dir(root, frames)
    return frames


def test_every_golden_call_through_video(tmp_path):
    """Video(path).downscale_frames with each fixture call's arguments writes the reference's files: the .raw files byte for byte as
    save_raw_float32_image writes them (header h, w, CV_32FC3 = 21, 12 as <iiiQ, then the B, G, R floats), the PNGs decoding to the
    reference's pixels."""
    import cv2
    g = np.load(GOLDEN)
    for name, subdir, ext, ms, al, sst in golden_calls(g):
        root = str(tmp_path / name)
        if not os.path.isdir(root):
            _golden_dir(g, name, root)
        video.Video(root).downscale_frames(subdir, ms, ext, align=al, short_side_target=sst)
        want = g[f"{name}/{subdir}"]
        for i, w in enumerate(want):
            fn = os.path.join(root, subdir, f"frame_{i:06d}.{ext}")
            if ext == "raw":
                h_, w_ = w.shape[:2]
                assert open(fn, "rb").read() == struct.pack("<iiiQ", h_, w_, 21, 12) + np.ascontiguousarray(w, np.float32).tobytes(), fn
            else:
                np.testing.assert_array_equal(cv2.imread(fn, cv2.IMREAD_UNCHANGED), w, err_msg=fn)


def test_downscale_all_end_to_end(tmp_path):
    """downscale_all on the fixture's process.py directory writes the reference's three outputs; lib_python then opens the directory
    and its "down" stream reads back the same floats.  A second call skips everything and changes no file."""
    import cv2
    g = np.load(GOLDEN)
    root = str(tmp_path / "v")
    _golden_dir(g, "45x33", root)
    stats = video.downscale_all(root)
    assert stats["outputs"] == ["color_down", "color_down_png", "color_flow"]
    for sub, ext in (("color_down", "raw"), ("color_down_png", "png"), ("color_flow", "png")):
        for i, want in enumerate(g[f"45x33/{sub}"]):
            fn = os.path.join(root, sub, f"frame_{i:06d}.{ext}")
            got = synthetic_files.read_raw(fn) if ext == "raw" else cv2.imread(fn, cv2.IMREAD_UNCHANGED)
            assert bits_equal(got, want) if ext == "raw" else np.array_equal(got, want), fn
    host = os.path.join(ROOT, "robust_cvd_b200", "host")
    if host not in sys.path:
        sys.path.insert(0, host)
    import lib_python as lp
    v = lp.DepthVideo()
    lp.DepthVideoImporter.importVideo(v, root, True)
    names = [v.colorStream(i).name() for i in range(v.numColorStreams())]
    down = names.index("down")
    for i, want in enumerate(g["45x33/color_down"]):
        assert bits_equal(v.colorFrame(down, i).image(), want)
    mtimes = {os.path.join(d, f): os.stat(os.path.join(root, d, f)).st_mtime_ns for d in ("color_down", "color_flow") for f in
              os.listdir(os.path.join(root, d))}
    assert video.downscale_all(root)["outputs"] == []
    assert mtimes == {k: os.stat(os.path.join(root, k)).st_mtime_ns for k in mtimes}


def test_chunks_and_one_output_skipped(tmp_path):
    """A directory read in many chunks (one frame each) writes what one chunk writes; an output that checks OK is left as it is while
    the others are written."""
    import cv2
    rng = np.random.default_rng(15)
    frames = rng.integers(0, 256, (5, 61, 97, 3), dtype=np.uint8)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    write_dir(a, frames)
    write_dir(b, frames)
    video.downscale_all(a, size=40, align=8)
    os.makedirs(os.path.join(b, "color_down_png"))
    for i in range(5):
        open(os.path.join(b, "color_down_png", f"frame_{i:06d}.png"), "wb").close()
    stats = video.downscale_all(b, size=40, align=8, chunk_bytes=1, workers=3)
    assert stats["outputs"] == ["color_down", "color_flow"]
    for i in range(5):
        for sub, ext in (("color_down", "raw"), ("color_flow", "png")):
            fn = f"{sub}/frame_{i:06d}.{ext}"
            x, y = os.path.join(a, fn), os.path.join(b, fn)
            if ext == "raw":
                assert open(x, "rb").read() == open(y, "rb").read()
            else:
                np.testing.assert_array_equal(cv2.imread(x), cv2.imread(y))
        assert os.path.getsize(os.path.join(b, "color_down_png", f"frame_{i:06d}.png")) == 0
    h, w = video.target_size(61, 97, 40, 8)
    raw, _ = cv2_outputs(frames[..., ::-1], h, w)
    for i in range(5):
        assert bits_equal(synthetic_files.read_raw(os.path.join(b, "color_down", f"frame_{i:06d}.raw")), raw[i])
