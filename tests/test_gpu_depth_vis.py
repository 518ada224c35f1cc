"""Depth visualisation on the GPU: rcvd_depth_visualize's order statistics against np.partition, its indices and pixels against the
numpy restatement tests/depth_vis_ref.py, visualize_depth_dir against the reference's own PNGs and arrays in
tests/golden/depth_vis_golden.npz (by decoded pixels), more than 65,535 frames in one call, more than one chunk with frames kept and read
again, the skip rule, and a 300-frame 384 x 224 directory end to end."""
import os

import numpy as np
import pytest

from tests import depth_vis_ref as ref
from robust_cvd_b200 import solver, visualization as vis
from robust_cvd_b200.png import png_rgb_bytes
from robust_cvd_b200.synthetic_files import write_raw
from robust_cvd_b200.video import _decode_png

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "depth_vis_golden.npz")


def _numpy_order_stats(frame, qs):
    """(n, [values at the ranks of both quantiles]) by np.partition of the finite values."""
    v = frame[np.isfinite(frame)].ravel() if frame.dtype == np.float32 else frame.ravel()
    if v.size == 0:
        return 0, None
    out = []
    for qf in qs:
        i0, i1, _ = vis._virtual_index(v.size, qf)
        s = v.copy()
        s.partition(np.unique([i0, i1]))
        out += [float(s[i0]), float(s[i1])]
    return v.size, out


def _check_range(frames, percentiles):
    dt = frames.dtype
    qs = [vis.quantile(p, dt) for p in percentiles]
    counts, stats = solver.depth_range(frames, [float(q) for q in qs])
    for f in range(frames.shape[0]):
        n, want = _numpy_order_stats(frames[f], qs)
        assert counts[f] == n, f
        if n:
            assert list(stats[f]) == want, (f, stats[f], want)


def _random_f32(rng, F, h, w):
    fr = rng.normal(0.5, 1.0, (F, h, w)).astype(np.float32)
    fr[:, ::7, ::5] = np.round(fr[:, ::7, ::5])   # ties
    if h >= 2 and w >= 4:
        fr[0, 0, :4] = [np.nan, np.inf, -np.inf, -0.0]
        fr[-1, 1, :3] = [0.0, -0.0, 1e30]
    if F > 2:
        fr[1] = np.nan
        fr[1, -1, -1] = 7.0   # n = 1
    return fr


def test_order_statistics_equal_np_partition():
    rng = np.random.default_rng(3)
    for F, h, w in ((5, 17, 23), (3, 224, 384), (2, 1, 1), (4, 61, 3)):
        fr = _random_f32(rng, F, h, w)
        for ps in ((0, 100), (2, 98), (37.5, 62.5), (50, 50), (0.001, 99.99)):
            _check_range(fr, ps)
        img = rng.integers(0, 256, (F, h, w, 3), dtype=np.uint8)
        img[0] = 9   # every value tied
        for ps in ((0, 100), (2, 98), (37.5, 62.5)):
            _check_range(img, ps)
    nan = np.full((2, 4, 5), np.nan, np.float32)
    counts, _ = solver.depth_range(nan, (0.0, 1.0))
    assert list(counts) == [0, 0]


def test_indices_and_pixels_equal_the_restatement():
    g = np.load(GOLDEN)
    _, lut_rgb = ref.tables(g["lut"])
    rng = np.random.default_rng(4)
    fr = _random_f32(rng, 6, 37, 29)
    fr[2] *= 1e6   # far outside the range: values wrap
    bounds = [(np.float32(-0.5), np.float32(1.5)), (np.float32(0.2), np.float32(0.2)), (np.float32(-2.0), 2.2250738585072014e-308),
              (1.7976931348623157e308, 2.2250738585072014e-308), (0, np.float32(3.0)), (0.1, 0.7), (np.float32(1.0), np.float32(-1.0))]
    for lo, hi in bounds:
        _, off, sc = vis.colour_bounds(np.float32, lo, hi)
        rgb, idx = solver.depth_colorize(fr, off, sc, lut_rgb, index=True)
        want = np.stack([ref.index(d, lo, hi) for d in fr])
        assert np.array_equal(idx, want), (lo, hi, np.argwhere(idx != want)[:5])
        assert np.array_equal(rgb, lut_rgb[want])
    img = rng.integers(0, 256, (4, 19, 13, 3), dtype=np.uint8)
    for lo, hi in [(np.float64(4.6), np.float64(251.0)), (88.0, 164.0), (np.float64(3.0), np.float64(3.0)), (0.0, 0.001)]:
        _, off, sc = vis.colour_bounds(np.uint8, lo, hi)
        rgb, idx = solver.depth_colorize(img, off, sc, lut_rgb, index=True)
        want = np.stack([ref.index(d, lo, hi) for d in img])
        assert np.array_equal(idx, want), (lo, hi)
        assert np.array_equal(rgb, lut_rgb[want])


def _write_inputs(src, names, arrays, ext):
    os.makedirs(src, exist_ok=True)
    for n, a in zip(names, arrays):
        if ext == ".raw":
            write_raw(os.path.join(src, n), a)
        else:
            with open(os.path.join(src, n), "wb") as f:
                f.write(png_rgb_bytes(a[..., ::-1]))


def test_golden_directories(tmp_path):
    g = np.load(GOLDEN)
    calls = 0
    for key in g.files:
        if not key.endswith("/args"):
            continue
        name, call = key.split("/")[:2]
        ext = str(g[f"{name}/ext"])
        names = [str(n) for n in g[f"{name}/names"]]
        arrays = [g[f"{name}/in_{k}"] for k in range(len(names))]
        src = str(tmp_path / name)
        if not os.path.isdir(src):
            _write_inputs(src, names, arrays, ext)
        lo, hi = (float(v) for v in g[key])
        dst = str(tmp_path / f"{name}_{call}")
        st = vis.visualize_depth_dir(src, dst, force=True, extension=ext, min_percentile=lo, max_percentile=hi, colormap=g["lut"])
        assert st["written"] == len(names)
        for k, n in enumerate(names):
            got = _decode_png(os.path.join(dst, os.path.splitext(n)[0] + ".png"))
            assert np.array_equal(got, g[f"{name}/{call}/png_{k}"]), (name, call, k)
            t64, _ = ref.tables(g["lut"])
            lo_, hi_ = ref.frame_range(arrays, lo, hi)
            vd = vis.visualize_depth(arrays[k], lo_, hi_, colormap=g["lut"])
            assert np.array_equal(vd, g[f"{name}/{call}/vis_{k}"]), (name, call, k)
        calls += 1
    assert calls == 12
    d = g["eval/depth"]
    assert np.array_equal(vis.visualize_depth(d, 0, d.max(), colormap=g["lut"]), g["eval/vis"])


def test_visualize_depth_defaults_include_inf():
    g = np.load(GOLDEN)
    t64, _ = ref.tables(g["lut"])
    d = np.linspace(-1, 3, 60, dtype=np.float32).reshape(6, 10)
    d[0, 0], d[1, 1] = np.nan, np.inf
    assert np.array_equal(vis.visualize_depth(d, colormap=g["lut"]), t64[ref.index(d, np.nanmin(d), np.nanmax(d))])


def test_more_than_65535_frames_in_one_call():
    rng = np.random.default_rng(5)
    fr = rng.uniform(-1, 2, (70_000, 3, 5)).astype(np.float32)
    fr[69_999, 0, 0] = np.nan
    _, lut = ref.tables(np.load(GOLDEN)["lut"])
    rgb, idx = solver.depth_colorize(fr, 0.0, 1.0, lut, index=True)
    assert np.array_equal(idx, ref.index(fr.reshape(-1, 5), np.float32(0.0), np.float32(1.0)).reshape(fr.shape))
    assert np.array_equal(rgb, lut[idx])
    _check_range(fr[-300:], (2, 98))
    counts, _ = solver.depth_range(fr, (0.0, 1.0))
    assert counts[69_999] == 14 and (counts[:69_999] == 15).all()


def test_chunks_kept_and_read_again_and_skip_rule(tmp_path):
    g = np.load(GOLDEN)
    rng = np.random.default_rng(6)
    frames = [rng.uniform(0.1, 2.0, (24, 40)).astype(np.float32) for _ in range(9)] + [rng.uniform(0, 1, (10, 7)).astype(np.float32)]
    names = [f"frame_{i:06d}.raw" for i in range(10)]
    src = str(tmp_path / "depth")
    _write_inputs(src, names, frames, ".raw")
    _, _, want = ref.visualize_dir(frames, 2, 98, g["lut"])
    outs = {}
    for tag, kw in (("kept", {}), ("reread", dict(resident_bytes=0))):
        dst = str(tmp_path / tag)
        st = vis.visualize_depth_dir(src, dst, force=True, min_percentile=2, max_percentile=98, colormap=g["lut"], chunk_bytes=8000, **kw)
        assert st["resident"] == (tag == "kept") and st["written"] == 10
        outs[tag] = [_decode_png(os.path.join(dst, n.replace(".raw", ".png")))[..., ::-1] for n in names]
        assert all(np.array_equal(a, b) for a, b in zip(outs[tag], want)), tag
    # without force, existing outputs are kept and the others written; with every output present nothing runs
    dst = str(tmp_path / "kept")
    os.remove(os.path.join(dst, "frame_000003.png"))
    with open(os.path.join(dst, "frame_000005.png"), "wb") as f:
        f.write(b"stale")
    st = vis.visualize_depth_dir(src, dst, min_percentile=2, max_percentile=98, colormap=g["lut"])
    assert st["written"] == 1
    assert open(os.path.join(dst, "frame_000005.png"), "rb").read() == b"stale"
    assert np.array_equal(_decode_png(os.path.join(dst, "frame_000003.png"))[..., ::-1], want[3])
    assert vis.visualize_depth_dir(src, dst, colormap=g["lut"]) is None


def test_300_frame_directory_end_to_end(tmp_path):
    g = np.load(GOLDEN)
    rng = np.random.default_rng(7)
    frames = []
    for i in range(300):
        d = (rng.uniform(0.2, 1.0, (224, 384)) * (1 + 0.002 * i)).astype(np.float32)
        d[rng.integers(0, 224, 40), rng.integers(0, 384, 40)] = np.nan
        frames.append(d)
    names = [f"frame_{i:06d}.raw" for i in range(300)]
    src = str(tmp_path / "depth")
    _write_inputs(src, names, frames, ".raw")
    st = vis.visualize_depth_dir(src, src, force=True, colormap=g["lut"])
    assert st["written"] == 300
    _, _, want = ref.visualize_dir(frames, 0, 100, g["lut"])
    for i, n in enumerate(names):
        assert np.array_equal(_decode_png(os.path.join(src, n.replace(".raw", ".png")))[..., ::-1], want[i]), i
