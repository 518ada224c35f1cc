"""Depth visualisation without a GPU: the numpy restatement tests/depth_vis_ref.py against the reference's own outputs
(tests/golden/depth_vis_golden.npz, written by tests/golden/make_depth_vis_golden.py from the reference's visualize_depth_dir and
visualize_depth), the host's percentile interpolation against np.percentile, the u8 cast and gray conversion the kernels restate, the
colour bounds' types, the skip rule's early returns, every refusal of robust_cvd_b200.visualization (all before anything is written),
the colormap resolution and the refusals of rcvd_depth_visualize, which need no device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tests import depth_vis_ref as ref
from robust_cvd_b200 import abi, solver, visualization as vis
from robust_cvd_b200.png import png_gray_bytes, png_rgb_bytes
from robust_cvd_b200.synthetic_files import write_raw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "depth_vis_golden.npz")


def golden_calls(g):
    """(directory, call, extension, [input arrays], (min_percentile, max_percentile)) of every call in the fixture."""
    for key in g.files:
        if key.endswith("/args"):
            name, call = key.split("/")[:2]
            n = len(g[f"{name}/names"])
            yield name, call, str(g[f"{name}/ext"]), [g[f"{name}/in_{k}"] for k in range(n)], tuple(float(v) for v in g[key])


def test_restatement_matches_reference_golden():
    g = np.load(GOLDEN)
    lut = g["lut"]
    t64, _ = ref.tables(lut)
    calls = 0
    for name, call, ext, frames, (lo, hi) in golden_calls(g):
        d_min, d_max, rgb = ref.visualize_dir(frames, lo, hi, lut)
        assert [type(d_min).__name__, type(d_max).__name__] == list(g[f"{name}/{call}/bounds_type"]), (name, call)
        assert np.float64(d_min) == g[f"{name}/{call}/d_min"] and np.float64(d_max) == g[f"{name}/{call}/d_max"], (name, call)
        for k, d in enumerate(frames):
            vis_ref = g[f"{name}/{call}/vis_{k}"]
            assert vis_ref.dtype == np.float64
            assert np.array_equal(t64[ref.index(d, d_min, d_max)], vis_ref), (name, call, k)
            assert np.array_equal(rgb[k], g[f"{name}/{call}/png_{k}"][..., ::-1]), (name, call, k)
        calls += 1
    assert calls == 12
    d = g["eval/depth"]
    assert np.array_equal(t64[ref.index(d, 0, d.max())], g["eval/vis"])


def test_golden_covers_the_cases():
    """Wrapped values, a frame without a finite value, Python's start value kept as d_max, a zero range, mixed sizes and the .png branch
    are all in the fixture."""
    g = np.load(GOLDEN)
    assert not np.isfinite(g["nonfinite/in_1"]).any() and (~np.isfinite(g["nonfinite/in_0"])).sum() == 3
    assert list(g["negative/p0_100/bounds_type"]) == ["float32", "float"] and g["negative/p0_100/d_max"] == sys.float_info.min
    assert g["constant/p0_100/d_min"] == g["constant/p0_100/d_max"]
    assert {g[f"mixed/in_{k}"].shape for k in range(3)} == {(31, 17), (9, 16)} and "frame_000001.RAW" in list(g["mixed/names"])
    assert str(g["png/ext"]) == ".png" and g["png/in_0"].dtype == np.uint8
    lo, hi = g["mixed/p37_62/d_min"].astype(np.float32), g["mixed/p37_62/d_max"].astype(np.float32)
    assert ((g["mixed/in_1"] - lo) / (hi - lo) > 1.01).any(), "values above the range wrap"


def test_host_interpolation_is_np_percentile():
    """percentile_from_ranks on the order statistics at _virtual_index's ranks equals np.percentile bit for bit, for float32 and u8
    values: ties, n = 1, +-0.0, fractional percentiles."""
    rng = np.random.default_rng(11)
    qs = [0, 100, 2, 98, 37.5, 62.5, 50, 33.333333, 99.99, 0.001]
    arrays = [np.array([1.5], np.float32), np.array([7], np.uint8), np.array([-0.0, 0.0, -0.0, 0.0], np.float32),
              np.array([0.0, -0.0], np.float32), np.full(10, 3.25, np.float32), np.array([1, 1, 2, 2, 2, 3], np.float32)]
    for n in (2, 3, 7, 100, 1001, 86016):
        arrays.append(rng.normal(0, 1, n).astype(np.float32))
        arrays.append(rng.integers(-3, 3, n).astype(np.float32))
        arrays.append(rng.integers(0, 256, n).astype(np.uint8))
    arrays.append(np.array([-3e38, 3e38], np.float32))
    checked = 0
    for a in arrays:
        for p in qs + [float(v) for v in rng.uniform(0, 100, 5)]:
            want = np.percentile(a, p)
            qf = vis.quantile(p, a.dtype)
            i0, i1, _ = vis._virtual_index(a.size, qf)
            s = a.copy()
            s.partition(np.unique([0, a.size - 1, i0, i1]))
            got = vis.percentile_from_ranks(a.size, qf, float(s[i0]), float(s[i1]), a.dtype)
            assert type(got) is type(want), (a.dtype, p)
            assert np.asarray(got).tobytes() == np.asarray(want).tobytes(), (a[:4], p, got, want)
            checked += 1
    assert checked > 300


def test_uint8_cast_and_gray_semantics():
    """The kernels' cast rule (NaN, +-inf and |x| >= 2^31 give 0, other values truncate and wrap modulo 256) and gray conversion are
    numpy's and cv2's on this host."""
    x = [np.nan, np.inf, -np.inf, 1e10, -1.0, 256.0, 300.5, 255.9, -0.5, 2.0 ** 31 + 5, -2.0 ** 31 - 7, 12345.7]
    want = [0, 0, 0, 0, 255, 0, 44, 255, 0, 0, 0, 57]
    with np.errstate(invalid="ignore"):
        assert list(np.uint8(np.array(x, np.float64))) == want
        assert list(np.uint8(np.array(x[:9] + [12345.7], np.float32))) == want[:9] + [57]
    cv2 = pytest.importorskip("cv2")
    v = np.arange(256, dtype=np.uint8)
    bgr = np.stack(np.meshgrid(v, v, v, indexing="ij"), -1).reshape(4096, 4096, 3)
    assert np.array_equal(ref.gray(bgr), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY))
    g = np.load(GOLDEN)
    img = g["png/in_0"]
    assert np.array_equal(cv2.applyColorMap(img, g["lut"].reshape(256, 1, 3)), g["lut"][ref.gray(img)])


def test_colour_tables_and_colormaps():
    g = np.load(GOLDEN)
    t64, rgb = vis.color_tables(g["lut"])
    r64, rrgb = ref.tables(g["lut"])
    assert np.array_equal(t64, r64) and np.array_equal(rgb, rrgb)
    assert np.array_equal(vis.resolve_colormap(g["lut"].reshape(256, 1, 3)), g["lut"])
    for bad in (g["lut"][:255], g["lut"].astype(np.int32), np.zeros((256, 1), np.uint8)):
        with pytest.raises(ValueError, match="colormap"):
            vis.resolve_colormap(bad)
    cv2 = pytest.importorskip("cv2")
    t = vis.resolve_colormap(cv2.COLORMAP_MAGMA)
    img = np.arange(256, dtype=np.uint8).reshape(16, 16)
    assert np.array_equal(t[img], cv2.applyColorMap(img, cv2.COLORMAP_MAGMA))


def test_default_colormap_needs_the_reference_module(tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "utils", None)
    with pytest.raises(RuntimeError, match="colormap="):
        vis.resolve_colormap(None)
    src = tmp_path / "depth"
    src.mkdir()
    write_raw(str(src / "frame_000000.raw"), np.ones((4, 5), np.float32))
    with pytest.raises(RuntimeError, match="colormap="):
        vis.visualize_depth_dir(str(src), str(tmp_path / "out"))
    assert not (tmp_path / "out").exists()
    with pytest.raises(RuntimeError, match="colormap="):
        vis.visualize_depth(np.ones((4, 5), np.float32))


def test_colour_bounds_follow_numpy_types():
    f32, u8 = np.float32, np.uint8
    assert vis.colour_bounds(f32, np.float32(0.25), np.float32(2.0)) == (0, 0.25, 1.75)
    assert vis.colour_bounds(f32, 0, np.float32(2.5)) == (0, 0.0, 2.5)
    k, off, sc = vis.colour_bounds(f32, np.float32(-2.0), sys.float_info.min)   # weak Python float: 2.2e-308 is 0 in float32
    assert (k, off, sc) == (0, -2.0, 2.0)
    k, off, sc = vis.colour_bounds(f32, sys.float_info.max, sys.float_info.min)
    assert k == 0 and off == np.inf and sc == -np.inf
    k, off, sc = vis.colour_bounds(f32, 0.1, 0.7)   # both Python floats: the difference is taken in double, then rounded
    assert off == float(np.float32(0.1)) and sc == float(np.float32(0.7 - 0.1)) != float(np.float32(0.7) - np.float32(0.1))
    assert vis.colour_bounds(u8, np.float64(4.6), np.float64(251.0)) == (1, 4.6, 251.0 - 4.6)
    for dt, lo, hi in ((f32, np.float64(0), 1.0), (u8, 0, 255), (u8, np.float32(1), np.float32(3)), (np.float64, 0.0, 1.0)):
        with pytest.raises(ValueError):
            vis.colour_bounds(dt, lo, hi)
    with pytest.raises(ValueError):
        vis.visualize_depth(np.ones((3, 4), np.float64), 0.0, 1.0, colormap=np.zeros((256, 3), np.uint8))


def _dir_with(tmp_path, files):
    src = tmp_path / "src"
    src.mkdir(exist_ok=True)
    for name, data in files.items():
        (src / name).write_bytes(data) if isinstance(data, bytes) else write_raw(str(src / name), data)
    return str(src)


def test_skip_rule_early_returns(tmp_path):
    lut = np.zeros((256, 3), np.uint8)
    src = _dir_with(tmp_path, {"a.txt": b"x", "frame_000000.raw": np.ones((3, 4), np.float32)})
    dst = tmp_path / "dst"
    dst.mkdir()
    assert vis.visualize_depth_dir(src, str(dst), extension=".exr", colormap=lut) is None
    (dst / "frame_000000.png").write_bytes(b"kept")
    assert vis.visualize_depth_dir(src, str(dst), colormap=lut) is None
    assert (dst / "frame_000000.png").read_bytes() == b"kept"
    assert sorted(os.listdir(dst)) == ["frame_000000.png"]


def test_refusals_before_anything_is_written(tmp_path):
    lut = np.zeros((256, 3), np.uint8)
    ok = np.ones((3, 4), np.float32)
    cases = [
        ({"frame_000000.raw": ok, "frame_000001.raw": np.ones((3, 4, 2), np.float32)}, ".raw", "single-channel float32"),
        ({"frame_000000.raw": ok, "frame_000001.raw": np.ones((3, 4), np.float64)}, ".raw", "single-channel float32"),
        ({"frame_000000.raw": ok, "frame_000001.raw": b"short"}, ".raw", "not a .raw"),
        ({"a.png": png_rgb_bytes(np.zeros((3, 4, 3), np.uint8)), "b.png": b"\xff\xd8\xff\xe0 a jpeg"}, ".png", "cannot be read"),
        ({"a.png": png_gray_bytes(np.zeros((3, 4), np.uint8)),
          "b.png": png_gray_bytes(np.zeros((3, 4), np.uint8))[:16] + b"\0\0\0\3\0\0\0\4\x10" + b"\0" * 20}, ".png", "cannot be read"),
    ]
    for k, (files, ext, msg) in enumerate(cases):
        src = _dir_with(tmp_path / str(k), files) if (tmp_path / str(k)).mkdir() is None else None
        dst = tmp_path / str(k) / "dst"
        with pytest.raises(ValueError, match=msg):
            vis.visualize_depth_dir(src, str(dst), extension=ext, colormap=lut)
        assert not dst.exists(), k
    src = _dir_with(tmp_path, {"frame_000000.raw": ok})
    for lo, hi in ((-1, 100), (0, 100.5)):
        with pytest.raises(ValueError, match="Percentiles"):
            vis.visualize_depth_dir(src, str(tmp_path / "dst"), min_percentile=lo, max_percentile=hi, colormap=lut)
    assert not (tmp_path / "dst").exists()


def test_no_device_fails_loudly(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lut = np.zeros((256, 3), np.uint8)
    src = _dir_with(tmp_path, {"frame_000000.raw": np.ones((3, 4), np.float32)})
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        vis.visualize_depth_dir(src, str(tmp_path / "dst"), colormap=lut)
    assert not (tmp_path / "dst").exists()
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        vis.visualize_depth(np.ones((3, 4), np.float32), colormap=lut)


def test_abi_refusals_need_no_device():
    """Every refusal of rcvd_depth_visualize happens on the host: on a machine without a GPU it still returns RCVD_ERR_INVALID (not
    RCVD_ERR_NO_DEVICE), and zero frames return RCVD_OK."""
    L = solver.lib()
    fr = np.zeros((2, 5, 7), np.float32)
    lut = np.zeros((256, 3), np.uint8)
    counts, stats = np.full(2, 7, np.int64), np.full((2, 4), 7.0)
    rgb = np.full((2, 5, 7, 3), 7, np.uint8)

    def prm(**over):
        q = dict(width=7, height=5, num_frames=2, kind=abi.DEPTH_VIS_F32, offset=0.0, scale=1.0)
        qv = over.pop("q", (0.0, 1.0))
        q.update(over)
        p = abi.DepthVisParams(**q)
        p.q[0], p.q[1] = qv
        return C.byref(p)
    frp, lp = C.c_void_p(fr.ctypes.data), lut.ctypes.data_as(C.POINTER(C.c_uint8))
    cp, sp = counts.ctypes.data_as(C.POINTER(C.c_int64)), stats.ctypes.data_as(C.POINTER(C.c_double))
    rp = rgb.ctypes.data_as(C.POINTER(C.c_uint8))
    bad = [dict(width=0), dict(height=-1), dict(width=1 << 15, height=1 << 15), dict(num_frames=-1), dict(kind=2), dict(q=(-0.1, 1.0)),
           dict(q=(0.0, 1.5)), dict(q=(float("nan"), 1.0))]
    for over in bad:
        assert L.rcvd_depth_visualize(prm(**over), 0, frp, lp, cp, sp, None, rp) == abi.ERR_INVALID, over
    assert L.rcvd_depth_visualize(None, 0, frp, lp, cp, sp, None, rp) == abi.ERR_INVALID
    assert L.rcvd_depth_visualize(prm(), 0, None, lp, cp, sp, None, rp) == abi.ERR_INVALID
    assert L.rcvd_depth_visualize(prm(), 0, frp, lp, cp, None, None, None) == abi.ERR_INVALID
    assert L.rcvd_depth_visualize(prm(), 0, frp, lp, None, sp, None, None) == abi.ERR_INVALID
    assert L.rcvd_depth_visualize(prm(), 0, frp, None, None, None, None, rp) == abi.ERR_INVALID
    assert np.all(counts == 7) and np.all(stats == 7.0) and np.all(rgb == 7)
    assert L.rcvd_depth_visualize(prm(num_frames=0), 0, None, lp, cp, sp, None, rp) == abi.OK
    a, b = C.c_double(), C.c_double()
    assert L.rcvd_debug_time_depth_visualize(prm(), 0, frp, lp, 0, C.byref(a), C.byref(b)) == abi.ERR_INVALID
    assert L.rcvd_debug_time_depth_visualize(prm(), 0, frp, None, 1, C.byref(a), C.byref(b)) == abi.ERR_INVALID
    with pytest.raises(ValueError):
        solver.depth_range(np.zeros((2, 5, 7), np.float64), (0.0, 1.0))
    with pytest.raises(ValueError):
        solver.depth_colorize(np.zeros((2, 5, 7, 2), np.uint8), 0.0, 1.0, lut)
    with pytest.raises(ValueError):
        solver.depth_colorize(fr, 0.0, 1.0)
