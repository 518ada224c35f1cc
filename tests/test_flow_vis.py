"""Flow visualisations without a GPU: the CPU restatement (tests/flow_vis_ref.py) against the reference's own outputs
(tests/golden/flow_vis_golden.npz, written by tests/golden/make_flow_vis_golden.py from the reference's Flow.visualize_flow), the
8-bit conversion against cv2's, the RGB PNG encoder, the file semantics of robust_cvd_b200.flow.visualize_flow (names, skip rule, input
checks) and the refusals of rcvd_flow_visualize, which all happen before a device is needed."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import flow_vis_ref as ref  # noqa: E402
from robust_cvd_b200 import abi, flow, solver, synthetic_files  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "flow_vis_golden.npz")
CASES = {"9x13": [(0, 1), (1, 2), (0, 2)], "11x7": [(0, 2), (1, 2)]}      # sorted pairs of each golden directory


def golden_pair(g, name, i, j):
    """Inputs of pair (i, j) of a golden case: colour i, colour j, flow_ij, flow_ji, mask_ij, mask_ji."""
    return (g[f"{name}/color/{i}"], g[f"{name}/color/{j}"], g[f"{name}/flow/{i}_{j}"], g[f"{name}/flow/{j}_{i}"],
            g[f"{name}/mask/{i}_{j}"], g[f"{name}/mask/{j}_{i}"])


def golden_pngs(g, name, i, j):
    """The reference's decoded PNGs of pair (i, j) in cv2's array channel order: vis, warp i_j, warp j_i."""
    return (g[f"{name}/vis_flow/frame_{i:06d}_{j:06d}.png"], g[f"{name}/vis_flow_warped/frame_{i:06d}_{j:06d}_warped.png"],
            g[f"{name}/vis_flow_warped/frame_{j:06d}_{i:06d}_warped.png"])


def test_fixture_records_numpy_2_dtypes():
    """The dtypes the restatement assumes are the ones the reference got: float64 normalised flow (NEP 50), a float64 composite and
    float32 warps handed to cv2.imwrite."""
    g = np.load(GOLDEN)
    assert int(str(g["numpy_version"]).split(".")[0]) >= 2
    assert str(g["dtype/normalised_uv"]) == "float64" and str(g["dtype/flow_image"]) == "uint8"
    assert str(g["dtype/vis_flow"]) == "float64" and str(g["dtype/vis_flow_warped"]) == "float32"
    assert str(g["dtype/warp_values"]) == "float32"


@pytest.mark.parametrize("name", list(CASES))
def test_flow_images_match_reference_golden(name):
    """flow_to_image and the normalised (u, v) bit for bit, for every flow: NaN (negated by max(-1, nan)), all-zero (divided by eps),
    unknown and ordinary flows."""
    g = np.load(GOLDEN)
    for key in [k for k in g.files if k.startswith(f"{name}/flow/")]:
        ab = key.rsplit("/", 1)[1]
        img, st = ref.flow_image(g[key])
        np.testing.assert_array_equal(img, g[f"{name}/flow_image/{ab}"], err_msg=key)
        assert np.array_equal(st["u"], g[f"{name}/u/{ab}"], equal_nan=True) and np.array_equal(st["v"], g[f"{name}/v/{ab}"], equal_nan=True)


@pytest.mark.parametrize("name", list(CASES))
def test_composite_and_warps_match_reference_golden(name):
    """The composite and the warp PNGs bit for bit; the warp values within WARP_TOL of torch's CPU grid_sample (the reference's device
    on a machine without a GPU)."""
    g = np.load(GOLDEN)
    differ = 0
    for i, j in CASES[name]:
        out = ref.visualize_pair(*golden_pair(g, name, i, j))
        vis, wij, wji = golden_pngs(g, name, i, j)
        np.testing.assert_array_equal(out["vis"], vis)
        np.testing.assert_array_equal(out["warp_ij"], wij)
        np.testing.assert_array_equal(out["warp_ji"], wji)
        for got, key in ((out["warp_values_ij"], f"{i}_{j}"), (out["warp_values_ji"], f"{j}_{i}")):
            want = g[f"{name}/warp_values/{key}"]
            assert np.all(np.abs(got - want) <= ref.WARP_TOL * (1 + np.abs(want)))
            differ += int((got != want).sum())
    print(f"{name}: {differ} warp values differ from torch's CPU grid_sample in their last bits")


def test_golden_covers_the_edge_cases():
    g = np.load(GOLDEN)
    stats = [ref.flow_stats(g[k]) for k in g.files if "/flow/" in k]
    assert any(s[1] for s in stats)                                   # a NaN flow: divided by -1 + eps
    assert any(s[0] == 0 and not s[1] for s in stats)                 # an all-zero flow: divided by eps
    assert any(s[2].any() for s in stats)                             # unknown pixels
    flows = [g[k] for k in g.files if "/flow/" in k]
    assert any(np.isinf(f).any() for f in flows) and any((np.abs(f) == 1e7).any() for f in flows)
    for k in (k for k in g.files if "/flow/" in k):
        f, (H, W) = g[k], g[k].shape[:2]
        X, Y = np.arange(W) + f[..., 0], np.arange(H)[:, None] + f[..., 1]
        if np.isfinite(f).all() and (f != 0).any():
            assert (X == 0).any() and (X == W - 1).any() and (Y == 0).any() and (Y == H - 1).any() and (X > W).any()
    masks = [g[k] for k in g.files if "/mask/" in k]
    assert all(0 < (m > 0).mean() < 1 for m in masks) and any(((m > 0) & (m < 255)).any() for m in masks)
    sizes = {g[k].shape[:2] for k in g.files if "/flow/" in k}
    assert all(h != w and h % 2 and w % 2 for h, w in sizes)
    # every branch of the colouring: inside and outside the unit disc, and the wheel's wrap k1 = 56 -> 1
    st = [ref.flow_image(g[k])[1] for k in g.files if "/flow/" in k]
    rads = np.concatenate([np.hypot(s["u"], s["v"]).ravel() for s in st])
    assert (rads <= 1).any() and (rads > 1).any()
    ang = np.concatenate([np.arctan2(-np.nan_to_num(s["v"]), -np.nan_to_num(s["u"])).ravel() for s in st])
    assert (ang == np.pi).any()                                       # fk = 55: k1 = 56 wraps to 1


def test_to_u8_is_cv2_imwrite(tmp_path):
    """cv2.imwrite's conversion of float images: round half to even, saturation, and 0 for NaN and for values beyond int32."""
    import cv2
    vals = np.array([0.5, 1.5, 2.5, 254.5, 255.5, 255.49, -0.5, -0.51, -3, 300, 1e10, -1e10, np.inf, -np.inf, np.nan, 76.5, 127.5,
                     2147483647.0, 2147483648.0, 1e-300], np.float64)
    for dt in (np.float64, np.float32):
        img = np.repeat(vals.astype(dt)[None, :, None], 3, axis=2)
        fn = str(tmp_path / f"v_{np.dtype(dt).name}.png")
        assert cv2.imwrite(fn, img)
        np.testing.assert_array_equal(cv2.imread(fn, cv2.IMREAD_UNCHANGED)[0, :, 0], ref.to_u8(vals.astype(dt)), err_msg=str(dt))


def test_rgb_png_encoder_round_trip(tmp_path):
    import cv2
    rng = np.random.default_rng(7)
    for h, w in ((1, 1), (7, 5), (448, 1536)):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        fn = str(tmp_path / f"c_{h}_{w}.png")
        with open(fn, "wb") as f:
            f.write(flow.png_rgb_bytes(img))
        np.testing.assert_array_equal(cv2.imread(fn, cv2.IMREAD_UNCHANGED), img[..., ::-1])     # cv2 returns BGR
    with pytest.raises(ValueError):
        flow.png_rgb_bytes(np.zeros((3, 4), np.uint8))


def _write_dir(root, frames, pairs, h=6, w=9, seed=0):
    rng = np.random.default_rng(seed)
    for d in ("flow", "flow_mask", "color_down"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for f in frames:
        synthetic_files.write_raw(os.path.join(root, flow.COLOR_FMT.format(f)), rng.random((h, w, 3)).astype(np.float32))
    for i, j in pairs:
        for a, b in ((i, j), (j, i)):
            synthetic_files.write_raw(os.path.join(root, flow.FLOW_FMT.format(a, b)), rng.normal(0, 1, (h, w, 2)).astype(np.float32))
            synthetic_files.write_png_gray(os.path.join(root, flow.MASK_FMT.format(a, b)), (rng.random((h, w)) < 0.5).astype(np.uint8) * 255)


def test_names_and_skip_rule(tmp_path):
    """Every flow/ entry is parsed and sorted to (i, j); a pair is skipped when its composite exists and, with warp, its sorted-index
    warp exists; a name that does not parse is refused."""
    root = str(tmp_path)
    _write_dir(root, [0, 1, 2, 3], [(0, 1), (2, 1), (3, 0)])
    assert flow.vis_pairs_to_compute(root) == [(0, 1), (0, 3), (1, 2)]
    os.makedirs(os.path.join(root, "vis_flow")); os.makedirs(os.path.join(root, "vis_flow_warped"))
    open(os.path.join(root, flow.VIS_FMT.format(0, 1)), "wb").close()
    open(os.path.join(root, flow.VIS_FMT.format(1, 2)), "wb").close()
    open(os.path.join(root, flow.WARP_FMT.format(2, 1)), "wb").close()     # the reverse-index warp does not count
    assert flow.vis_pairs_to_compute(root) == [(0, 3)]
    assert flow.vis_pairs_to_compute(root, warp=True) == [(0, 1), (0, 3), (1, 2)]
    open(os.path.join(root, flow.WARP_FMT.format(1, 2)), "wb").close()
    assert flow.vis_pairs_to_compute(root, warp=True) == [(0, 1), (0, 3)]
    for bad in ("notes.txt", "flow_1.raw", "flow_a_2.raw", "flow_1_2_3.raw"):
        open(os.path.join(root, "flow", bad), "wb").close()
        with pytest.raises(ValueError, match="not a flow"):
            flow.vis_pairs_to_compute(root)
        os.remove(os.path.join(root, "flow", bad))


def test_input_checks(tmp_path):
    """A missing reverse flow, mask or colour, and a size mismatch, are refused; nothing is written."""
    root = str(tmp_path)
    _write_dir(root, [0, 1, 2], [(0, 1), (1, 2)])
    flow._check_vis_inputs(root, [(0, 1), (1, 2)])
    for fn in (flow.FLOW_FMT.format(2, 1), flow.MASK_FMT.format(1, 0), flow.COLOR_FMT.format(2)):
        full = os.path.join(root, fn)
        keep = open(full, "rb").read()
        os.remove(full)
        with pytest.raises(FileNotFoundError, match="is missing"):
            flow._check_vis_inputs(root, flow.vis_pairs_to_compute(root))
        open(full, "wb").write(keep)
    synthetic_files.write_png_gray(os.path.join(root, flow.MASK_FMT.format(2, 1)), np.zeros((6, 8), np.uint8))
    with pytest.raises(ValueError, match="differ in size"):
        flow._check_vis_inputs(root, [(1, 2)])
    _write_dir(str(tmp_path / "thin"), [0, 1], [(0, 1)], h=5, w=1)
    with pytest.raises(ValueError, match="divides by width - 1"):
        flow._check_vis_inputs(str(tmp_path / "thin"), [(0, 1)])
    assert not os.path.exists(os.path.join(root, "vis_flow"))


def test_abi_refusals_need_no_device():
    """Every refusal of rcvd_flow_visualize happens on the host: on a machine without a GPU it still returns RCVD_ERR_INVALID (not
    RCVD_ERR_NO_DEVICE), and zero pairs return RCVD_OK."""
    L = solver.lib()
    H, W = 4, 5
    colors = np.zeros((2, H, W, 3), np.float32); fl = np.zeros((1, H, W, 2), np.float32); m = np.zeros((1, H, W), np.uint8)
    vis = np.full((1, 2 * H, 4 * W, 3), 77, np.uint8); wa = np.full((1, H, W, 3), 77, np.uint8); wb = wa.copy()
    pf = np.array([[0, 1]], np.int32)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    good = dict(width=W, height=H, num_pairs=1, num_frames=2, warp=1)

    def call(prm, args=None):
        args = args or [P(pf, C.c_int32), P(fl, C.c_float), P(fl, C.c_float), P(m, C.c_uint8), P(m, C.c_uint8), P(colors, C.c_float),
                        P(vis, C.c_uint8), P(wa, C.c_uint8), P(wb, C.c_uint8)]
        return L.rcvd_flow_visualize(prm, 0, *args, None, None, None)
    bad = [dict(width=1), dict(height=1), dict(width=0), dict(num_pairs=-1), dict(num_frames=0), dict(width=1 << 14, height=1 << 14),
           dict(num_frames=1)]                                                # the last: pair frame 1 out of range
    for over in bad:
        assert call(C.byref(abi.FlowVisParams(**{**good, **over}))) == abi.ERR_INVALID, over
    assert call(None) == abi.ERR_INVALID
    prm = abi.FlowVisParams(**good)
    for k in range(9):
        args = [P(pf, C.c_int32), P(fl, C.c_float), P(fl, C.c_float), P(m, C.c_uint8), P(m, C.c_uint8), P(colors, C.c_float),
                P(vis, C.c_uint8), P(wa, C.c_uint8), P(wb, C.c_uint8)]
        args[k] = None
        assert call(C.byref(prm), args) == abi.ERR_INVALID, k
    neg = np.array([[-1, 0]], np.int32)
    assert call(C.byref(prm), [P(neg, C.c_int32), P(fl, C.c_float), P(fl, C.c_float), P(m, C.c_uint8), P(m, C.c_uint8),
                               P(colors, C.c_float), P(vis, C.c_uint8), P(wa, C.c_uint8), P(wb, C.c_uint8)]) == abi.ERR_INVALID
    assert np.all(vis == 77) and np.all(wa == 77) and np.all(wb == 77)
    empty = abi.FlowVisParams(**{**good, "num_pairs": 0})
    assert L.rcvd_flow_visualize(C.byref(empty), 0, *([None] * 12)) == abi.OK
    with pytest.raises(ValueError):
        solver.flow_visualize(colors, pf, fl, fl, m, np.zeros((1, H, W + 1), np.uint8))


def test_no_device_fails_loudly(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        flow.visualize_flow(str(tmp_path))
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        flow.Flow(str(tmp_path), str(tmp_path)).visualize_flow(warp=True)
    assert os.listdir(tmp_path) == []
