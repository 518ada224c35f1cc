"""Flow visualisations on the GPU (csrc/rcvd_flowvis.cuh, rcvd_flow_visualize, robust_cvd_b200.flow.visualize_flow) against the CPU
restatement (tests/flow_vis_ref.py), the reference's own golden outputs and torch's CUDA grid_sample.

Stated bounds:
  * composite bytes equal the restatement's and the fixture's, except in the flow tiles at pixels whose colour changes when atan2's
    result moves by 4 ulps (flow_vis_ref.flow_image_margin): CUDA's float64 atan2 is within 2 ulps of the correctly rounded value, not
    equal to numpy's.  Every other step is the reference's IEEE arithmetic.  The tests report the margin pixels and the pixels that
    differ, and require no difference outside the margin;
  * warp values within WARP_TOL (1 + |v|) of torch.nn.functional.grid_sample on this GPU (the reference's own device path), and warp
    bytes equal outside the margin of WARP_TOL around a half-way point."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import flow_vis_ref as ref  # noqa: E402
from tests.test_flow_vis import CASES, GOLDEN, golden_pair, golden_pngs  # noqa: E402
from robust_cvd_b200 import abi, flow, solver, synthetic, synthetic_files  # noqa: E402

pytestmark = pytest.mark.gpu


def launches():
    L = solver.lib()
    L.rcvd_flow_vis_launch_count.restype = C.c_int64
    return L.rcvd_flow_vis_launch_count()


def allowed_vis_mismatch(margin_ij, margin_ji):
    """[2H, 4W] bool: the flow-tile pixels (both rows) that may differ."""
    H, W = margin_ij.shape
    out = np.zeros((2 * H, 4 * W), bool)
    for r in (0, H):
        out[r:r + H, 2 * W:3 * W] = margin_ij
        out[r:r + H, 3 * W:] = margin_ji
    return out


def check_pair(got_vis, got_wij, got_wji, got_values, inputs, want_vis=None, want_wij=None, want_wji=None):
    """One pair's GPU outputs (PNG byte order) against the restatement, torch's CUDA warp and optional golden PNGs (cv2 array order).
    Returns (composite margin pixels, composite pixels that differ, warp values differing from torch's, warp margin pixels)."""
    ci, cj, fij, fji, mij, mji = inputs
    r = ref.visualize_pair(ci, cj, fij, fji, mij, mji)
    allowed = allowed_vis_mismatch(ref.flow_image_margin(fij), ref.flow_image_margin(fji))
    vis = got_vis[..., ::-1]                                            # PNG order -> cv2's array order
    vdiff = 0
    for want in (r["vis"], want_vis):
        if want is not None:
            bad = (vis != want).any(axis=-1)
            assert not (bad & ~allowed).any(), f"{int((bad & ~allowed).sum())} composite pixels differ outside the margin"
            vdiff = max(vdiff, int(bad.sum()))
    differ = wmargin = 0
    if got_wij is not None:
        for d, (got, color, fl, want_png) in enumerate(((got_wij, cj, fij, want_wij), (got_wji, ci, fji, want_wji))):
            torch_v = ref.warp_torch(color, fl, device="cuda")
            gv = got_values[d]
            assert np.all(np.abs(gv - torch_v) <= ref.WARP_TOL * (1 + np.abs(torch_v))), "warp values outside the bound"
            differ += int((gv != torch_v).sum())
            near = ref.round_margin(torch_v)
            wmargin += int(near.sum())
            for want in (ref.to_u8(torch_v), want_png):
                if want is not None:
                    bad = (got[..., ::-1] != want).any(axis=-1)
                    assert not (bad & ~near).any(), "warp bytes differ outside the rounding margin"
    return int(allowed.sum()), vdiff, differ, wmargin


@pytest.mark.parametrize("name", list(CASES))
def test_kernel_matches_reference_golden(name):
    """Every pair of a golden directory in one batch, colours passed once per frame: the reference's composite and warp PNGs, its
    max rad and NaN flags."""
    g = np.load(GOLDEN)
    pairs = CASES[name]
    frames = sorted({f for p in pairs for f in p})
    colors = np.stack([g[f"{name}/color/{f}"] for f in frames])
    pf = np.array([[frames.index(i), frames.index(j)] for i, j in pairs], np.int32)
    ins = [golden_pair(g, name, i, j) for i, j in pairs]
    vis, wij, wji, wv, mr, nan = solver.flow_visualize(colors, pf, np.stack([x[2] for x in ins]), np.stack([x[3] for x in ins]),
                                                       np.stack([x[4] for x in ins]), np.stack([x[5] for x in ins]), warp=True, want_values=True)
    totals = np.zeros(4, int)
    for n, (i, j) in enumerate(pairs):
        for d, fl in enumerate((ins[n][2], ins[n][3])):
            m, has_nan, *_ = ref.flow_stats(fl)
            assert nan[n, d] == has_nan and mr[n, d] == m
        totals += check_pair(vis[n], wij[n], wji[n], wv[n], ins[n], *golden_pngs(g, name, i, j))
    print(f"{name}: {totals[0]} composite pixels in the atan2 margin, {totals[1]} of them differ; {totals[2]} warp values differ from "
          f"torch's in their bits, {totals[3]} warp pixels in the rounding margin")


def random_case(F, pairs, H, W, seed):
    """Colours [F,H,W,3] in [0, 1] with a few out of range, and per pair flows with large and small motion, off-image targets, border
    hits, integer steps, NaN in some flows and unknown values, plus masks."""
    rng = np.random.default_rng(seed)
    iy, ix = np.mgrid[0:H, 0:W]
    colors = rng.random((F, H, W, 3)).astype(np.float32)
    colors[:, 0, 0] = (-0.2, 1.3, 0.5)
    fij, fji, mij, mji = [], [], [], []
    for n, _ in enumerate(pairs):
        for out, mo in ((fij, mij), (fji, mji)):
            a, b = rng.normal(0, 4, 2)
            f = np.stack((a + 3 * np.sin(0.05 * iy), b + 3 * np.cos(0.07 * ix)), axis=-1) + rng.normal(0, 1, (H, W, 2))
            k = rng.integers(0, 25, (H, W))
            f[..., 0] = np.where(k == 0, -ix, f[..., 0]); f[..., 0] = np.where(k == 1, W - 1 - ix, f[..., 0])
            f[..., 1] = np.where(k == 2, -iy, f[..., 1]); f[..., 1] = np.where(k == 3, H - 1 - iy, f[..., 1])
            f = np.where((k == 4)[..., None], np.round(f), f).astype(np.float32)
            if n % 3 == 1:
                f[k == 5] = np.nan
                f[-1, -1, 1] = np.nan
            f[k == 6, 0] = 5e7
            out.append(f)
            mo.append(np.where(rng.random((H, W)) < 0.7, 255, 0).astype(np.uint8))
    return colors, np.array(pairs, np.int32), np.stack(fij), np.stack(fji), np.stack(mij), np.stack(mji)


@pytest.mark.parametrize("shape,seed", [((224, 384), 1), ((61, 97), 2), ((2, 3), 3)])
def test_kernel_matches_restatement_random(shape, seed):
    H, W = shape
    pairs = [(0, 1), (1, 0), (1, 2), (0, 2), (3, 1), (2, 2)]
    colors, pf, fij, fji, mij, mji = random_case(4, pairs, H, W, seed)
    l0 = launches()
    vis, wij, wji, wv, mr, nan = solver.flow_visualize(colors, pf, fij, fji, mij, mji, warp=True, want_values=True)
    assert launches() - l0 == 2
    totals = np.zeros(4, int)
    for p, (i, j) in enumerate(pf):
        totals += check_pair(vis[p], wij[p], wji[p], wv[p], (colors[i], colors[j], fij[p], fji[p], mij[p], mji[p]))
    assert nan.any() and not nan.all()
    again = solver.flow_visualize(colors, pf, fij, fji, mij, mji, warp=True, want_values=True)
    for x, y in zip((vis, wij, wji, wv, mr, nan), again):
        assert x.tobytes() == y.tobytes()
    # without warp: the same composite, no warps
    v2, a, b = solver.flow_visualize(colors, pf, fij, fji, mij, mji)
    assert a is None and b is None and v2.tobytes() == vis.tobytes()
    print(f"{shape}: {totals[0]} composite pixels in the atan2 margin, {totals[1]} of them differ; {totals[2]} warp values differ from "
          f"torch's in their bits, {totals[3]} warp pixels in the rounding margin")


def test_batch_equals_pair_by_pair():
    """Many pairs sharing frames in one call give the same bytes as one call per pair."""
    H, W = 37, 53
    rng = np.random.default_rng(9)
    pairs = [tuple(int(x) for x in rng.integers(0, 6, 2)) for _ in range(40)]
    colors, pf, fij, fji, mij, mji = random_case(6, pairs, H, W, 9)
    vis, wij, wji = solver.flow_visualize(colors, pf, fij, fji, mij, mji, warp=True)
    for p, (i, j) in enumerate(pf):
        v1, a1, b1 = solver.flow_visualize(colors[[i, j]], np.array([[0, 1]]), fij[p:p + 1], fji[p:p + 1], mij[p:p + 1], mji[p:p + 1], warp=True)
        assert v1[0].tobytes() == vis[p].tobytes() and a1[0].tobytes() == wij[p].tobytes() and b1[0].tobytes() == wji[p].tobytes()


def test_refusals_launch_nothing():
    L = solver.lib()
    H, W = 4, 5
    colors = np.zeros((2, H, W, 3), np.float32); fl = np.zeros((1, H, W, 2), np.float32); m = np.zeros((1, H, W), np.uint8)
    vis = np.full((1, 2 * H, 4 * W, 3), 77, np.uint8)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    l0 = launches()
    for over in (dict(width=1), dict(num_frames=1), dict(warp=1)):      # the last: warp outputs null
        prm = abi.FlowVisParams(**{**dict(width=W, height=H, num_pairs=1, num_frames=2, warp=0), **over})
        assert L.rcvd_flow_visualize(C.byref(prm), 0, P(np.array([[0, 1]], np.int32), C.c_int32), P(fl, C.c_float), P(fl, C.c_float),
                                     P(m, C.c_uint8), P(m, C.c_uint8), P(colors, C.c_float), P(vis, C.c_uint8), None, None, None, None, None) == abi.ERR_INVALID
    assert launches() == l0 and np.all(vis == 77)


def _scene(tmp_path, N=6, W=96, H=64, seed=11):
    root = str(tmp_path / "scene")
    sc = synthetic.Scene(N, W, H, seed=seed, motion=0.04, rot_deg=0.5)
    pairs = synthetic_files.write_scene(sc, root)
    return root, pairs


def _read_dir(root, d):
    import cv2
    full = os.path.join(root, d)
    return {n: cv2.imread(os.path.join(full, n), cv2.IMREAD_UNCHANGED) for n in sorted(os.listdir(full))}


def test_end_to_end(tmp_path):
    """visualize_flow on a synthetic directory: decoded PNGs equal the restatement's, the skip rule, and a refused directory left
    without any file."""
    import cv2
    root, pairs = _scene(tmp_path)
    und = sorted({tuple(sorted(p)) for p in pairs})
    l0 = launches()
    st = flow.visualize_flow(root, warp=True, chunk_bytes=300_000)       # several chunks
    assert launches() - l0 >= 4 and st["pairs"] == len(und)
    vis, warps = _read_dir(root, "vis_flow"), _read_dir(root, "vis_flow_warped")
    assert len(vis) == len(und) and len(warps) == 2 * len(und)
    rd = lambda fmt, *k: synthetic_files.read_raw(os.path.join(root, fmt.format(*k)))
    margin = differ = 0
    for i, j in und:
        ins = (rd(flow.COLOR_FMT, i), rd(flow.COLOR_FMT, j), rd(flow.FLOW_FMT, i, j), rd(flow.FLOW_FMT, j, i),
               cv2.imread(os.path.join(root, flow.MASK_FMT.format(i, j)), 0), cv2.imread(os.path.join(root, flow.MASK_FMT.format(j, i)), 0))
        r = ref.visualize_pair(*ins)
        got = vis[os.path.basename(flow.VIS_FMT.format(i, j))]
        allowed = allowed_vis_mismatch(ref.flow_image_margin(ins[2]), ref.flow_image_margin(ins[3]))
        bad = (got != r["vis"]).any(axis=-1)
        assert not (bad & ~allowed).any()
        margin += int(allowed.sum()); differ += int(bad.sum())
        for key, (a, b), color, fl in (("warp_ij", (i, j), ins[1], ins[2]), ("warp_ji", (j, i), ins[0], ins[3])):
            tv = ref.warp_torch(color, fl, device="cuda")
            bad = (warps[os.path.basename(flow.WARP_FMT.format(a, b))] != ref.to_u8(tv)).any(axis=-1)
            assert not (bad & ~ref.round_margin(tv)).any()
    print(f"{margin} composite pixels in the atan2 margin, {differ} of them differ")
    # the skip rule: nothing to do; then a missing composite or sorted-index warp reruns its pair, rewriting both warps
    assert flow.visualize_flow(root, warp=True)["pairs"] == 0
    (a, b), (c, e) = und[0], und[1]
    os.remove(os.path.join(root, flow.VIS_FMT.format(a, b)))
    os.remove(os.path.join(root, flow.WARP_FMT.format(c, e)))
    sentinel = np.zeros((64, 96, 3), np.uint8)
    cv2.imwrite(os.path.join(root, flow.WARP_FMT.format(e, c)), sentinel)
    os.remove(os.path.join(root, flow.WARP_FMT.format(und[2][1], und[2][0])))      # a reverse-index warp alone does not rerun
    assert flow.visualize_flow(root)["pairs"] == 1                                     # without warp only the composite counts
    assert flow.Flow(root, root).visualize_flow(warp=True) is None
    after = _read_dir(root, "vis_flow_warped")
    assert np.array_equal(after[os.path.basename(flow.WARP_FMT.format(e, c))], warps[os.path.basename(flow.WARP_FMT.format(e, c))])
    assert os.path.basename(flow.WARP_FMT.format(und[2][1], und[2][0])) not in after
    assert np.array_equal(_read_dir(root, "vis_flow")[os.path.basename(flow.VIS_FMT.format(a, b))], vis[os.path.basename(flow.VIS_FMT.format(a, b))])
    # a refused directory: no file, no output directory
    other = str(tmp_path / "refused")
    shutil.copytree(root, other, ignore=shutil.ignore_patterns("vis_flow*"))
    os.remove(os.path.join(other, flow.MASK_FMT.format(*und[-1][::-1])))
    with pytest.raises(FileNotFoundError):
        flow.visualize_flow(other, warp=True)
    assert not os.path.exists(os.path.join(other, "vis_flow")) and not os.path.exists(os.path.join(other, "vis_flow_warped"))
    open(os.path.join(other, "flow", "readme.txt"), "w").close()
    with pytest.raises(ValueError):
        flow.visualize_flow(other)
    assert not os.path.exists(os.path.join(other, "vis_flow"))
