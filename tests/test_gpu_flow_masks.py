"""Flow-consistency masks on the GPU (csrc/rcvd_flowmask.cuh, rcvd_flow_masks, robust_cvd_b200.flow) against the CPU restatement
(tests/flow_masks_ref.py: numpy plus torch's CPU grid_sample, what the reference runs) and the reference's own golden outputs.

The stated bound: sse values within 1e-4 (1 + sse) of torch's, and equal mask decisions at every pixel whose torch sse lies farther
than that from its threshold.  The kernel computes the sampling as torch's vectorised CPU kernel does, so on AVX2 / AVX-512 hosts the
measured difference is none: the tests report the differing values and the margin pixels, and expect zero there."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import flow_masks_ref as ref  # noqa: E402
from tests.test_flow_masks import CASES, GOLDEN, SSE_TOL, THRESHOLDS, golden_case  # noqa: E402
from robust_cvd_b200 import abi, flow, solver, synthetic, synthetic_files  # noqa: E402

pytestmark = pytest.mark.gpu
CV_32FC3, CV_8UC1 = 21, 0


def launches():
    L = solver.lib()
    L.rcvd_flow_mask_launch_count.restype = C.c_int64
    return L.rcvd_flow_mask_launch_count()


def random_case(F, pairs, H, W, seed):
    """Colours [F,H,W,3] and per-pair flows with smooth consistent parts, off-image targets, border hits, integer steps and NaN."""
    rng = np.random.default_rng(seed)
    iy, ix = np.mgrid[0:H, 0:W]
    colors = (0.5 + 0.4 * np.sin(ix * 0.3)[None, ..., None] * np.cos(iy[None, ..., None] * 0.2 + np.arange(3))
              + rng.normal(0, 0.2, (F, H, W, 3))).astype(np.float32)
    fij, fji = [], []
    for _ in pairs:
        a, b = rng.normal(0, 3, 2)
        smooth = np.stack((a + 2 * np.sin(0.05 * iy), b + 2 * np.cos(0.07 * ix)), axis=-1)
        f = (smooth + rng.normal(0, 0.1, (H, W, 2))).astype(np.float32)
        k = rng.integers(0, 20, (H, W))
        f[..., 0] = np.where(k == 0, -ix, f[..., 0]); f[..., 0] = np.where(k == 1, W - 1 - ix, f[..., 0])
        f[..., 1] = np.where(k == 2, -iy, f[..., 1]); f[..., 1] = np.where(k == 3, H - 1 - iy, f[..., 1])
        f = np.where((k == 4)[..., None], np.round(f), f).astype(np.float32)
        f[k == 5] = np.nan
        g = (-smooth + rng.normal(0, 0.5, (H, W, 2))).astype(np.float32)
        fij.append(f); fji.append(g)
    return colors, np.array(pairs, np.int32), np.stack(fij), np.stack(fji)


def check_against_restatement(colors, pf, fij, fji, flow_thresh, color_thresh, want=None):
    """GPU vs restatement on every pair and direction: sse within the bound, masks equal outside the margin, counts equal to the masks'
    sums, a bit-identical rerun.  want: optional golden masks per (pair, direction).  Returns (values that differ, margin pixels)."""
    fsq, csq = ref.thresholds(flow_thresh, color_thresh)
    l0 = launches()
    mij, mji, cnt, sf, sc = solver.flow_masks(colors, pf, fij, fji, fsq, csq, want_sse=True)
    assert launches() > l0
    differ = margin = 0
    for p, (i, j) in enumerate(pf):
        dirs = ref.flow_masks(fij[p], fji[p], colors[i], colors[j], flow_thresh, color_thresh)
        for d, (out, m) in enumerate(zip(dirs, (mij[p], mji[p]))):
            assert set(np.unique(m)) <= {0, 255}
            ok = ~out["nan_pos"]
            assert np.all(np.isnan(sf[p, d][~ok])) and np.all(np.isnan(sc[p, d][~ok]))
            near = np.zeros_like(ok)
            for key, got, thr in (("sse_flow", sf[p, d], fsq), ("sse_color", sc[p, d], csq)):
                w = out[key]
                both_nan = np.isnan(got) & np.isnan(w)
                assert np.all((both_nan | (got == w) | (np.abs(got - w) <= SSE_TOL * (1 + np.abs(w))))[ok]), key
                differ += int((~both_nan & (got != w))[ok].sum())
                near |= ok & (np.abs(w - thr) <= SSE_TOL * (1 + thr))
            mism = (m == 255) != out["mask"]
            assert not (mism & ~near).any(), f"pair {p} dir {d}: masks differ away from the threshold margin"
            margin += int(near.sum())
            if want is not None:
                np.testing.assert_array_equal(m == 255, want[p][d])
        assert cnt[p, 0] == np.count_nonzero(mij[p]) and cnt[p, 1] == np.count_nonzero(mji[p])
    again = solver.flow_masks(colors, pf, fij, fji, fsq, csq, want_sse=True)
    for x, y in zip((mij, mji, cnt, sf, sc), again):
        assert x.tobytes() == y.tobytes()
    print(f"{differ} sse values differ from torch's in their bits; {margin} pixels within the threshold margin")
    if ref.torch_is_vectorised():
        assert differ == 0
    return differ, margin


@pytest.mark.parametrize("shape,seed", [((224, 384), 1), ((61, 97), 2), ((64, 64), 3)])
@pytest.mark.parametrize("thresh", [(1, 1), (0.7, 0.7), (2.5, 0.3)])
def test_kernel_matches_restatement_random(shape, seed, thresh):
    H, W = shape
    pairs = [(0, 1), (1, 0), (1, 2), (0, 2), (3, 1)]           # frames shared by several pairs, both orders
    colors, pf, fij, fji = random_case(4, pairs, H, W, seed)
    check_against_restatement(colors, pf, fij, fji, *thresh)


@pytest.mark.parametrize("name", CASES)
def test_kernel_matches_reference_golden(name):
    """Each golden case as a pair (0, 1) and reversed as (1, 0) in one batch: the reference's masks exactly, and its sse values."""
    g = np.load(GOLDEN)
    fij, fji, ci, cj = golden_case(g, name)
    colors = np.stack([ci, cj]); pf = np.array([[0, 1], [1, 0]], np.int32)
    for ft, ct in THRESHOLDS:
        want = [[g[f"{name}/0/mask_{ft}_{ct}"], g[f"{name}/1/mask_{ft}_{ct}"]], [g[f"{name}/1/mask_{ft}_{ct}"], g[f"{name}/0/mask_{ft}_{ct}"]]]
        check_against_restatement(colors, pf, np.stack([fij, fji]), np.stack([fji, fij]), ft, ct, want)
    _, _, _, sf, sc = solver.flow_masks(colors, pf[:1], fij[None], fji[None], *ref.thresholds(), want_sse=True)
    for d, f in enumerate((fij, fji)):
        X, Y, _ = ref.target_positions(f)
        ok = ~np.isnan(X) & ~np.isnan(Y)
        for key, got in (("sse_flow", sf[0, d]), ("sse_color", sc[0, d])):
            w = g[f"{name}/{d}/{key}"]
            both_nan = np.isnan(got) & np.isnan(w)
            assert np.all((both_nan | (got == w) | (np.abs(got - w) <= SSE_TOL * (1 + np.abs(w))))[ok]), key
            if ref.torch_is_vectorised():
                assert np.all((both_nan | (got == w))[ok]), key


def test_many_pairs_one_launch_per_65535():
    """A batch over the grid.y limit: every pair computed, the same as in small batches."""
    H, W = 2, 3
    P = 65600
    rng = np.random.default_rng(4)
    colors = rng.random((3, H, W, 3)).astype(np.float32)
    pf = rng.integers(0, 3, (P, 2)).astype(np.int32)
    fij = rng.normal(0, 0.7, (P, H, W, 2)).astype(np.float32); fji = rng.normal(0, 0.7, (P, H, W, 2)).astype(np.float32)
    l0 = launches()
    mij, mji, cnt = solver.flow_masks(colors, pf, fij, fji)
    assert launches() - l0 == 2
    for s in (slice(0, 5), slice(65530, 65600)):
        a, b, c = solver.flow_masks(colors, pf[s], fij[s], fji[s])
        np.testing.assert_array_equal(a, mij[s]); np.testing.assert_array_equal(b, mji[s]); np.testing.assert_array_equal(c, cnt[s])
    assert 0 < cnt.sum() < 2 * P * H * W


def test_bad_arguments_refused_with_nothing_written():
    L = solver.lib()
    H, W = 4, 5
    colors = np.zeros((2, H, W, 3), np.float32); fl = np.zeros((1, H, W, 2), np.float32)
    pf = np.array([[0, 1]], np.int32)
    mij = np.full((1, H, W), 77, np.uint8); mji = mij.copy(); cnt = np.full((1, 2), -5, np.int64)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    good = dict(width=W, height=H, num_pairs=1, num_frames=2, flow_thresh_sq=1.0, color_thresh_sq=3.0)
    bad = [dict(width=0), dict(height=-1), dict(num_pairs=-1), dict(num_frames=0), dict(flow_thresh_sq=float("nan")),
           dict(color_thresh_sq=float("nan")), dict(width=1 << 16, height=1 << 15), dict(num_frames=1)]     # the last: pair frame 1 out of range
    l0 = launches()
    for over in bad:
        prm = abi.FlowMaskParams(**{**good, **over})
        rc = L.rcvd_flow_masks(C.byref(prm), 0, P(pf, C.c_int32), P(fl, C.c_float), P(fl, C.c_float), P(colors, C.c_float),
                               P(mij, C.c_uint8), P(mji, C.c_uint8), P(cnt, C.c_int64), None, None)
        assert rc == abi.ERR_INVALID, over
    prm = abi.FlowMaskParams(**good)
    assert L.rcvd_flow_masks(None, 0, P(pf, C.c_int32), P(fl, C.c_float), P(fl, C.c_float), P(colors, C.c_float), P(mij, C.c_uint8), P(mji, C.c_uint8), None, None, None) == abi.ERR_INVALID
    for k in range(6):
        args = [P(pf, C.c_int32), P(fl, C.c_float), P(fl, C.c_float), P(colors, C.c_float), P(mij, C.c_uint8), P(mji, C.c_uint8)]
        args[k] = None
        assert L.rcvd_flow_masks(C.byref(prm), 0, *args, None, None, None) == abi.ERR_INVALID
    neg = np.array([[0, -1]], np.int32)
    assert L.rcvd_flow_masks(C.byref(prm), 0, P(neg, C.c_int32), P(fl, C.c_float), P(fl, C.c_float), P(colors, C.c_float), P(mij, C.c_uint8), P(mji, C.c_uint8), None, None, None) == abi.ERR_INVALID
    assert launches() == l0
    assert np.all(mij == 77) and np.all(mji == 77) and np.all(cnt == -5)
    with pytest.raises(ValueError):
        solver.flow_masks(colors, pf, fl, np.zeros((1, H, W + 1, 2), np.float32))
    empty = abi.FlowMaskParams(**{**good, "num_pairs": 0})
    assert L.rcvd_flow_masks(C.byref(empty), 0, None, None, None, None, None, None, None, None, None) == abi.OK


def _scene(tmp_path, name="scene", N=8, W=96, H=64, seed=11):
    root = str(tmp_path / name)
    sc = synthetic.Scene(N, W, H, seed=seed, motion=0.04, rot_deg=0.5)
    pairs = synthetic_files.write_scene(sc, root)
    return root, pairs


def _read_masks(root):
    import cv2
    d = os.path.join(root, "flow_mask")
    return {n: cv2.imread(os.path.join(d, n), cv2.IMREAD_UNCHANGED) for n in sorted(os.listdir(d))}


def _restatement_files(root, pairs):
    """flow_mask/ and flow_list.json of root written by the CPU restatement (the reference's arithmetic and file semantics)."""
    import json
    import cv2
    rows, seen = [["frame0", "frame1", "mask_ratio"]], set()
    col = lambda f: synthetic_files.read_raw(os.path.join(root, flow.COLOR_FMT.format(f)))
    fl = lambda a, b: synthetic_files.read_raw(os.path.join(root, flow.FLOW_FMT.format(a, b)))
    os.makedirs(os.path.join(root, "flow_mask"), exist_ok=True)
    for i, j in flow.pairs_to_compute(root):
        for (a, b), out in zip(((i, j), (j, i)), ref.flow_masks(fl(i, j), fl(j, i), col(i), col(j))):
            cv2.imwrite(os.path.join(root, flow.MASK_FMT.format(a, b)), out["mask"].astype(np.uint8) * 255)
    for p in pairs:
        if p in seen:
            continue
        seen.update([p, p[::-1]])
        r = min(np.sum(m > 0) / np.prod(m.shape[:2]) for m in (cv2.imread(os.path.join(root, flow.MASK_FMT.format(*q)), 0) for q in (p, p[::-1])))
        rows += [[p[0], p[1], r], [p[1], p[0], r]]
    with open(os.path.join(root, "flow_list.json"), "w") as f:
        json.dump(rows, f)


def _constraints(root):
    import lib_python as lp
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", CV_32FC3)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True); fp.matchSeparation = 4; fp.doNotUseCache = True
    fc = lp.FlowConstraintsCollection(v, fp)
    return {k: np.asarray(v[0]) for k, v in fc._pairs().items()}


def test_end_to_end_regenerates_the_files(tmp_path):
    """flow_mask/ and flow_list.json deleted from a synthetic directory are regenerated by compute_flow_masks + compute_flow_pair_stats
    equal to the restatement's files, and FlowConstraintsCollection reads the same constraint lists from both."""
    root, pairs = _scene(tmp_path)
    other = str(tmp_path / "restated")
    shutil.rmtree(os.path.join(root, "flow_mask")); os.remove(os.path.join(root, "flow_list.json"))
    shutil.copytree(root, other)
    l0 = launches()
    stats = flow.compute_flow_masks(root, chunk_bytes=200_000)          # several chunks
    assert launches() > l0 and stats["pairs"] == len(pairs) // 2
    assert flow.compute_flow_pair_stats(root, pairs) is None
    _restatement_files(other, pairs)
    gm, rm = _read_masks(root), _read_masks(other)
    assert gm.keys() == rm.keys() and len(gm) == len(pairs)
    for n in gm:
        assert gm[n].dtype == np.uint8 and gm[n].ndim == 2
        np.testing.assert_array_equal(gm[n], rm[n], err_msg=n)
    assert 0.3 < np.mean([m.mean() / 255 for m in gm.values()]) < 1
    assert open(os.path.join(root, "flow_list.json"), "rb").read() == open(os.path.join(other, "flow_list.json"), "rb").read()
    cg, cr = _constraints(root), _constraints(other)
    assert cg.keys() == cr.keys() and sum(len(v) for v in cg.values()) > 100
    for k in cg:
        np.testing.assert_array_equal(cg[k], cr[k])
    # a second run finds every mask and computes nothing
    assert flow.compute_flow_masks(root)["pairs"] == 0
    # the Flow class is the same drop-in
    shutil.rmtree(os.path.join(root, "flow_mask"))
    flow.Flow(root, root).compute_flow_masks()
    assert _read_masks(root).keys() == gm.keys() and all((_read_masks(root)[n] == gm[n]).all() for n in gm)


def test_skip_rule_and_errors(tmp_path):
    """Only pairs with a missing mask are computed, and both of their masks are rewritten; a missing reverse flow and a size mismatch
    raise before any mask is written."""
    root, pairs = _scene(tmp_path, N=5, W=40, H=24)
    shutil.rmtree(os.path.join(root, "flow_mask")); os.makedirs(os.path.join(root, "flow_mask"))
    sentinel = np.full((24, 40), 7, np.uint8)
    und = sorted({tuple(sorted(p)) for p in pairs})
    keep_both, keep_one = und[0], und[1]
    for a, b in (keep_both, keep_both[::-1], keep_one):
        synthetic_files.write_png_gray(os.path.join(root, flow.MASK_FMT.format(a, b)), sentinel)
    todo = {frozenset(p) for p in flow.pairs_to_compute(root)}
    assert todo == {frozenset(p) for p in und[1:]}
    stats = flow.compute_flow_masks(root)
    assert stats["pairs"] == len(und) - 1
    m = _read_masks(root)
    assert len(m) == len(pairs)
    for a, b in pairs:
        is_sentinel = bool((m[os.path.basename(flow.MASK_FMT.format(a, b))] == 7).all())
        assert is_sentinel == (tuple(sorted((a, b))) == keep_both), (a, b)
    # errors: nothing written
    shutil.rmtree(os.path.join(root, "flow_mask")); os.makedirs(os.path.join(root, "flow_mask"))
    a, b = und[-1]
    os.remove(os.path.join(root, flow.FLOW_FMT.format(b, a)))
    with pytest.raises(FileNotFoundError):
        flow.compute_flow_masks(root)
    assert os.listdir(os.path.join(root, "flow_mask")) == []
    synthetic_files.write_raw(os.path.join(root, flow.FLOW_FMT.format(b, a)), np.zeros((24, 41, 2), np.float32))
    with pytest.raises(ValueError):
        flow.compute_flow_masks(root)
    assert os.listdir(os.path.join(root, "flow_mask")) == []
