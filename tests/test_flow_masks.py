"""Flow-consistency masks without a GPU: the CPU restatement (tests/flow_masks_ref.py) against the reference's own outputs
(tests/golden/flow_masks_golden.npz, written by tests/golden/make_flow_masks_golden.py from utils/consistency.py), the float32 FMA
formulation the kernel computes, and the file semantics of robust_cvd_b200.flow: the skip rule, the input checks, the PNG encoder and
flow_list.json."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import flow_masks_ref as ref  # noqa: E402
from robust_cvd_b200 import flow, synthetic_files  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "flow_masks_golden.npz")
CASES = ("12x16", "9x13", "20x20")
THRESHOLDS = ((1, 1), (0.7, 0.7))
# The documented bound where torch's CPU grid_sample is not the vectorised FMA kernel: sampled values within 1e-5 (1 + |v|), sse
# within 1e-4 (1 + sse).  Measured differences on AVX2 / AVX-512 hosts: none.
SAMPLE_TOL, SSE_TOL = 1e-5, 1e-4


def golden_case(g, name):
    return g[f"{name}/flow_ij"], g[f"{name}/flow_ji"], g[f"{name}/color_i"], g[f"{name}/color_j"]


def compare(got, want, tol, exact):
    """Number of values that differ in their bits; asserts equality (exact) or the tolerance (NaN where both are NaN)."""
    both_nan = np.isnan(got) & np.isnan(want)
    diff = ~both_nan & (got != want)
    if exact:
        assert not diff.any(), f"{diff.sum()} values differ, max {np.nanmax(np.abs(got - want))}"
    else:
        assert np.all(both_nan | (got == want) | (np.abs(got - want) <= tol * (1 + np.abs(want))))
    return int(diff.sum())


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("sampler", ["torch", "fma"])
def test_restatement_matches_reference_golden(name, sampler):
    """Masks equal the reference's exactly; the sampled arrays and sse values to the last bit away from NaN target positions.
    sample_fma is plain float arithmetic, so it is exact on every host; torch is exact where its vectorised CPU kernel runs."""
    g = np.load(GOLDEN)
    fij, fji, ci, cj = golden_case(g, name)
    fn = ref.sample_torch if sampler == "torch" else ref.sample_fma
    exact = sampler == "fma" or ref.torch_is_vectorised()
    for ft, ct in THRESHOLDS:
        dirs = ref.flow_masks(fij, fji, ci, cj, ft, ct, sampler=fn)
        for d, out in enumerate(dirs):
            np.testing.assert_array_equal(out["mask"], g[f"{name}/{d}/mask_{ft}_{ct}"])
            ok = ~out["nan_pos"]
            assert out["nan_pos"].sum() >= 1 if d == 0 else True     # the case has NaN target positions
            for key, tol in (("flow_sample", SAMPLE_TOL), ("color_sample", SAMPLE_TOL), ("sse_flow", SSE_TOL), ("sse_color", SSE_TOL)):
                n = compare(out[key][ok], g[f"{name}/{d}/{key}"][ok], tol, exact)
                if n:
                    print(f"{name} dir {d} {key}: {n} values differ in their last bits")


def test_golden_covers_the_edge_cases():
    """The fixture holds targets exactly on every border, on pixel centres, off the image, NaN and inf, and masks of both values."""
    g = np.load(GOLDEN)
    for name in CASES:
        fij = g[f"{name}/flow_ij"]
        H, W = fij.shape[:2]
        X, Y, inside = ref.target_positions(fij)
        assert (X == 0).any() and (X == W - 1).any() and (Y == 0).any() and (Y == H - 1).any()
        assert (inside & (X == np.round(X)) & (Y == np.round(Y))).any()
        assert (~inside & np.isfinite(X) & np.isfinite(Y)).any() and np.isnan(X).any() and np.isinf(X).any()
        for d in range(2):
            for ft, ct in THRESHOLDS:
                m = g[f"{name}/{d}/mask_{ft}_{ct}"]
                assert 0 < m.mean() < 1
    assert any(g[f"{n}/flow_ij"].shape[0] != g[f"{n}/flow_ij"].shape[1] for n in CASES)
    # 0.7^2 is not a float32: the threshold changes the masks
    assert any((g[f"{n}/0/mask_1_1"] != g[f"{n}/0/mask_0.7_0.7"]).any() for n in CASES)


def test_thresholds_are_float32():
    assert ref.thresholds(1, 1) == (np.float32(1), np.float32(3))
    fsq, csq = ref.thresholds(0.7, 0.7)
    assert fsq == np.float32(0.7 ** 2) and csq == np.float32(3 * 0.7 ** 2) and float(fsq) != 0.49


def _touch_flows(root, pairs):
    os.makedirs(os.path.join(root, "flow"), exist_ok=True)
    os.makedirs(os.path.join(root, "flow_mask"), exist_ok=True)
    for i, j in pairs:
        for a, b in ((i, j), (j, i)):
            open(os.path.join(root, flow.FLOW_FMT.format(a, b)), "wb").close()


def test_skip_rule(tmp_path):
    """A pair is computed, once, when either of its masks is missing; a pair with both masks is skipped."""
    root = str(tmp_path)
    pairs = [(0, 1), (1, 2), (2, 3), (0, 4), (3, 7)]
    _touch_flows(root, pairs)
    open(os.path.join(root, "flow", "notes.txt"), "w").close()          # not a flow file
    present = [(0, 1), (1, 0), (2, 1), (3, 2), (7, 3)]                    # (0,1) complete, (1,2), (2,3), (3,7) half, (0,4) none
    for a, b in present:
        open(os.path.join(root, flow.MASK_FMT.format(a, b)), "wb").close()
    got = flow.pairs_to_compute(root)
    assert len(got) == len({frozenset(p) for p in got})
    assert {frozenset(p) for p in got} == {frozenset(p) for p in [(1, 2), (2, 3), (3, 7), (0, 4)]}
    # each is computed from the first of its flows that the listing gives and whose mask is missing
    listing = [n for n in os.listdir(os.path.join(root, "flow")) if n.startswith("flow_")]
    for i, j in got:
        assert not os.path.isfile(os.path.join(root, flow.MASK_FMT.format(i, j)))
        first = min((listing.index(os.path.basename(flow.FLOW_FMT.format(a, b))), (a, b)) for a, b in ((i, j), (j, i))
                    if not os.path.isfile(os.path.join(root, flow.MASK_FMT.format(a, b))))
        assert first[1] == (i, j)
    for a, b in [(1, 2), (2, 1), (2, 3), (3, 2), (0, 4), (4, 0), (0, 1), (1, 0), (3, 7), (7, 3)]:
        open(os.path.join(root, flow.MASK_FMT.format(a, b)), "wb").close()
    assert flow.pairs_to_compute(root) == []


def _write_case(root, frames, pairs, h=6, w=9, seed=0):
    rng = np.random.default_rng(seed)
    for d in ("flow", "flow_mask", "color_down"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for f in frames:
        synthetic_files.write_raw(os.path.join(root, flow.COLOR_FMT.format(f)), rng.random((h, w, 3)).astype(np.float32))
    for i, j in pairs:
        for a, b in ((i, j), (j, i)):
            synthetic_files.write_raw(os.path.join(root, flow.FLOW_FMT.format(a, b)), rng.normal(0, 1, (h, w, 2)).astype(np.float32))


def test_input_checks(tmp_path):
    """A missing reverse flow or colour, and a flow whose size differs from its colours, are refused before anything is written."""
    root = str(tmp_path)
    _write_case(root, [0, 1, 2], [(0, 1), (1, 2)])
    flow._check_inputs(root, [(0, 1), (1, 2)])
    os.remove(os.path.join(root, flow.FLOW_FMT.format(2, 1)))
    with pytest.raises(FileNotFoundError, match="flow 2 -> 1 is missing"):
        flow._check_inputs(root, flow.pairs_to_compute(root))
    synthetic_files.write_raw(os.path.join(root, flow.FLOW_FMT.format(2, 1)), np.zeros((6, 8, 2), np.float32))
    with pytest.raises(ValueError, match="differ in size"):
        flow._check_inputs(root, [(1, 2)])
    os.remove(os.path.join(root, flow.COLOR_FMT.format(0)))
    with pytest.raises(FileNotFoundError):
        flow._check_inputs(root, [(0, 1)])
    assert os.listdir(os.path.join(root, "flow_mask")) == []


def test_png_encoder_round_trip(tmp_path):
    import cv2
    import lib_python as lp
    rng = np.random.default_rng(3)
    for h, w in ((1, 1), (7, 5), (224, 384)):
        img = (rng.random((h, w)) > 0.4).astype(np.uint8) * 255
        fn = str(tmp_path / f"m_{h}_{w}.png")
        with open(fn, "wb") as f:
            f.write(flow.png_gray_bytes(img))
        np.testing.assert_array_equal(cv2.imread(fn, cv2.IMREAD_UNCHANGED), img)
        np.testing.assert_array_equal(lp._imreadPng(fn, True), img)


def reference_rows(root, frame_pairs):
    """The reference's flow_list.json rows, restated: cv2.imread(fn, 0), np.sum(mask > 0) / np.prod(mask.shape[:2]), min of the two."""
    import cv2
    rows, seen = [["frame0", "frame1", "mask_ratio"]], set()
    for pair in frame_pairs:
        if pair in seen:
            continue
        seen.update([pair, pair[::-1]])
        r = min(np.sum(m > 0) / np.prod(m.shape[:2]) for m in (cv2.imread(os.path.join(root, flow.MASK_FMT.format(*p)), 0) for p in (pair, pair[::-1])))
        rows += [[pair[0], pair[1], r], [pair[1], pair[0], r]]
    return rows


def test_pair_stats_json(tmp_path):
    """flow_list.json is byte-equal to json.dump of the reference's rows, and an existing file is returned untouched."""
    root = str(tmp_path)
    os.makedirs(os.path.join(root, "flow_mask"))
    rng = np.random.default_rng(5)
    pairs = [(0, 1), (1, 2), (1, 0), (0, 2), (2, 1), (3, 0), (0, 3)]
    for i, j in pairs:
        for a, b in ((i, j), (j, i)):
            m = (rng.random((7, 11)) < rng.random()).astype(np.uint8) * 255
            synthetic_files.write_png_gray(os.path.join(root, flow.MASK_FMT.format(a, b)), m)
    assert flow.compute_flow_pair_stats(root, pairs) is None
    path = os.path.join(root, "flow_list.json")
    got = open(path, "rb").read()
    import io
    buf = io.StringIO()
    json.dump(reference_rows(root, pairs), buf)
    assert got == buf.getvalue().encode()
    assert len(json.loads(got)) == 1 + 2 * 4
    os.remove(os.path.join(root, flow.MASK_FMT.format(0, 1)))           # an existing list is not recomputed
    assert flow.compute_flow_pair_stats(root, pairs) == path
    assert open(path, "rb").read() == got


def test_pair_stats_missing_mask(tmp_path):
    os.makedirs(tmp_path / "flow_mask")
    with pytest.raises(FileNotFoundError):
        flow.compute_flow_pair_stats(str(tmp_path), [(0, 1)])
    assert not os.path.exists(tmp_path / "flow_list.json")


def test_no_device_fails_loudly(tmp_path):
    """No CPU fallback: without a usable GPU compute_flow_masks raises before it looks at the directory."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        flow.compute_flow_masks(str(tmp_path))
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        flow.Flow(str(tmp_path), str(tmp_path)).compute_flow_masks()
