"""CPU tests of the homography-registered flows (flow.compute_flow): the restatement tests/flow_register_ref.py against OpenCV and numpy
live, the reference's fixture (tests/golden/flow_register_golden.npz), the host homography estimation and its fallbacks, and the
refusals of compute_flow."""
import os
import struct
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import pytest

from robust_cvd_b200 import flow as F
from robust_cvd_b200.synthetic_files import write_raw
from tests import flow_register_ref as R

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "flow_register_golden.npz"))
CASES = [str(c) for c in GOLDEN["cases"]]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _warp_matrices(rng, W, H):
    """A seeded sweep of H_BA: identity, subpixel translations, rotations about the centre, strong perspective whose W = 0 line crosses
    the image, and maps that send every pixel outside."""
    out = [np.eye(3)]
    for _ in range(3):
        out.append(np.array([[1, 0, rng.uniform(-3, 3)], [0, 1, rng.uniform(-3, 3)], [0, 0, 1.0]]))
    for a in (0.01, -0.2, 1.3):
        c, s = np.cos(a), np.sin(a)
        T = np.array([[1, 0, W / 2], [0, 1, H / 2], [0, 0, 1.0]])
        out.append(T @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]) @ np.linalg.inv(T))
    for _ in range(3):
        out.append(np.eye(3) + rng.normal(0, [[0.05, 0.05, 3], [0.05, 0.05, 3], [3e-4, 3e-4, 0]]))
    # W = 0 where 1 + p x + q y = 0: the line through the image's centre
    p = 2.0 / W
    out.append(np.array([[1, 0.1, 0], [0.05, 1, 0], [p, (-1 - p * W / 2) / (H / 2), 1.0]]))
    out.append(np.array([[1, 0, 5 * W], [0, 1, 0], [0, 0, 1.0]]))
    out.append(np.array([[0.5, 0, -3 * W], [0, 0.5, -3 * H], [0, 0, 1.0]]))
    return out


@pytest.mark.parametrize("W,H", [(1024, 576), (97, 61), (333, 17), (64, 16), (5, 3), (1, 1)])
def test_warp_matches_cv2(W, H):
    rng = np.random.default_rng(W * 1000 + H)
    img = rng.integers(0, 256, (H, W, 3), np.uint8)
    for n, M in enumerate(_warp_matrices(rng, W, H)):
        got = R.warp_perspective(img, M)
        ref = cv2.warpPerspective(img, M, (W, H))
        assert np.array_equal(got, ref), (W, H, n, np.count_nonzero(got != ref))


def test_warp_block_width():
    assert R.warp_block_width(1024, 576) == 64
    assert R.warp_block_width(97, 61) == 64
    assert R.warp_block_width(333, 5) == 204
    assert R.warp_block_width(40, 3) == 40


def test_inverse_matches_cv2():
    rng = np.random.default_rng(7)
    mats = [rng.normal(size=(3, 3)) for _ in range(500)] + [np.eye(3) + rng.normal(0, 1e-3, (3, 3)) for _ in range(100)]
    mats.append(np.array([[1, 2, 3], [2, 4, 6], [0, 0, 1.0]]))   # det 0
    for M in mats:
        _, ref = cv2.invert(M)
        assert np.array_equal(F.cv_invert3(M), ref)
        assert np.array_equal(R.cv_invert3(M), ref)


def test_fma_emulation():
    rng = np.random.default_rng(3)
    a, b, c = rng.normal(size=(3, 10000))
    from fractions import Fraction
    got = R.fma(a, b, c)
    for k in range(0, 10000, 97):
        assert got[k] == float(Fraction(a[k]) * Fraction(b[k]) + Fraction(c[k]))


def _numpy_unregister(flow, H_BA):
    """infer's un-registration, as the reference writes it."""
    H, W = flow.shape[:2]
    fy, fx = np.mgrid[0:H, 0:W].astype(np.float32)
    fxx = fx + flow[:, :, 0]
    fyy = fy + flow[:, :, 1]
    x, y, z = np.linalg.inv(H_BA).dot(np.concatenate((fxx.reshape(1, -1), fyy.reshape(1, -1), np.ones_like(fyy).reshape(1, -1)), 0))
    x, y = x / z, y / z
    return np.concatenate((x.reshape(H, W, 1) - fx.reshape(H, W, 1), y.reshape(H, W, 1) - fy.reshape(H, W, 1)), 2)


def test_composition_matches_numpy_dot():
    rng = np.random.default_rng(11)
    H, W = 576, 1024
    found = {}
    for t in range(3):
        H_BA = np.eye(3) + rng.normal(0, [[0.05, 0.05, 3], [0.05, 0.05, 3], [2e-4, 2e-4, 0]])
        flow = rng.normal(0, 3, (H, W, 2)).astype(np.float32)
        ref = _numpy_unregister(flow, H_BA)
        for order in ("fma", "plain"):
            found.setdefault(order, []).append(float(np.mean(_bits(R.unregister(flow, np.linalg.inv(H_BA), order)) == _bits(ref))))
        assert np.array_equal(_bits(R.unregister(flow, np.linalg.inv(H_BA), "fma")), _bits(ref)), t
    print(f"np.dot order on this host: fma chain (bit-equal fraction {found['fma']}); plain sum bit-equal fraction {found['plain']}")


@pytest.mark.parametrize("src,dst", [((1024, 576), (384, 224)), ((96, 64), (41, 23)), ((40, 30), (97, 71)), ((1024, 576), (1024, 576)),
                                     ((7, 5), (3, 2)), ((384, 224), (192, 96)), ((5, 4), (2, 9)), ((3, 1), (11, 1))])
def test_cubic_matches_cv2(src, dst):
    rng = np.random.default_rng(src[0] * dst[0])
    img = rng.normal(0, 5, (src[1], src[0], 2))
    img[0, 0, 0] = -0.0
    ref = cv2.resize(img, dst, interpolation=cv2.INTER_CUBIC)
    assert np.array_equal(_bits(R.resize_cubic(img, *dst)), _bits(ref))


def test_cubic_signed_zero_at_border_columns():
    """A border column sums from 0 + p0, so an all -0 sum is +0 there and -0 inside."""
    img = np.full((6, 9, 2), -0.0)
    ref = cv2.resize(img, (5, 4), interpolation=cv2.INTER_CUBIC)
    assert np.array_equal(_bits(R.resize_cubic(img, 5, 4)), _bits(ref))


@pytest.mark.parametrize("case", CASES)
def test_restatement_matches_fixture(case, tmp_path):
    g = {k.split("/", 1)[1]: GOLDEN[k] for k in GOLDEN.files if k.startswith(case + "/")}
    H_BA = g["H_BA"]
    assert np.array_equal(R.warp_perspective(g["frame2"], H_BA), g["registered"])
    flow = R.unregister(g["model_flow"], np.linalg.inv(H_BA))
    assert np.array_equal(_bits(flow), _bits(g["flow"]))
    w, h = (int(v) for v in g["size"])
    resized = R.resize_flow(flow, w, h)
    assert np.array_equal(_bits(resized), _bits(g["resized"]))
    fn = tmp_path / "flow.raw"
    write_raw(str(fn), resized.astype(np.float32))
    assert fn.read_bytes() == g["raw"].tobytes()
    assert np.array_equal(_bits(R.flow_raw_values(g["model_flow"], np.linalg.inv(H_BA), w, h)), _bits(resized.astype(np.float32)))


def _sift():
    return cv2.SIFT_create()


@pytest.mark.parametrize("case", CASES)
def test_homography_matches_reference(case):
    f1, f2 = GOLDEN[case + "/frame1"], GOLDEN[case + "/frame2"]
    det = _sift()
    H = F.homography(F.frame_features(f1, det), F.frame_features(f2, det))
    assert np.array_equal(H, GOLDEN[case + "/H_BA"])


def test_homography_cached_threaded_equals_per_pair():
    """Features cached per frame and pairs matched on threads give the H of features recomputed per pair, in order."""
    rng = np.random.default_rng(5)
    base = GOLDEN["perspective/frame1"]
    frames = [base] + [cv2.warpPerspective(base, np.eye(3) + rng.normal(0, [[0.02, 0.02, 2], [0.02, 0.02, 2], [1e-4, 1e-4, 0]]),
                                           base.shape[1::-1], borderMode=cv2.BORDER_REFLECT) for _ in range(4)]
    pairs = [(i, j) for i in range(5) for j in range(5) if i != j]
    serial = [F.homography(F.frame_features(frames[i], _sift()), F.frame_features(frames[j], _sift())) for i, j in pairs]
    with ThreadPoolExecutor(4) as pool:
        feats = list(pool.map(lambda f: F.frame_features(f, _sift()), frames))
        threaded = list(pool.map(lambda p: F.homography(feats[p[0]], feats[p[1]]), pairs))
    assert any(not np.array_equal(h, np.eye(3)) for h in serial)
    for a, b in zip(serial, threaded):
        assert np.array_equal(a, b)


def test_homography_fallbacks(monkeypatch):
    eye = np.eye(3)
    rng = np.random.default_rng(2)
    kps = rng.uniform(0, 50, (8, 2)).astype(np.float32)
    des = rng.random((8, 128)).astype(np.float32)
    # no keypoints: knnMatch raises on a None descriptor set
    assert np.array_equal(F.homography((np.float32([]), None), (kps, des)), eye)
    assert np.array_equal(F.homography((kps, des), (np.float32([]), None)), eye)
    # at most 4 matches pass the ratio test
    assert np.array_equal(F.homography((kps[:4], des[:4]), (kps[:4], des[:4])), eye)
    # findHomography returning None, a singular matrix, or raising
    for ret in (lambda *a, **k: (None, None), lambda *a, **k: (np.ones((3, 3)), None)):
        monkeypatch.setattr(cv2, "findHomography", ret)
        assert np.array_equal(F.homography((kps, des), (kps + 1, des)), eye)

    def boom(*a, **k):
        raise cv2.error("findHomography")
    monkeypatch.setattr(cv2, "findHomography", boom)
    assert np.array_equal(F.homography((kps, des), (kps + 1, des)), eye)


def test_homography_five_matches_reaches_findhomography(monkeypatch):
    calls = []
    rng = np.random.default_rng(4)
    kps = rng.uniform(0, 50, (5, 2)).astype(np.float32)
    des = rng.random((5, 128)).astype(np.float32)

    def record(src, dst, method, thresh):
        calls.append((src.copy(), dst.copy(), method, thresh))
        return np.diag([2.0, 2.0, 1.0]), None
    monkeypatch.setattr(cv2, "findHomography", record)
    H = F.homography((kps, des), (kps + 3, des))
    assert np.array_equal(H, np.diag([2.0, 2.0, 1.0]))
    (src, dst, method, thresh), = calls
    assert method == cv2.RANSAC and thresh == 4.0 and src.dtype == np.float32
    assert np.array_equal(src, kps + 3) and np.array_equal(dst, kps)


def _write_png(fn, img):
    os.makedirs(os.path.dirname(fn), exist_ok=True)
    cv2.imwrite(fn, img)


def _make_dir(root, n=3, size=(40, 64), down=(16, 24)):
    rng = np.random.default_rng(9)
    for f in range(n):
        _write_png(os.path.join(root, F.FRAME_FMT.format(f)), rng.integers(0, 256, size + (3,), np.uint8))
    os.makedirs(os.path.join(root, "color_down"), exist_ok=True)
    write_raw(os.path.join(root, F.COLOR_FMT.format(0)), np.zeros(down + (3,), np.float32))


def _listing(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs) + \
        sorted(os.path.relpath(d, root) for d, _, _ in os.walk(root))


def test_refusals_write_nothing(tmp_path):
    root = str(tmp_path)
    _make_dir(root)
    before = _listing(root)
    pairs = [(0, 1), (1, 2)]
    with pytest.raises(ValueError):
        F.compute_flow(root, pairs, flow_model="flownet")
    if not hasattr(cv2, "xfeatures2d"):
        with pytest.raises(RuntimeError, match="features="):
            F.compute_flow(root, pairs, model=lambda *a, **k: None)
    with pytest.raises(RuntimeError, match="model="):
        F.compute_flow(root, pairs, features=cv2.SIFT_create)   # the reference's RAFT is not importable here
    with pytest.raises(FileNotFoundError):
        F.compute_flow(root, [(0, 5)], model=lambda *a, **k: None, features=cv2.SIFT_create)
    _write_png(os.path.join(root, F.FRAME_FMT.format(3)), np.zeros((40, 65, 3), np.uint8))
    with pytest.raises(ValueError, match="frame 0"):
        F.compute_flow(root, [(0, 3)], model=lambda *a, **k: None, features=cv2.SIFT_create)
    os.remove(os.path.join(root, F.FRAME_FMT.format(3)))
    os.remove(os.path.join(root, F.COLOR_FMT.format(0)))
    with pytest.raises(FileNotFoundError, match="color_down"):
        F.compute_flow(root, pairs, model=lambda *a, **k: None, features=cv2.SIFT_create)
    write_raw(os.path.join(root, F.COLOR_FMT.format(0)), np.zeros((16, 24, 3), np.float32))
    assert _listing(root) == before


def test_all_present_does_nothing(tmp_path):
    root = str(tmp_path)
    os.makedirs(os.path.join(root, "flow"))
    for i, j in [(0, 1), (1, 0)]:
        write_raw(os.path.join(root, F.FLOW_FMT.format(i, j)), np.zeros((4, 5, 2), np.float32))

    def no_model(*a, **k):
        raise AssertionError("the model ran")
    stats = F.compute_flow(root, [(0, 1), (1, 0)], model=no_model, features=no_model)
    assert stats["pairs"] == 0
    assert F.Flow(root, root).check_flow_files([(0, 1), (1, 0)])
    assert not F.Flow(root, root).check_flow_files([(0, 1), (0, 2)])


def test_pairs_to_compute(tmp_path):
    root = str(tmp_path)
    os.makedirs(os.path.join(root, "flow"))
    write_raw(os.path.join(root, F.FLOW_FMT.format(1, 0)), np.zeros((4, 5, 2), np.float32))
    assert F.flow_pairs_to_compute(root, [(0, 1), (1, 0), (0, 1), (2, 1)]) == [(0, 1), (2, 1)]


def test_raw_header_of_fixture():
    for case in CASES:
        raw = GOLDEN[case + "/raw"].tobytes()
        rows, cols, typ, es = struct.unpack("<iiiQ", raw[:20])
        w, h = (int(v) for v in GOLDEN[case + "/size"])
        assert (rows, cols, typ, es) == (h, w, 13, 8) and len(raw) == 20 + h * w * 8
