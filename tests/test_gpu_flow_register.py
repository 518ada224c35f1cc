"""GPU tests of the homography-registered flows: rcvd_homography_warp and rcvd_flow_unregister against the restatement
(tests/flow_register_ref.py), OpenCV and the reference's fixture, their grid.y split, and flow.compute_flow end to end on a synthetic
directory with a stub model, against a replay of the reference's sequence in cv2 and numpy."""
import os

import cv2
import numpy as np
import pytest

from robust_cvd_b200 import flow as F
from robust_cvd_b200 import solver
from robust_cvd_b200.synthetic_files import read_raw, write_raw
from tests import flow_register_ref as R

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "flow_register_golden.npz"))
CASES = [str(c) for c in GOLDEN["cases"]]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _matrices(rng, W, H, n):
    out = [np.eye(3), np.array([[1, 0, 0.37], [0, 1, -0.61], [0, 0, 1.0]])]
    p = 2.0 / W
    out.append(np.array([[1, 0.1, 0], [0.05, 1, 0], [p, (-1 - p * W / 2) / (H / 2), 1.0]]))   # W = 0 through the centre
    out.append(np.array([[1, 0, 5 * W], [0, 1, 0], [0, 0, 1.0]]))                           # everything outside
    while len(out) < n:
        out.append(np.eye(3) + rng.normal(0, [[0.05, 0.05, 3], [0.05, 0.05, 3], [3e-4, 3e-4, 0]]))
    return out


@pytest.mark.parametrize("W,H", [(1024, 576), (97, 61), (333, 17), (5, 3)])
def test_warp_kernel_matches_restatement_and_cv2(W, H):
    rng = np.random.default_rng(W + H)
    frames = rng.integers(0, 256, (3, H, W, 3), np.uint8)
    mats = _matrices(rng, W, H, 8)
    pf = [k % 3 for k in range(len(mats))]
    got = solver.homography_warp(frames, pf, [F.cv_invert3(M) for M in mats])
    for k, M in enumerate(mats):
        ref = cv2.warpPerspective(frames[pf[k]], M, (W, H))
        assert np.array_equal(got[k], ref), (k, np.count_nonzero(got[k] != ref))
        assert np.array_equal(got[k], R.warp_perspective(frames[pf[k]], M))


@pytest.mark.parametrize("src,dst", [((1024, 576), (384, 224)), ((97, 61), (41, 23)), ((40, 30), (97, 71)), ((64, 48), (64, 48)),
                                     ((7, 5), (3, 2))])
def test_unregister_kernel_matches_restatement(src, dst):
    rng = np.random.default_rng(src[0] + dst[0])
    W, H = src
    mats = _matrices(rng, W, H, 5)[:1] + _matrices(rng, W, H, 5)[4:] + [np.eye(3) + rng.normal(0, [[0.05, 0.05, 3], [0.05, 0.05, 3], [3e-4, 3e-4, 0]])]
    flows = rng.normal(0, 4, (len(mats), H, W, 2)).astype(np.float32)
    hinv = [np.linalg.inv(M) for M in mats]
    got = solver.flow_unregister(flows, hinv, dst)
    for k in range(len(mats)):
        ref = R.flow_raw_values(flows[k], hinv[k], *dst)
        assert np.array_equal(_bits(got[k]), _bits(ref)), (k, np.count_nonzero(got[k] != ref))


def test_kernels_match_fixture():
    for case in CASES:
        g = {k.split("/", 1)[1]: GOLDEN[k] for k in GOLDEN.files if k.startswith(case + "/")}
        reg = solver.homography_warp(g["frame2"][None], [0], [F.cv_invert3(g["H_BA"])])
        assert np.array_equal(reg[0], g["registered"]), case
        out = solver.flow_unregister(g["model_flow"][None], [np.linalg.inv(g["H_BA"])], tuple(int(v) for v in g["size"]))
        assert np.array_equal(_bits(out[0]), _bits(g["resized"].astype(np.float32))), case


def test_grid_y_split():
    """65537 pairs: two launches per kernel; each pair's result is its own."""
    rng = np.random.default_rng(1)
    P, W, H = 65537, 6, 4
    frames = rng.integers(0, 256, (5, H, W, 3), np.uint8)
    mats = _matrices(rng, W, H, 7)
    pf = np.arange(P) % 5
    mi = np.arange(P) % 7
    reg = solver.homography_warp(frames, pf, np.stack([F.cv_invert3(mats[m]) for m in mi]))
    ref = {(f, m): R.warp_perspective(frames[f], mats[m]) for f in range(5) for m in range(7)}
    for p in list(range(0, P, 997)) + [65534, 65535, 65536]:
        assert np.array_equal(reg[p], ref[(pf[p], mi[p])]), p
    base = rng.normal(0, 2, (11, H, W, 2)).astype(np.float32)
    fi = np.arange(P) % 11
    hinv = np.stack([np.linalg.inv(mats[m]) for m in mi])
    out = solver.flow_unregister(base[fi], hinv, (3, 2))
    for p in list(range(0, P, 997)) + [65534, 65535, 65536]:
        assert np.array_equal(_bits(out[p]), _bits(R.flow_raw_values(base[fi[p]], hinv[p], 3, 2))), p


def test_refusals():
    with pytest.raises(RuntimeError, match="rcvd error 1"):
        solver.homography_warp(np.zeros((1, 4, 4, 3), np.uint8), [1], [np.eye(3)])
    with pytest.raises(ValueError):
        solver.homography_warp(np.zeros((1, 4, 4, 3), np.uint8), [0, 0], [np.eye(3)])
    with pytest.raises(RuntimeError, match="rcvd error 1"):
        solver.flow_unregister(np.zeros((1, 4, 4, 2), np.float32), [np.eye(3)], (0, 3))
    assert solver.homography_warp(np.zeros((1, 4, 4, 3), np.uint8), np.zeros(0, np.int32), np.zeros((0, 9))).shape == (0, 4, 4, 3)


class StubModel:
    """A deterministic torch model with fractional flows that depend on both inputs; records what it receives."""

    def __init__(self):
        self.calls = []

    def __call__(self, img1, img2, iters=None, test_mode=None):
        self.calls.append((img1.detach().cpu().clone(), img2.detach().cpu().clone(), img1.dtype, img1.device.type, img1.is_contiguous(),
                           img2.is_contiguous(), iters, test_mode, torch.is_grad_enabled()))
        _, _, H, W = img1.shape
        yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=img1.device),
                                torch.arange(W, dtype=torch.float32, device=img1.device), indexing="ij")
        d = (img1 - img2).mean(1)[0] / 255
        up = torch.stack([1.7 * torch.sin(xx * 0.05) + 0.25 * d + 0.125, -1.3 * torch.cos(yy * 0.07) - 0.25 * d])[None]
        return up / 8, up


def _scene(root, n=5, size=(72, 128), down=(28, 48)):
    base = GOLDEN["perspective/frame1"]
    base = cv2.resize(base, size[::-1], interpolation=cv2.INTER_LINEAR)
    rng = np.random.default_rng(8)
    os.makedirs(os.path.join(root, "color_flow"))
    os.makedirs(os.path.join(root, "color_down"))
    for f in range(n):
        M = np.eye(3) + (rng.normal(0, [[0.02, 0.02, 2], [0.02, 0.02, 2], [1e-4, 1e-4, 0]]) if f else 0)
        img = base if f == 0 else cv2.warpPerspective(base, M, size[::-1], borderMode=cv2.BORDER_REFLECT)
        if f == n - 1:
            img = np.full_like(base, 90)   # no keypoints: the identity fallback
        cv2.imwrite(os.path.join(root, F.FRAME_FMT.format(f)), img)
    write_raw(os.path.join(root, F.COLOR_FMT.format(0)), np.zeros(down + (3,), np.float32))


def _replay(root, i, j, size):
    """The reference's sequence for pair (i, j), in cv2 and numpy: imread, SIFT, matchKeypoints, warpPerspective, the model on the
    reference's tensors, the un-registration through np.linalg.inv(H).dot, resize_flow and the float32 cast."""
    f1 = cv2.imread(os.path.join(root, F.FRAME_FMT.format(i)))
    f2 = cv2.imread(os.path.join(root, F.FRAME_FMT.format(j)))
    sift = cv2.SIFT_create()
    k1, d1 = sift.detectAndCompute(f1, None)
    k2, d2 = sift.detectAndCompute(f2, None)
    H_BA = np.eye(3)
    try:
        raw = cv2.DescriptorMatcher_create("BruteForce").knnMatch(d2, d1, 2)
        m = [(r[0].trainIdx, r[0].queryIdx) for r in raw if len(r) == 2 and r[0].distance < r[1].distance * 0.75]
        if len(m) > 4:
            p2 = np.float32([k2[q].pt for _, q in m])
            p1 = np.float32([k1[t].pt for t, _ in m])
            H, _ = cv2.findHomography(p2, p1, cv2.RANSAC, 4.0)
            if H is not None:
                np.linalg.inv(H)
                H_BA = H
    except Exception:
        H_BA = np.eye(3)
    reg = cv2.warpPerspective(f2, H_BA, (f1.shape[1], f1.shape[0]))
    t1 = torch.from_numpy(f1).permute(2, 0, 1).contiguous().float()[None]
    t2 = torch.from_numpy(reg).permute(2, 0, 1).contiguous().float()[None]
    with torch.no_grad():
        _, up = StubModel()(t1.cuda(), t2.cuda())
    flow = up[0].permute(1, 2, 0).cpu().numpy()
    Hh, Ww = flow.shape[:2]
    fy, fx = np.mgrid[0:Hh, 0:Ww].astype(np.float32)
    fxx, fyy = fx + flow[:, :, 0], fy + flow[:, :, 1]
    x, y, z = np.linalg.inv(H_BA).dot(np.concatenate((fxx.reshape(1, -1), fyy.reshape(1, -1), np.ones_like(fyy).reshape(1, -1)), 0))
    un = np.concatenate(((x / z).reshape(Hh, Ww, 1) - fx.reshape(Hh, Ww, 1), (y / z).reshape(Hh, Ww, 1) - fy.reshape(Hh, Ww, 1)), 2)
    res = cv2.resize(un, size, interpolation=cv2.INTER_CUBIC) * np.array((size[0] / float(Ww), size[1] / float(Hh))).reshape(1, 1, -1)
    return t1, t2, H_BA, res.astype(np.float32)


def test_compute_flow_end_to_end(tmp_path, capsys):
    root = str(tmp_path)
    _scene(root)
    pairs = [(0, 1), (1, 0), (1, 2), (2, 3), (3, 1), (0, 4), (4, 2), (2, 0)]
    model = StubModel()
    stats = F.compute_flow(root, pairs, model=model, features=cv2.SIFT_create, batch=3)
    assert "Resizing flow to (48, 28)" in capsys.readouterr().out
    assert stats["pairs"] == len(pairs) and len(model.calls) == len(pairs)
    nonident = 0
    for n, (i, j) in enumerate(pairs):
        t1, t2, H_BA, ref = _replay(root, i, j, (48, 28))
        nonident += not np.array_equal(H_BA, np.eye(3))
        a, b, dtype, dev, c1, c2, iters, test_mode, grad = model.calls[n]
        assert torch.equal(a, t1) and torch.equal(b, t2), (i, j)
        assert a.shape == t1.shape and dtype == torch.float32 and dev == "cuda" and c1 and c2
        assert iters == 20 and test_mode is True and grad is False
        got = read_raw(os.path.join(root, F.FLOW_FMT.format(i, j)))
        assert np.array_equal(_bits(got), _bits(ref)), (i, j)
        with open(os.path.join(root, F.FLOW_FMT.format(i, j)), "rb") as f:
            body = f.read()[20:]
        assert body == ref.tobytes()
    assert nonident >= 3

    # all present: nothing runs
    again = StubModel()
    assert F.compute_flow(root, pairs, model=again, features=cv2.SIFT_create)["pairs"] == 0 and not again.calls
    # a partial set: only the missing pairs run, the others are untouched
    mtimes = {p: os.stat(os.path.join(root, F.FLOW_FMT.format(*p))).st_mtime_ns for p in pairs}
    for p in [(1, 2), (4, 2)]:
        os.remove(os.path.join(root, F.FLOW_FMT.format(*p)))
    part = StubModel()
    assert F.compute_flow(root, pairs, model=part, features=cv2.SIFT_create)["pairs"] == 2 and len(part.calls) == 2
    for p in pairs:
        fn = os.path.join(root, F.FLOW_FMT.format(*p))
        if p in [(1, 2), (4, 2)]:
            assert np.array_equal(_bits(read_raw(fn)), _bits(_replay(root, *p, (48, 28))[3]))
        else:
            assert os.stat(fn).st_mtime_ns == mtimes[p]
