#!/usr/bin/env python3
"""Times the homography-registered flows (robust_cvd_b200.flow.compute_flow: rcvd_homography_warp, rcvd_flow_unregister) on a seeded
300-frame 1024 x 576 color_flow directory (a textured frame under drifting homographies, written to a temporary directory) with the
1766 hierarchical2 pairs of tests/golden/hierarchical2_pairs.json, and color_down at 384 x 224.

The flow model is a stub (a few elementwise torch ops on the GPU) and the features are cv2.SIFT_create: RAFT needs weights and SURF
needs opencv-contrib, neither of which is here, so neither RAFT's nor SURF's time is measured.  Reports, as one JSON object with the
card's name and power limit:
  kernels       device ms per pair of each kernel alone (CUDA events over `--reps` passes on `--kernel-pairs` pairs, inputs resident)
  call          the whole compute_flow call on the host clock, with its split (stub model, kernels with their copies, waits on
                decoding, SIFT and matching)
  cpu_baseline  ms per pair of the reference's non-model per-pair work restated on this host: two cv2.imread, cv2.warpPerspective, the
                numpy un-registration, resize_flow and the .raw write, over `--baseline-pairs` pairs (features and matching excluded)
Nothing is written to the tree.

  python tools/bench_flow.py [--frames 300] [--reps 20] [--kernel-pairs 64] [--baseline-pairs 40]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

W, H, DOWN = 1024, 576, (384, 224)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"name": name, "power_limit": power, "cpus": os.cpu_count()}


def _write_dir(root, frames):
    import cv2
    from robust_cvd_b200 import flow as F
    from robust_cvd_b200.synthetic_files import write_raw
    rng = np.random.default_rng(0)
    img = np.zeros((H, W, 3))
    for s in (2, 5, 13, 41):
        img += cv2.resize(rng.random((H // s + 2, W // s + 2, 3)), (W, H), interpolation=cv2.INTER_CUBIC) * s
    base = np.clip((img - img.min()) / (img.max() - img.min()) * 255, 0, 255).astype(np.uint8)
    os.makedirs(os.path.join(root, "color_flow"))
    os.makedirs(os.path.join(root, "color_down"))
    M = np.eye(3)
    for f in range(frames):
        cv2.imwrite(os.path.join(root, F.FRAME_FMT.format(f)), cv2.warpPerspective(base, M, (W, H), borderMode=cv2.BORDER_REFLECT))
        M = M @ (np.eye(3) + rng.normal(0, [[2e-3, 2e-3, 0.8], [2e-3, 2e-3, 0.8], [2e-6, 2e-6, 0]]))
    write_raw(os.path.join(root, F.COLOR_FMT.format(0)), np.zeros((DOWN[1], DOWN[0], 3), np.float32))


def stub_model(img1, img2, iters=20, test_mode=True):
    import torch
    d = (img1 - img2).mean(1, keepdim=True) / 255
    up = torch.cat([0.25 * d + 0.125, -0.25 * d - 0.375], 1)
    return up / 8, up


def _baseline(root, pairs):
    """The reference's per-pair work besides the model and the features, restated: two imreads, the warp, the un-registration in numpy,
    resize_flow and the write."""
    import cv2
    from robust_cvd_b200 import flow as F
    from robust_cvd_b200.synthetic_files import write_raw
    rng = np.random.default_rng(1)
    out = os.path.join(root, "baseline.raw")
    t = time.perf_counter()
    for i, j in pairs:
        f1 = cv2.imread(os.path.join(root, F.FRAME_FMT.format(i)))
        f2 = cv2.imread(os.path.join(root, F.FRAME_FMT.format(j)))
        H_BA = np.eye(3) + rng.normal(0, [[1e-2, 1e-2, 2], [1e-2, 1e-2, 2], [1e-5, 1e-5, 0]])
        cv2.warpPerspective(f2, H_BA, (W, H))
        flow = rng.normal(0, 2, (H, W, 2)).astype(np.float32)
        fy, fx = np.mgrid[0:H, 0:W].astype(np.float32)
        fxx, fyy = fx + flow[:, :, 0], fy + flow[:, :, 1]
        x, y, z = np.linalg.inv(H_BA).dot(np.concatenate((fxx.reshape(1, -1), fyy.reshape(1, -1), np.ones_like(fyy).reshape(1, -1)), 0))
        un = np.concatenate(((x / z).reshape(H, W, 1) - fx.reshape(H, W, 1), (y / z).reshape(H, W, 1) - fy.reshape(H, W, 1)), 2)
        res = cv2.resize(un, DOWN, interpolation=cv2.INTER_CUBIC) * np.array((DOWN[0] / W, DOWN[1] / H)).reshape(1, 1, -1)
        write_raw(out, res.astype(np.float32))
    return (time.perf_counter() - t) / len(pairs) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--kernel-pairs", type=int, default=64)
    ap.add_argument("--baseline-pairs", type=int, default=40)
    a = ap.parse_args()
    import cv2
    import torch
    from robust_cvd_b200 import flow as F
    from robust_cvd_b200 import solver
    with open(os.path.join(ROOT, "tests", "golden", "hierarchical2_pairs.json")) as f:
        pairs = [tuple(p) for p in json.load(f)[str(a.frames)]]
    res = {"card": _card(), "frames": a.frames, "pairs": len(pairs), "size": [W, H], "down": list(DOWN)}

    rng = np.random.default_rng(2)
    P = a.kernel_pairs
    frames = rng.integers(0, 256, (8, H, W, 3), np.uint8)
    mats = [np.eye(3) + rng.normal(0, [[1e-2, 1e-2, 2], [1e-2, 1e-2, 2], [1e-5, 1e-5, 0]]) for _ in range(P)]
    flows = rng.normal(0, 2, (P, H, W, 2)).astype(np.float32)
    warp_ms = solver.time_homography_warp(frames, np.arange(P) % 8, [F.cv_invert3(m) for m in mats], reps=a.reps)
    unreg_ms = solver.time_flow_unregister(flows, [np.linalg.inv(m) for m in mats], DOWN, reps=a.reps)
    res["kernels"] = {"homography_warp_us_per_pair": warp_ms / P * 1e3, "flow_unregister_us_per_pair": unreg_ms / P * 1e3}

    tmp = tempfile.mkdtemp(prefix="bench_flow_")
    try:
        t = time.perf_counter()
        _write_dir(tmp, a.frames)
        res["write_dir_s"] = time.perf_counter() - t
        torch.cuda.synchronize()
        st = F.compute_flow(tmp, pairs, model=stub_model, features=cv2.SIFT_create)
        res["call"] = st
        res["call_ms_per_pair"] = st["total_s"] / len(pairs) * 1e3
        res["cpu_baseline_ms_per_pair"] = _baseline(tmp, pairs[:a.baseline_pairs])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
