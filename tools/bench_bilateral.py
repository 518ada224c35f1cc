"""Times the joint depth / colour bilateral filter (rcvd_bilateral_filter, host buffers in/out) at config-2 size (300 frames, 384 x 224)
in four settings, and checks a few frames of each against the float32 restatement (tests/bilateral_ref.py::bilateral_filter).

Per setting: wall ms per frame of the whole call (host-to-device copies of the stacks, kernels, copy back), device ms per frame of its
kernels alone (torch.profiler), samples/s of the kernels, and the HBM bound: the stack bytes read once plus the output written once at
3.35 TB/s (H100 SXM data sheet).  Writes nothing.

  python tools/bench_bilateral.py [--reps 3]"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tests import bilateral_ref  # noqa: E402
from robust_cvd_b200 import abi, solver  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
F, W, H = 300, 384, 224
SETTINGS = [  # name, kwargs (the defaults first: r 0, frame radius 2, depthSigma 0.3, mean, in place)
    ("defaults (r0 fr2 sd0.3 mean, in place)", dict(spatial_radius=0, frame_radius=2, depth_sigma=0.3, color_sigma=0.0, median=False, in_place=True)),
    ("r2 fr2 sd0.3 sc0.1 mean", dict(spatial_radius=2, frame_radius=2, depth_sigma=0.3, color_sigma=0.1, median=False)),
    ("r2 fr2 sd0.3 sc0.1 median", dict(spatial_radius=2, frame_radius=2, depth_sigma=0.3, color_sigma=0.1, median=True)),
    ("r5 fr3 sd0.3 median", dict(spatial_radius=5, frame_radius=3, depth_sigma=0.3, color_sigma=0.0, median=True)),
]


def stacks(seed=0):
    rng = np.random.default_rng(seed)
    iy, ix = np.mgrid[0:H, 0:W].astype(np.float32)
    t = np.arange(F, dtype=np.float32)[:, None, None]
    depth = (1.5 + 0.5 * np.sin(ix * 0.031 + t * 0.05) * np.cos(iy * 0.047 - t * 0.03) + rng.normal(0, 0.05, (F, H, W))).astype(np.float32)
    color = (0.5 + 0.3 * np.sin(ix[..., None] * np.array([0.11, 0.07, 0.05], np.float32) + t[..., None] * 0.1)
             + rng.normal(0, 0.05, (F, H, W, 3))).astype(np.float32)
    return depth, color


def samples(frame_radius, r):
    ax = lambda n: (np.minimum(np.arange(n) + r, n - 1) - np.maximum(np.arange(n) - r, 0) + 1).astype(np.int64)   # noqa: E731
    spatial = int(ax(H).sum() * ax(W).sum())
    return sum(min(F - 1, f + frame_radius) - max(0, f - frame_radius) + 1 for f in range(F)) * spatial


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        limit = "unknown"
    return name, limit


def kernel_ms(fn):
    """Device time of the kernels one call launches (k_bilateral_* and, in place, k_dense), from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    total = 0.0
    for e in prof.events():
        if e.device_type.name == "CUDA" and ("bilateral" in e.name or "k_dense" in e.name):
            total += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    return total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check-frames", type=int, default=2)
    args = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}; {F} frames {W}x{H}; HBM bound at {HBM_BYTES_PER_S / 1e12:.2f} TB/s")
    depth, color = stacks()
    cfg = abi.default_config(1, W / H)                         # Global Scale depth transform
    scale = np.linspace(0.8, 1.2, F).reshape(-1, 1)
    out_frames = list(range(F))
    plane = W * H
    for label, kw in SETTINGS:
        kw = dict(kw)
        in_place = kw.pop("in_place", False)
        extra = dict(in_place=True, xform_cfg=cfg, xform_params=scale) if in_place else {}
        col = color if kw["color_sigma"] > 0 else None
        call = lambda: solver.bilateral_filter(depth, out_frames, col, **kw, **extra)   # noqa: E731
        call()                                                  # warm-up
        ts = []
        for _ in range(args.reps):
            t = time.perf_counter(); out = call(); ts.append(time.perf_counter() - t)
        wall = min(ts)
        try:
            dev = kernel_ms(call) / 1e3
        except Exception as err:                                # the profiler is a side measurement
            print(f"  (torch.profiler unavailable: {err})"); dev = float("nan")
        S = samples(kw["frame_radius"], kw["spatial_radius"])
        bytes_once = F * plane * 4 * (4 if col is not None else 1) + F * plane * 4
        print(f"{label}: wall {wall * 1e3 / F:.3f} ms/frame ({wall * 1e3:.1f} ms per call), kernels {dev * 1e3 / F:.4f} ms/frame, "
              f"{S / dev / 1e9:.2f} G samples/s, HBM bound {bytes_once / HBM_BYTES_PER_S * 1e3 / F:.4f} ms/frame "
              f"(kernels at {bytes_once / HBM_BYTES_PER_S / dev * 100:.1f}% of it)")
        # a few frames against the restatement; in place the first frames (the recurrence starts at frame 0)
        k = args.check_frames
        sub = slice(0, k + kw["frame_radius"])
        fr = list(range(k))
        want = bilateral_ref.bilateral_filter(depth[sub], fr, None if col is None else col[sub], **kw,
                                              retransform=(lambda f, img: solver.depth_apply(cfg, scale[f], img)) if in_place else None)
        got = out[:k]
        if kw["median"]:
            eq = (got == want).mean()
            print(f"  check: {k} frames, {eq * 100:.3f}% of pixels bit-equal to the restatement")
            assert eq >= 0.995
        else:
            rel = float(np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-30)))
            print(f"  check: {k} frames, max relative difference to the restatement {rel:.2e}")
            assert rel <= 1e-5


if __name__ == "__main__":
    main()
