"""Times the long point tracker (DepthVideoProcessor::computeTracks on the GPU) at config-2 size: 300 frames at 384 x 224 with the
consecutive flows written by synthetic_files.write_scene, default Params (spawn 20, prune 5, min dynamic distance 3, min length 4),
without and with dynamic masks.  Checks the first frames against the float32 restatement (tests/tracks_ref.py).

Per setting: wall ms of the C ABI call (rcvd_compute_tracks from host stacks: colour upload, kernels, frame loop, copy back), wall ms
of lib_python's computeTracks including the file reads, and device ms per kernel from torch.profiler in a separate run.  The scene is
written to a temporary directory; nothing is written to the tree.

  python tools/bench_tracks.py [--reps 3] [--frames 300]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))
import numpy as np  # noqa: E402

from tests import tracks_ref  # noqa: E402
from robust_cvd_b200 import solver, synthetic, synthetic_files  # noqa: E402

W, H = 384, 224
CV_8UC1, CV_32FC3 = 0, 21


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        limit = "unknown"
    return name, limit


def masks(N, seed=1):
    """A few moving dynamic blobs per frame (< 127 = dynamic)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    c = rng.uniform([0, 0], [H, W], (4, 2)); v = rng.normal(0, 1.5, (4, 2)); r = rng.uniform(10, 30, 4)
    m = np.full((N, H, W), 255, np.uint8)
    for f in range(N):
        for k in range(4):
            cy, cx = (c[k] + f * v[k]) % [H, W]
            m[f][(yy - cy) ** 2 + (xx - cx) ** 2 <= r[k] ** 2] = 0
    return m


def kernel_ms(fn):
    """Device ms per kernel name of one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out = defaultdict(float)
    for e in prof.events():
        if e.device_type.name == "CUDA":
            out[e.name.split("(")[0].split("<")[0]] += (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--check-frames", type=int, default=4)
    args = ap.parse_args()
    N = args.frames
    name, limit = card()
    print(f"card: {name}, power limit {limit}; {N} frames {W}x{H}, default Params")
    import lib_python as lp
    with tempfile.TemporaryDirectory() as tmp:
        sc = synthetic.Scene(N, W, H, seed=2)
        root = os.path.join(tmp, "scene")
        t = time.perf_counter()
        synthetic_files.write_scene(sc, root, pairs=[(i, i + 1) for i in range(N - 1)], dynamic_masks=masks(N), workers=min(8, os.cpu_count() or 1))
        print(f"scene written in {time.perf_counter() - t:.1f} s")
        for dynamic in (False, True):
            label = "with dynamic masks" if dynamic else "no dynamic mask"
            kw = dict(spawn_distance=20, prune_distance=5, min_dynamic_distance=3, inv_aspect=sc.inv_aspect32)
            color, flags, flow, fmask, dyn = tracks_ref.load_inputs(root, list(range(N)), W, H, dynamic=dynamic)
            call = lambda: solver.compute_tracks(color, flags, flow, fmask, dyn, **kw)   # noqa: E731
            call()
            ts = []
            for _ in range(args.reps):
                t = time.perf_counter(); off, ids, locs, n = call(); ts.append(time.perf_counter() - t)

            def lib_call():
                v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
                v.createColorStream("down", "color_down", ".raw", CV_32FC3)
                if dynamic:
                    v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
                p = lp.DepthVideoProcessor.Params(); p.frameRange.fromString(f"0-{N - 1}")
                return lp.DepthVideoProcessor(v).computeTracks(p)
            lib_call()
            tl = []
            for _ in range(args.reps):
                t = time.perf_counter(); table = lib_call(); tl.append(time.perf_counter() - t)
            kept = sum(tr is not None for tr in table._tracks())
            print(f"{label}: C ABI call {min(ts) * 1e3:.1f} ms ({min(ts) * 1e3 / N:.3f} ms/frame; runs {', '.join(f'{x * 1e3:.1f}' for x in ts)}), "
                  f"lib_python computeTracks with file reads {min(tl) * 1e3:.1f} ms; {n} ids created, {kept} kept (length >= 4), "
                  f"{off[-1]} observations, {off[-1] / N:.0f} live tracks per frame")
            try:
                km = kernel_ms(call)
                tot = sum(km.values())
                print(f"  kernels {tot:.1f} ms in all:", ", ".join(f"{k} {v:.2f}" for k, v in sorted(km.items(), key=lambda kv: -kv[1])[:10]))
            except Exception as err:                                    # the profiler is a side measurement
                print(f"  (torch.profiler unavailable: {err})")
            # frames 0 .. K-2 of a K-frame run are those of the full run (only the last frame of a range does not spawn)
            K = args.check_frames
            sub = dict(color=color[:K], flags=flags[:K], flow=flow[:K], flow_mask=fmask[:K], dyn_masks=None if dyn is None else dyn[:K])
            tracks, _ = tracks_ref.compute_tracks(**sub, **kw)
            roff, rids, rlocs = tracks_ref.frame_lists(tracks, K)
            m = int(roff[K - 1])
            assert np.array_equal(off[:K], roff[:K])
            assert np.array_equal(ids[:m], rids[:m]) and locs[:m].tobytes() == rlocs[:m].tobytes()
            print(f"  check: frames 0-{K - 2} ({m} observations) equal to the restatement")


if __name__ == "__main__":
    main()
