"""Times FlowConstraintsCollection.pruneStaticFlag through lib_python at config-2 size: 300 frames at 384 x 224, hierarchical2 pairs,
moving dynamic blobs, constraints from the GPU builder, then setStaticFlagFromDynamicMask(8) and pruneStaticFlag(d) for d = 5 (the
trackPruneDistance default) and 20.  The device path (default) and the sequential host restatement (RCVD_CONSTRAINT_BUILDER=host)
are timed in alternating runs after a warm-up, and their flags are compared.  Kernel times come from torch.profiler in a separate run.
The scene is written to a temporary directory; nothing is written to the tree.

  python tools/bench_prune.py [--reps 5] [--frames 300]"""
import argparse
import os
import statistics
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))
import numpy as np  # noqa: E402

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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=300)
    args = ap.parse_args()
    N = args.frames
    name, limit = card()
    import lib_python as lp
    with tempfile.TemporaryDirectory() as tmp:
        sc = synthetic.Scene(N, W, H, seed=2)
        root = os.path.join(tmp, "scene")
        t = time.perf_counter()
        pairs = synthetic_files.write_scene(sc, root, dynamic_masks=list(masks(N)), workers=min(8, os.cpu_count() or 1))
        print(f"scene written in {time.perf_counter() - t:.1f} s: {N} frames {W}x{H}, {len(pairs)} hierarchical2 pairs")
        v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
        v.createColorStream("down", "color_down", ".raw", CV_32FC3); v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
        fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True); fp.doNotUseCache = True
        os.environ.pop("RCVD_CONSTRAINT_BUILDER", None)
        fc = lp.FlowConstraintsCollection(v, fp)
        n_pairs = sum(len(a[0]) for a in fc._pairs().values()); n_trips = sum(len(a[0]) for a in fc._triplets().values())

        def flags():
            return (np.concatenate([np.asarray(a[1]) for _, a in sorted(fc._pairs().items())]),
                    np.concatenate([np.asarray(a[1]) for _, a in sorted(fc._triplets().items())]))

        def prune(which, d):
            os.environ.pop("RCVD_CONSTRAINT_BUILDER", None)
            fc.setStaticFlagFromDynamicMask(8)                  # fresh input flags, on the device
            os.environ["RCVD_CONSTRAINT_BUILDER"] = which
            t0 = time.perf_counter()
            fc.pruneStaticFlag(d)
            dt = time.perf_counter() - t0
            os.environ.pop("RCVD_CONSTRAINT_BUILDER", None)
            return dt
        os.environ.pop("RCVD_CONSTRAINT_BUILDER", None)
        fc.setStaticFlagFromDynamicMask(8)
        dyn = int((~flags()[0]).sum())
        print(f"card: {name}, power limit {limit}; {n_pairs} pair and {n_trips} triplet constraints, {dyn} pair constraints non-static after "
              f"setStaticFlagFromDynamicMask(8)")
        for d in (5, 20):
            prune("gpu", d); prune("host", d)                    # warm-up of both paths
            times = {"gpu": [], "host": []}
            result = {}
            for _ in range(args.reps):
                for which in ("gpu", "host"):
                    times[which].append(prune(which, d))
                    result[which] = flags()
            same = all(np.array_equal(a, b) for a, b in zip(result["gpu"], result["host"]))
            pruned = int((~result["gpu"][0]).sum()) - dyn
            g, h = (statistics.median(times[k]) * 1e3 for k in ("gpu", "host"))
            print(f"pruneStaticFlag({d}): device {g:.2f} ms (runs {', '.join(f'{x * 1e3:.2f}' for x in times['gpu'])}), host {h:.2f} ms "
                  f"(runs {', '.join(f'{x * 1e3:.2f}' for x in times['host'])}); medians of {args.reps} alternating runs; "
                  f"{pruned} more pair constraints non-static; device flags {'equal to' if same else 'DIFFERENT FROM'} host")
            assert same
            try:
                os.environ.pop("RCVD_CONSTRAINT_BUILDER", None)
                fc.setStaticFlagFromDynamicMask(8)
                km = kernel_ms(lambda: fc.pruneStaticFlag(d))
                print(f"  kernels of one device call ({sum(km.values()):.3f} ms in all):", ", ".join(f"{k} {v:.3f}" for k, v in sorted(km.items(), key=lambda kv: -kv[1])))
            except Exception as err:                                    # the profiler is a side measurement
                print(f"  (torch.profiler unavailable: {err})")
        print(f"measured on {name} at a {limit} power limit")


if __name__ == "__main__":
    main()
