#!/usr/bin/env python3
"""Times the flow visualisations (robust_cvd_b200.flow.visualize_flow with warp, rcvd_flow_visualize) on the 300-frame 384 x 224
directory of bench.py's config 2 (hierarchical2 pairs, written by synthetic_files.write_scene to a temporary directory).

Reports, as one JSON object with the card's name and power limit and the host's CPU count:
  call          the whole visualize_flow(warp=True) call on the host clock, split into read (flows, masks, colours; reader time) / kernels
                (the rcvd_flow_visualize calls: uploads, both kernels, copy-back) / PNG (encode + write, summed over the writer threads) and
                the time the calling thread waited; a first run and a second one with the inputs in the page cache
  gpu_call      one rcvd_flow_visualize call on `--kernel-pairs` pairs with the inputs in host memory, and its device time from
                torch.profiler (both kernels)
  cpu_baseline  ms per pair of tests/flow_vis_ref.py (the numpy restatement of the reference's arithmetic: both flow colourings, the
                composite and both warps; no file I/O) on this host's CPU, and the directory estimate from it
Nothing is written to the tree.

  python tools/bench_flow_vis.py [--frames 300] [--kernel-pairs 256] [--baseline-pairs 10]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tools.bench_flow_masks import _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--kernel-pairs", type=int, default=256)
    ap.add_argument("--baseline-pairs", type=int, default=10)
    args = ap.parse_args()
    from robust_cvd_b200 import flow, solver, synthetic, synthetic_files
    from robust_cvd_b200.synthetic_files import read_raw
    from tests import flow_vis_ref
    W, H = 384, 224
    out = {"what": "flow visualisations: robust_cvd_b200.flow.visualize_flow(warp=True)", "frames": args.frames, "image": [W, H], "card": _card()}
    root = tempfile.mkdtemp(prefix="rcvd_flowvis_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    try:
        sc = synthetic.Scene(args.frames, W, H, seed=2)
        pairs = synthetic_files.write_scene(sc, root, workers=min(16, os.cpu_count() or 1))
        out["directed_pairs"] = len(pairs)

        def clean():
            for d in ("vis_flow", "vis_flow_warped"):
                shutil.rmtree(os.path.join(root, d), ignore_errors=True)
        clean()
        todo = flow.vis_pairs_to_compute(root, warp=True)
        out["unordered_pairs"] = len(todo)
        # ---- one GPU call, inputs in host memory ----
        sel = todo[:args.kernel_pairs]
        frames = sorted({f for p in sel for f in p}); local = {f: k for k, f in enumerate(frames)}
        colors = np.stack([read_raw(os.path.join(root, flow.COLOR_FMT.format(f))) for f in frames])
        fij = np.stack([read_raw(os.path.join(root, flow.FLOW_FMT.format(i, j))) for i, j in sel])
        fji = np.stack([read_raw(os.path.join(root, flow.FLOW_FMT.format(j, i))) for i, j in sel])
        mij = np.stack([flow._read_mask(os.path.join(root, flow.MASK_FMT.format(i, j))) for i, j in sel])
        mji = np.stack([flow._read_mask(os.path.join(root, flow.MASK_FMT.format(j, i))) for i, j in sel])
        pf = np.array([[local[i], local[j]] for i, j in sel], np.int32)
        solver.flow_visualize(colors, pf, fij, fji, mij, mji, warp=True)          # warm-up
        t = time.perf_counter()
        solver.flow_visualize(colors, pf, fij, fji, mij, mji, warp=True)
        call_ms = 1e3 * (time.perf_counter() - t)
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            solver.flow_visualize(colors, pf, fij, fji, mij, mji, warp=True)
            torch.cuda.synchronize()
        dev = {e.key: e.device_time_total / 1e3 for e in prof.key_averages() if "k_flow_vis" in e.key}
        out["gpu_call"] = {"pairs": len(sel), "host_ms": call_ms, "host_ms_per_pair": call_ms / len(sel),
                           "kernel_device_ms": dev, "kernel_device_us_per_pair": 1e3 * sum(dev.values()) / len(sel)}
        # ---- the whole call ----
        runs = []
        for _ in range(2):
            clean()
            s = flow.visualize_flow(root, warp=True)
            runs.append({k: (round(v, 4) if isinstance(v, float) else v) for k, v in s.items()})
        out["call"] = {"first": runs[0], "second": runs[1], "ms_per_pair_second": 1e3 * runs[1]["total_s"] / max(runs[1]["pairs"], 1)}
        # ---- CPU baseline: the numpy restatement per pair, no I/O ----
        n = min(args.baseline_pairs, len(sel))
        ins = lambda k: (colors[pf[k, 0]], colors[pf[k, 1]], fij[k], fji[k], mij[k], mji[k])
        flow_vis_ref.visualize_pair(*ins(0))                                      # warm-up
        t = time.perf_counter()
        for k in range(n):
            flow_vis_ref.visualize_pair(*ins(k))
        cpu_ms = 1e3 * (time.perf_counter() - t) / n
        out["cpu_baseline"] = {"code": "tests/flow_vis_ref.py (numpy, one pair at a time)", "ms_per_pair": cpu_ms, "pairs_timed": n,
                               "whole_directory_s_estimate_arithmetic_only": cpu_ms * len(todo) / 1e3}
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
