#!/usr/bin/env python3
"""Times the flow-consistency masks (robust_cvd_b200.flow.compute_flow_masks, rcvd_flow_masks) on the 300-frame 384 x 224 directory of
bench.py's config 2 (hierarchical2 pairs, written by synthetic_files.write_scene to a temporary directory), with its masks deleted first.

Reports, as one JSON object with the card's name and power limit:
  kernel      device ms per pair of the kernel alone (CUDA events over `--reps` launches on `--kernel-pairs` pairs, inputs resident)
  call        the whole compute_flow_masks call on the host clock, split into read / compute / PNG (encode + write, summed over the
              writer threads) and the time the calling thread waited; a first run and a second one with the files in the page cache
  pair_stats  compute_flow_pair_stats on the new masks
  cpu_baseline  ms per unordered pair of the CPU arithmetic the reference runs (numpy + torch's CPU grid_sample, both directions, no
              file I/O) on this machine's CPU: the reference's own consistent_flow_masks when ROBUST_CVD_DIR names a checkout, else
              tests/flow_masks_ref.py, which restates it
Nothing is written to the tree.

  python tools/bench_flow_masks.py [--frames 300] [--reps 50] [--kernel-pairs 256] [--baseline-pairs 20]"""
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


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"name": name, "power_limit": power, "cpus": os.cpu_count()}


def _baseline_fn():
    ref_dir = os.environ.get("ROBUST_CVD_DIR", "")
    if os.path.isfile(os.path.join(ref_dir, "utils", "consistency.py")):
        import importlib.util
        spec = importlib.util.spec_from_file_location("ref_consistency", os.path.join(ref_dir, "utils", "consistency.py"))
        cons = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(cons)
        return "reference utils/consistency.py", lambda fij, fji, ci, cj: cons.consistent_flow_masks([fij, fji], [ci, cj], 1, 1)
    from tests import flow_masks_ref
    return "tests/flow_masks_ref.py (numpy + torch CPU grid_sample)", lambda fij, fji, ci, cj: flow_masks_ref.flow_masks(fij, fji, ci, cj)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--kernel-pairs", type=int, default=256)
    ap.add_argument("--baseline-pairs", type=int, default=20)
    args = ap.parse_args()
    import warnings
    warnings.filterwarnings("ignore", message="Default grid_sample")
    from robust_cvd_b200 import flow, solver, synthetic, synthetic_files
    from robust_cvd_b200.synthetic_files import read_raw
    W, H = 384, 224
    out = {"what": "flow-consistency masks: robust_cvd_b200.flow.compute_flow_masks", "frames": args.frames, "image": [W, H], "card": _card()}
    root = tempfile.mkdtemp(prefix="rcvd_flowmask_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    try:
        sc = synthetic.Scene(args.frames, W, H, seed=2)
        pairs = synthetic_files.write_scene(sc, root, workers=min(16, os.cpu_count() or 1))
        out["directed_pairs"] = len(pairs)

        def clean():
            shutil.rmtree(os.path.join(root, "flow_mask"), ignore_errors=True)
            if os.path.exists(os.path.join(root, "flow_list.json")):
                os.remove(os.path.join(root, "flow_list.json"))
        clean()
        todo = flow.pairs_to_compute(root)
        out["unordered_pairs"] = len(todo)
        # ---- the kernel alone ----
        sel = todo[:args.kernel_pairs]
        frames = sorted({f for p in sel for f in p}); local = {f: k for k, f in enumerate(frames)}
        colors = np.stack([read_raw(os.path.join(root, flow.COLOR_FMT.format(f))) for f in frames])
        fij = np.stack([read_raw(os.path.join(root, flow.FLOW_FMT.format(i, j))) for i, j in sel])
        fji = np.stack([read_raw(os.path.join(root, flow.FLOW_FMT.format(j, i))) for i, j in sel])
        pf = np.array([[local[i], local[j]] for i, j in sel], np.int32)
        ms = solver.time_flow_masks(colors, pf, fij, fji, reps=args.reps)
        out["kernel"] = {"pairs_per_launch": len(sel), "launches": args.reps, "device_ms_per_launch": ms, "device_us_per_pair": 1e3 * ms / len(sel)}
        # ---- the whole call ----
        runs = []
        for _ in range(2):
            clean()
            s = flow.compute_flow_masks(root)
            runs.append({k: (round(v, 4) if isinstance(v, float) else v) for k, v in s.items()})
        out["call"] = {"first": runs[0], "second": runs[1], "ms_per_pair_second": 1e3 * runs[1]["total_s"] / max(runs[1]["pairs"], 1)}
        t = time.perf_counter()
        import contextlib
        import io
        with contextlib.redirect_stdout(io.StringIO()):
            flow.compute_flow_pair_stats(root, pairs)
        out["pair_stats_s"] = round(time.perf_counter() - t, 4)
        # ---- CPU baseline: the reference's arithmetic per unordered pair, no I/O ----
        name, fn = _baseline_fn()
        fn(fij[0], fji[0], colors[pf[0, 0]], colors[pf[0, 1]])          # warm-up
        n = min(args.baseline_pairs, len(sel))
        t = time.perf_counter()
        for k in range(n):
            fn(fij[k], fji[k], colors[pf[k, 0]], colors[pf[k, 1]])
        cpu_ms = 1e3 * (time.perf_counter() - t) / n
        out["cpu_baseline"] = {"code": name, "ms_per_unordered_pair": cpu_ms, "pairs_timed": n,
                               "whole_directory_s_estimate": cpu_ms * len(todo) / 1e3}
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
