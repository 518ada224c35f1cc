#!/usr/bin/env python3
"""Depth normalisation wall-clock in both modes: `DepthVideoProcessor.normalizeDepth` through lib_python with
normalizeDepthFromFirstFrame = true (the scale regulariser alone, frame 0's transform copied to all) and = false (one
DisparityDissimilarityCost row per flow constraint, k_depth_pairs), on a synthetic scene written to disk (default: 300 frames,
384 x 224, hierarchical2 pairs, Global/Scale transforms -- the size of bench.py's config 2).

  python tools/bench_normalize.py [--frames 300] [--runs 3] [--max-iterations 1000] [--keep DIR]

Per mode: the whole call timed with the host clock (the call ends in a device synchronise: the state is read back), a warm-up call
first, then alternating runs; the per-solve split (eval / linear / cost ms, iterations) from the solver summary of a replay of the same
problem arrays through the C ABI; in a separate run, the device time of k_depth_pairs from torch.profiler.  Prints one JSON object with
the card's name and power limit.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

CV_32FC3 = 21


def _open(lp, root):
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", CV_32FC3)
    v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
    return v


def _params(lp, v, frames, max_iterations, pairwise):
    params = lp.DepthVideoProcessor.Params()
    params.depthStream = v.numDepthStreams() - 1
    fs = f"0-{frames - 1}"
    params.frameRange.fromString(fs); params.poseOptimizer.frameRange.fromString(fs)
    params.poseOptimizer.maxIterations = max_iterations
    params.poseOptimizer.normalizeDepthFromFirstFrame = not pairwise
    params.op = lp.DepthVideoProcessor.Op.ResetDepthXforms
    params.depthXformDesc.type = lp.XformType.Depth; params.depthXformDesc.depthType = lp.DepthXformType.Global; params.depthXformDesc.valueXform = lp.ValueXformType.Scale
    return params


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"name": name, "power_limit_and_max_sm_clock": power}


def run(frames=300, w=384, h=224, runs=3, max_iterations=1000, keep=None, seed=2):
    import lib_python as lp
    from robust_cvd_b200 import abi, solver, synthetic, synthetic_files
    out = {"frames": frames, "image": [w, h], "card": _card(), "max_iterations": max_iterations,
           "what": "DepthVideoProcessor.normalizeDepth, Global/Scale, Cauchy 0.5, scaleReg 1, lower bound 0; first-frame vs pairwise"}
    root = keep or tempfile.mkdtemp(prefix="rcvd_norm_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    try:
        sc = synthetic.Scene(frames, w, h, seed=seed)
        out["pairs"] = len(synthetic_files.write_scene(sc, root, workers=min(16, os.cpu_count() or 1)))
        v = _open(lp, root)
        fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True); fp.doNotUseCache = True
        fc = lp.FlowConstraintsCollection(v, fp)
        fc.resetStaticFlag()
        out["constraints"] = int(sum(len(x[0]) for x in fc._pairs().values()))
        modes = {"first_frame": False, "pairwise": True}

        def call(pairwise):
            vv = _open(lp, root); proc = lp.DepthVideoProcessor(vv); params = _params(lp, vv, frames, max_iterations, pairwise)
            proc.process(params)
            t0 = time.perf_counter()
            proc.normalizeDepth(params, fc)
            dt = time.perf_counter() - t0
            ds = vv.depthStream(params.depthStream)
            return dt, np.array([ds.frame(f).depthXform().params()[0] for f in range(frames)])

        for pw in modes.values():              # warm-up: module load and pool growth of the first call in the process
            call(pw)
        times = {m: [] for m in modes}; scales = {}
        for _ in range(runs):                  # alternating
            for m, pw in modes.items():
                dt, s = call(pw); times[m].append(dt); scales[m] = s
        out["normalize_depth_s"] = {m: {"median": float(np.median(t)), "min": float(np.min(t)), "runs": t} for m, t in times.items()}
        out["scales"] = {m: {"min": float(s.min()), "max": float(s.max()), "distinct": int(np.unique(s).size)} for m, s in scales.items()}
        # per-solve split: the same problem arrays through the C ABI
        split = {}
        for m, pw in modes.items():
            vv = _open(lp, root); proc = lp.DepthVideoProcessor(vv); params = _params(lp, vv, frames, max_iterations, pw); proc.process(params)
            d = lp.DepthVideoPoseOptimizer(vv, params.depthStream)._buildProblem(params.poseOptimizer, fc, 0.0, True)
            cfg = abi.Config.from_buffer_copy(d["config"])
            G = solver.Problem(cfg, device=0)
            G.set_frames(d["in_range"], d["median"])
            if pw:
                G.set_depth_pairs(d["dpair_frames"], d["dpair_offsets"], d["dpair_records"])
            G.set_state(d["state"])
            s = G.solve(abi.default_solve_options(max_iterations=max_iterations))
            split[m] = {"iterations": s.iterations, "total_ms": s.total_ms, "eval_ms": s.eval_ms, "linear_ms": s.linear_ms, "cost_ms": s.cost_ms,
                        "kernel_launches": int(s.gpu_launches), "depth_pair_constraints": int(d["dpair_offsets"][-1]),
                        "termination": s.termination, "initial_cost": s.initial_cost, "final_cost": s.final_cost}
            if pw:
                keep_arrays = (cfg, d)
        out["solve_split"] = split
        # kernel time of k_depth_pairs (separate run: the profiler slows the host)
        import torch
        from torch.profiler import ProfilerActivity, profile
        cfg, d = keep_arrays
        G = solver.Problem(cfg, device=0)
        G.set_frames(d["in_range"], d["median"]); G.set_depth_pairs(d["dpair_frames"], d["dpair_offsets"], d["dpair_records"]); G.set_state(d["state"])
        G.solve(abi.default_solve_options(max_iterations=2))      # warm
        G.set_state(d["state"])
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            G.solve(abi.default_solve_options(max_iterations=max_iterations))
            torch.cuda.synchronize()
        kern = {}
        modes_of = ["Cost", "CostGrad", "CostGradH", "MarkActive"]      # rcvd::EvalMode
        for e in prof.events():
            if "k_depth_pairs" in e.name:
                m = re.search(r"EvalMode\)(\d)|EvalModeE(\d)", e.name)
                mode = modes_of[int(m.group(1) or m.group(2))] if m else e.name
                k = kern.setdefault(mode, {"launches": 0, "device_us": 0.0})
                k["launches"] += 1; k["device_us"] += e.device_time
        C = int(d["dpair_offsets"][-1])
        for k in kern.values():
            k["us_per_launch"] = k["device_us"] / max(k["launches"], 1)
            k["input_bytes_per_launch"] = 24 * C
            k["input_GB_per_s"] = 24 * C / (k["us_per_launch"] * 1e-6) / 1e9 if k["us_per_launch"] > 0 else None
        out["k_depth_pairs"] = kern
        out["cpu_baseline"] = "not measured"
        return out
    finally:
        if keep is None:
            shutil.rmtree(root, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--width", type=int, default=384)
    ap.add_argument("--height", type=int, default=224)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--max-iterations", type=int, default=1000)
    ap.add_argument("--keep", default=None)
    a = ap.parse_args()
    print(json.dumps(run(a.frames, a.width, a.height, a.runs, a.max_iterations, a.keep)))


if __name__ == "__main__":
    main()
