"""Runs a couple of LM-iteration-equivalents of the bench workload (for ncu launch lists / captures)."""
import argparse, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import bench
from robust_cvd_b200 import solver

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="config2_300f_384x224_grid16x12_sep10")
ap.add_argument("--frames", type=int, default=None)
ap.add_argument("--sep", type=int, default=None)
ap.add_argument("--iters", type=int, default=1)
ap.add_argument("--accumulate-only", action="store_true")
ap.add_argument("--slack", type=int, default=None)
ap.add_argument("--no-overlap", action="store_true")
ap.add_argument("--classes", action="store_true", help="also print the serialised per-kernel-class times")
a = ap.parse_args()
spec, sc, cfg, pairs, offs, rec, med = bench.build_case(a.workload, frames=a.frames, sep=a.sep)
P = solver.Problem(cfg)
if a.slack is not None: P.set_order_slack(a.slack)
if a.no_overlap: P.set_overlap(False)
P.set_frames(np.ones(cfg.num_frames, np.uint8), med); P.set_constraints(pairs, offs, rec); P.set_state(bench.initial_state(sc, cfg, P.stride))
if a.accumulate_only:
    print("accumulate ms", P.time_accumulate(iters=a.iters))
else:
    print(P.time_iteration(iters=a.iters), P.structure_info(), "C", rec.shape[0])
    if a.classes:
        pl = P.profile_linear(reps=3)
        pl["gemm_tflops"] = pl["gemm_flops"] / (pl["gemm_ms"] * 1e-3) / 1e12
        print({k: round(v, 3) if v < 1e6 else v for k, v in pl.items()})
        pl = P.profile_linear(reps=-3)
        print("overlapped, main-stream view:", {k: round(v, 3) if v < 1e6 else v for k, v in pl.items()}, "sum", round(sum(pl[k] for k in ("load_ms", "potrf_ms", "trinv_ms", "trsm_ms", "gemm_ms", "solve_ms")), 3))
