"""The long fine-grid video that the block Cholesky cannot hold: 1000 frames at 640x384 with a 32x24 depth grid (npad 784), hierarchical2
pairs, matchSeparation 10 -- the config-4 scene of bench.py over 1000 frames, built with robust_cvd_b200/synthetic.py.  Its factor would
take ~107 GB, so the handle solves with block-Jacobi preconditioned conjugate gradients (robust_cvd_b200/csrc/rcvd_cg.cuh).  Prints one
JSON line: the card and its power limit (read in the same run), the linear solver's device bytes, CG iterations per LM step, linear ms
per LM iteration, and the achieved bandwidth of the CG matrix product (H streamed once per product) against the H100 SXM's 3.35 TB/s.
With --compare-frames > 0 it also runs config 2 (300 frames, 16x12 grid) twice with the same LM iteration cap, once on the block
Cholesky the handle chooses and once forced to CG, and reports linear ms and final cost side by side.

Usage: python tools/bench_long.py [--frames 1000] [--lm-iterations 10] [--compare-frames 300]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from robust_cvd_b200 import abi, solver  # noqa: E402
from tests import helpers  # noqa: E402

HBM_PEAK_GBS = 3350.0   # H100 SXM data sheet, HBM3


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm,memory.total", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, sm, mem = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "sm_max_clock": sm, "memory": mem}


def problem(workload, frames):
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case(workload, frames=frames)
    P = solver.Problem(cfg)
    helpers.setup_problem(P, cfg, pairs, offs, rec, med, bench.initial_state(sc, cfg, solver.frame_stride(cfg)))
    return P, len(pairs), int(rec.shape[0])


def run(P, lm_iterations):
    opt = abi.default_solve_options(max_iterations=lm_iterations)
    opt.initial_radius = 1.0          # as tests/test_gpu_parity_at_size.py: Ceres' 1e4 spends the first iterations shrinking the region here
    t = time.perf_counter()
    s = P.solve(opt)
    wall = time.perf_counter() - t
    info = P.linear_info()
    it = max(s.iterations, 1)
    out = {"lm_iterations": s.iterations, "successful_steps": s.num_successful_steps, "initial_cost": s.initial_cost, "final_cost": s.final_cost,
           "linear_ms_per_lm_iteration": s.linear_ms / it, "eval_ms_total": s.eval_ms, "solve_wall_s": wall,
           "solver": "cg" if info["solver"] == abi.LINEAR_CG else "cholesky", "linear_device_bytes": info["device_bytes"],
           "cholesky_bytes_needed": info["cholesky_bytes"]}
    if info["solver"] == abi.LINEAR_CG:
        out.update({"cg_iterations_total": info["cg_iterations"], "cg_iterations_per_step": info["cg_iterations"] / max(info["cg_solves"], 1),
                    "cg_iterations_max": info["cg_max_iterations"], "cg_capped_steps": info["cg_capped_steps"]})
    return out


def product_bandwidth(P, reps):
    """Achieved GB/s of one CG product: the H blocks' nf x nf interiors read once, the row and the column slot of every block written
    and read back (nf each), S, D2, the direction and the result."""
    st = P.structure_info()
    nf, npad, N, nH = st["stride"], st["npad"], st["frames"], st["h_blocks"]
    ms = P.time_cg_product(reps)
    nbytes = 8.0 * (nH * nf * nf + 2 * 2 * nH * nf + 4 * N * npad)
    return {"product_ms": ms, "product_bytes": nbytes, "achieved_GBps": nbytes / ms / 1e6, "share_of_hbm_peak": nbytes / ms / 1e6 / HBM_PEAK_GBS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--lm-iterations", type=int, default=10)
    ap.add_argument("--product-reps", type=int, default=20)
    ap.add_argument("--compare-frames", type=int, default=300, help="config-2 frames of the Cholesky / CG comparison (0: skip)")
    args = ap.parse_args()
    line = {"card": card()}
    P, npairs, ncons = problem("config4_600f_640x384_grid32x24_sep10", args.frames)
    line["long"] = {"frames": args.frames, "image": [640, 384], "depth_grid": [32, 24], "pairs": npairs, "constraints": ncons, **run(P, args.lm_iterations)}
    if line["long"]["solver"] == "cg":
        line["long"].update(product_bandwidth(P, args.product_reps))
    P.close()
    if args.compare_frames > 0:
        cmp = {}
        for name, budget in (("cholesky", -1), ("cg", 0)):
            Q, _, _ = problem("config2_300f_384x224_grid16x12_sep10", args.compare_frames)
            Q.set_factor_budget(budget)
            cmp[name] = run(Q, args.lm_iterations)
            Q.close()
        line["config2"] = {"frames": args.compare_frames, **cmp}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
