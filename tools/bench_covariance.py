"""Time rcvd_covariance (the selected inversion of the block-Cholesky factor) on the bench workloads and print one JSON line per
workload: the call's wall time and its device phases (factorisation with the rank test, selected inversion, gather and copy-out), the
selected inversion's algorithmic flops and rate against the live fp64 tensor-core peak, and the update flops of one factorisation
beside it.  Frame 0's pose is held (the gauge).  Config 2 asks for every diagonal block and every coupled pair; config 4 for the 600
diagonal blocks (its pair blocks alone would be ~14 GB of host output).  Needs an H100."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
import bench  # noqa: E402
from robust_cvd_b200 import solver  # noqa: E402
from tests import helpers  # noqa: E402

WORKLOADS = {"config2": ("config2_300f_384x224_grid16x12_sep10", True), "config4": ("config4_600f_640x384_grid32x24_sep10", False)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(name, reps):
    wl, with_pairs = WORKLOADS[name]
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case(wl)
    P = solver.Problem(cfg)
    helpers.setup_problem(P, cfg, pairs, offs, rec, med, bench.initial_state(sc, cfg, solver.frame_stride(cfg)))
    N = P.N
    blocks = [(f, f) for f in range(N)]
    if with_pairs:
        for a, b in sorted({(min(a, b), max(a, b)) for a, b in np.asarray(pairs).reshape(-1, 2)}):
            blocks += [(a, b), (b, a)]
    blocks = np.array(blocks, np.int32)
    hold = np.zeros(P.U, bool); hold[:6] = True
    P.covariance(blocks, hold)                       # warm-up: structure, task lists, factorisation graph
    walls, profs = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        P.covariance(blocks, hold)
        walls.append((time.perf_counter() - t0) * 1e3)
        profs.append(P.covariance_profile())
    i = int(np.argsort(walls)[len(walls) // 2])
    prof = profs[i]
    lin = P.profile_linear(reps=1)
    peak = solver.fp64_tensor_peaks()["m16n8k4"]
    tflops = prof["selinv_flops"] / (prof["selinv_ms"] * 1e-3) / 1e12
    return {"workload": wl, "gpu": gpu_info(), "frames": N, "stride": P.stride, "blocks": len(blocks), "wall_ms_median": walls[i],
            "factor_ms": prof["factor_ms"], "selinv_ms": prof["selinv_ms"], "gather_ms": prof["gather_ms"],
            "selinv_gflop": prof["selinv_flops"] / 1e9, "selinv_products": prof["selinv_products"], "selinv_tflops": tflops,
            "fp64_tc_peak_tflops": peak, "share_of_peak": tflops / peak, "factor_update_gflop": lin["gemm_flops"] / 1e9,
            "linear_info": P.linear_info()["device_bytes"], "launches": P.covariance_launches(), "min_pivot": P.last_min_pivot}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="config2,config4")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    for name in args.workloads.split(","):
        print(json.dumps(run(name, args.reps)), flush=True)


if __name__ == "__main__":
    main()
