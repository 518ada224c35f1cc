#!/usr/bin/env python3
"""Times the depth visualisation (robust_cvd_b200.visualization.visualize_depth_dir, rcvd_depth_visualize) on a seeded directory of
`--frames` float32 .raw disparities of `--width` x `--height` (default 300 frames of 384 x 224 with a few NaN pixels, written to a
temporary directory), at save_depth's settings (percentiles 0 / 100, force, the PNGs written next to the .raw files).

Reports, as one JSON object with the card's name and power limit and the host's CPU count:
  kernel     device time per frame of the range pass and of the colour pass (rcvd_debug_time_depth_visualize: CUDA events over
             `--reps` passes over all the frames, resident on the device)
  call       the whole visualize_depth_dir on the host clock, split into reads (reader time), GPU calls (uploads, kernels, copy-back) and
             PNG encoding and writing (summed over the writer threads); a first run and a second one
  numpy      the numpy restatement tests/depth_vis_ref.py (np.percentile per frame, then the index and the colour table per frame) on
             the frames in memory, no file I/O, one thread; its pixels are compared with the written PNGs
Nothing is written to the tree.  The colormap is a seeded 256-entry table: the timing does not depend on its values.

  python tools/bench_depth_vis.py [--frames 300] [--width 384] [--height 224] [--reps 20]"""
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

from tools.bench_flow_masks import _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--width", type=int, default=384)
    ap.add_argument("--height", type=int, default=224)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    from robust_cvd_b200 import solver, visualization as vis
    from robust_cvd_b200.synthetic_files import write_raw
    from robust_cvd_b200.video import _decode_png
    from tests import depth_vis_ref as ref

    rng = np.random.default_rng(0)
    lut = rng.integers(0, 256, (256, 3), dtype=np.uint8)
    frames = []
    for i in range(args.frames):
        d = (rng.uniform(0.2, 1.0, (args.height, args.width)) * (1 + 0.002 * i)).astype(np.float32)
        d[rng.integers(0, args.height, 40), rng.integers(0, args.width, 40)] = np.nan
        frames.append(d)
    stack = np.stack(frames)
    out = {"card": _card(), "frames": args.frames, "width": args.width, "height": args.height}

    t64, rgb_lut = vis.color_tables(lut)
    ms_range, ms_color = solver.time_depth_visualize(stack, (0.0, 1.0), 0.2, 1.0, rgb_lut, reps=args.reps)
    out["kernel"] = {"range_ms_per_frame": ms_range / args.frames, "color_ms_per_frame": ms_color / args.frames,
                     "range_ms_per_pass": ms_range, "color_ms_per_pass": ms_color}

    tmp = tempfile.mkdtemp()
    try:
        src = os.path.join(tmp, "depth")
        os.makedirs(src)
        for i, d in enumerate(frames):
            write_raw(os.path.join(src, f"frame_{i:06d}.raw"), d)
        runs = []
        for _ in range(2):
            devnull = open(os.devnull, "w")
            real, sys.stdout = sys.stdout, devnull
            try:
                st = vis.visualize_depth_dir(src, src, force=True, colormap=lut)
            finally:
                sys.stdout = real
                devnull.close()
            runs.append({k: st[k] for k in ("total_s", "read_s", "compute_s", "write_s")})
        out["call"] = runs

        t = time.perf_counter()
        _, _, want = ref.visualize_dir(frames, 0, 100, lut)
        out["numpy"] = {"total_s": time.perf_counter() - t}
        out["numpy"]["ms_per_frame"] = 1e3 * out["numpy"]["total_s"] / args.frames
        diff = sum(int(not np.array_equal(_decode_png(os.path.join(src, f"frame_{i:06d}.png"))[..., ::-1], want[i]))
                   for i in range(args.frames))
        out["frames_differing_from_numpy"] = diff
    finally:
        shutil.rmtree(tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
