#!/usr/bin/env python3
"""Times the frame downscaling (robust_cvd_b200.video.downscale_all, rcvd_resize_area) on a seeded color_full directory of `--frames`
8-bit RGB PNGs of `--width` x `--height` (default 300 frames of 1920 x 1080, smooth gradients plus noise, written to a temporary
directory).

Reports, as one JSON object with the card's name and power limit and the host's CPU count:
  kernel     device time of rcvd_resize_area's kernels per frame (rcvd_debug_time_resize_area: CUDA events over `--reps` passes of
             `--kernel-frames` resident frames, all three outputs of process.py)
  call       the whole downscale_all(path) on the host clock (color_down .raw, color_down_png and color_flow), split into decode (reader
             time), GPU calls (upload, kernels, copy-back), file writes (summed over the writer threads) and the calling thread's wait;
             a first run and a second one
  reference  the reference's three Video.downscale_frames calls (process.py's DatasetProcessor.downscale_frames) on the same directory
             and host, one frame at a time on one thread: with --reference DIR the reference's own video.py from that checkout; without,
             the same per-frame steps restated with the same libraries (Pillow decode, np.float32(img) / 255.0, cv2.resize(INTER_AREA),
             the B, G, R swap, the .raw writer's format, cv2.imwrite(fn, img * 255)).  Its outputs are compared with downscale_all's:
             .raw files byte for byte, PNGs by decoded pixels.
Nothing is written to the tree.

  python tools/bench_downscale.py [--frames 300] [--width 1920] [--height 1080] [--reference DIR] [--reference-frames N]"""
import argparse
import json
import os
import shutil
import struct
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_flow_masks import _card  # noqa: E402

# process.py's three calls: (subdir, max_size, ext, align); size 384, align 32, and Flow.max_size() = 1024 at align 64
CALLS = [("color_down", 384, "raw", 32), ("color_down_png", 384, "png", 32), ("color_flow", 1024, "png", 64)]


def write_frames(root, n, W, H, seed=0):
    from robust_cvd_b200.png import png_rgb_bytes
    full = os.path.join(root, "color_full")
    os.makedirs(full)
    iy, ix = np.mgrid[0:H, 0:W].astype(np.float32)

    def one(i):
        rng = np.random.default_rng(seed * 100003 + i)
        base = np.stack([ix * (255.0 / W), iy * (255.0 / H), (ix + iy + 7 * i) % 256], axis=-1)
        img = np.clip(base + rng.normal(0, 12, (H, W, 3)).astype(np.float32), 0, 255).astype(np.uint8)
        with open(os.path.join(full, f"frame_{i:06d}.png"), "wb") as f:
            f.write(png_rgb_bytes(img, level=6))
        return os.path.getsize(os.path.join(full, f"frame_{i:06d}.png"))
    with ThreadPoolExecutor(min(16, os.cpu_count() or 1)) as ex:
        sizes = list(ex.map(one, range(n)))
    with open(os.path.join(root, "frames.txt"), "w") as f:
        f.write(f"{n}\n{W}\n{H}\n" + "".join(f"{i / 30.0:.6f}\n" for i in range(n)))
    return sizes


def reference_restated(root, n):
    """The reference's three downscale_frames loops (video.py:154-182 with image_io.load_image / resize_to_target /
    save_raw_float32_image), one frame at a time, into <root>/ref_<subdir>."""
    import cv2
    from PIL import Image
    from robust_cvd_b200.video import target_size
    for subdir, max_size, ext, align in CALLS:
        out = os.path.join(root, "ref_" + subdir)
        os.makedirs(out, exist_ok=True)
        for i in range(n):
            with Image.open(os.path.join(root, "color_full", f"frame_{i:06d}.png")) as im:
                img = np.float32(im) / 255.0
            h, w = target_size(img.shape[0], img.shape[1], max_size, align)
            img = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)[..., ::-1]
            fn = os.path.join(out, f"frame_{i:06d}.{ext}")
            if ext == "raw":
                with open(fn, "wb") as f:
                    f.write(struct.pack("<iiiQ", h, w, 21, 12) + np.ascontiguousarray(img, np.float32).tobytes())
            else:
                cv2.imwrite(fn, img * 255)


def reference_own(root, ref_dir, n):
    """The reference's own Video.downscale_frames from a checkout, writing <root>/ref_<subdir> (its frames.txt counts n frames)."""
    sys.path.insert(0, ref_dir)
    import video as ref_video
    v = ref_video.Video(root)
    v.frame_count = n
    for subdir, max_size, ext, align in CALLS:
        v.downscale_frames("ref_" + subdir, max_size, ext, align=align)


def compare(root, n):
    import cv2
    differ = 0
    for subdir, _, ext, _ in CALLS:
        for i in range(n):
            a, b = (os.path.join(root, d, f"frame_{i:06d}.{ext}") for d in (subdir, "ref_" + subdir))
            if ext == "raw":
                differ += open(a, "rb").read() != open(b, "rb").read()
            else:
                differ += not np.array_equal(cv2.imread(a, cv2.IMREAD_UNCHANGED), cv2.imread(b, cv2.IMREAD_UNCHANGED))
    return differ


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--kernel-frames", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--reference", default="", help="a checkout of the reference, to time its own video.py")
    ap.add_argument("--reference-frames", type=int, default=0, help="frames the reference path runs on (default: all)")
    args = ap.parse_args()
    from robust_cvd_b200 import solver, video
    W, H = args.width, args.height
    out = {"what": "frame downscaling: robust_cvd_b200.video.downscale_all", "frames": args.frames, "source": [W, H], "card": _card()}
    root = tempfile.mkdtemp(prefix="rcvd_downscale_")
    try:
        t = time.perf_counter()
        sizes = write_frames(root, args.frames, W, H)
        out["input"] = {"mean_png_bytes": int(np.mean(sizes)), "write_s": time.perf_counter() - t}
        targets = [(*video.target_size(H, W, ms, al), ext) for _, ms, ext, al in CALLS]
        out["outputs"] = [[w, h, ext] for h, w, ext in targets]
        # ---- kernels alone, frames resident on the device ----
        k = min(args.kernel_frames, args.frames)
        frames = np.stack([video._decode_png(os.path.join(root, "color_full", f"frame_{i:06d}.png")) for i in range(k)])
        ms = solver.time_resize_area(frames, targets, reps=args.reps)
        out["kernel"] = {"frames": k, "reps": args.reps, "device_ms_per_pass": ms, "device_us_per_frame": 1e3 * ms / k}
        del frames
        # ---- the whole call ----
        runs = []
        for _ in range(2):
            for sub, *_ in CALLS:
                shutil.rmtree(os.path.join(root, sub), ignore_errors=True)
            s = video.downscale_all(root)
            runs.append({key: (round(v, 4) if isinstance(v, float) else v) for key, v in s.items()})
        out["call"] = {"first": runs[0], "second": runs[1], "ms_per_frame_second": 1e3 * runs[1]["total_s"] / max(args.frames, 1)}
        # ---- the reference's path, same directory and host ----
        n = args.reference_frames or args.frames
        t = time.perf_counter()
        if args.reference:
            reference_own(root, args.reference, n)
            code = f"the reference's video.Video.downscale_frames ({args.reference})"
        else:
            reference_restated(root, n)
            code = "the reference's per-frame steps restated (Pillow, numpy, cv2.resize INTER_AREA, cv2.imwrite)"
        ref_s = time.perf_counter() - t
        out["reference"] = {"code": code, "frames": n, "s": ref_s, "ms_per_frame": 1e3 * ref_s / n,
                            "whole_directory_s_estimate": ref_s * args.frames / n, "files_differing_from_downscale_all": compare(root, n)}
        out["speedup_vs_reference_second_run"] = out["reference"]["whole_directory_s_estimate"] / runs[1]["total_s"]
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
