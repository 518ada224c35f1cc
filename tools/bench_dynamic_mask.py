#!/usr/bin/env python3
"""Times the dynamic-mask stage (robust_cvd_b200.dynamic_mask, rcvd_dynamic_masks) at 1920 x 1080.

Reports, as one JSON object with the card's name and power limit and the host's CPU count:
  kernel     device time per frame of rcvd_dynamic_masks' kernels alone with K dynamic instances per frame (`--instances`), d = 5,
             without and with the anonymised frame (rcvd_debug_time_dynamic_masks: CUDA events over `--reps` passes over a batch of
             `--batch` frames resident on the device), and at d = 101
  call       the whole compute_dynamic_mask on a seeded `--frames`-frame color_full (written to a temporary directory), with a stub
             predictor: a few torch ops on the GPU that return K bool masks of the frame's size on the device; split into decoding
             (summed over threads), the predictor, the GPU calls (mask copy-in, kernels, copy-back) and PNG writing (summed over
             threads); with and without --save_anno
  reference  the reference's per-frame post-processing restated on the same host (tests/dynamic_mask_ref.reference_frame: boolean
             index writes, cv2.dilate, cv2.bitwise_not, plus cv2.imwrite of the mask) on the same masks, one thread; the detectron2
             Visualizer drawing is added only when detectron2 is importable
Nothing is written to the tree.

  python tools/bench_dynamic_mask.py [--frames 300] [--instances 4] [--batch 30] [--reps 20]"""
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

H, W = 1080, 1920


def _masks(rng, K):
    m = np.zeros((K, H, W), bool)
    for k in range(K):
        y0, x0 = rng.integers(0, H - 300), rng.integers(0, W - 300)
        m[k, y0:y0 + rng.integers(50, 300), x0:x0 + rng.integers(50, 300)] = True
    return m


class StubInstances:
    def __init__(self, classes, masks):
        self.f = {"pred_classes": classes, "pred_masks": masks}

    def __len__(self):
        return len(self.f["pred_classes"])

    def get(self, k):
        return self.f[k]


class StubPredictor:
    """K dynamic instances per frame from a few torch ops on the GPU: boxes placed by the frame's mean colour."""
    def __init__(self, K):
        import torch
        self.torch, self.K = torch, K
        self.yy = torch.arange(H, device="cuda").view(1, H, 1)
        self.xx = torch.arange(W, device="cuda").view(1, 1, W)
        self.classes = torch.zeros(K, dtype=torch.int64, device="cuda")

    def __call__(self, img):
        t = self.torch.from_numpy(img).cuda()
        s = t.float().mean(dim=(0, 1))
        c = (s.sum() * 7).long() % 500 + self.torch.arange(self.K, device="cuda").view(self.K, 1, 1) * 100
        masks = (self.yy >= c) & (self.yy < c + 200) & (self.xx >= 2 * c) & (self.xx < 2 * c + 300)
        self.torch.cuda.synchronize()
        return {"instances": StubInstances(self.classes, masks)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--instances", type=int, default=4)
    ap.add_argument("--batch", type=int, default=30)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import cv2
    from robust_cvd_b200 import dynamic_mask as dm, solver
    from robust_cvd_b200.png import write_png
    from tests import dynamic_mask_ref as ref

    K = args.instances
    rng = np.random.default_rng(0)
    out = {"card": _card(), "cpus": os.cpu_count(), "width": W, "height": H, "instances_per_frame": K, "frames": args.frames}

    ins = np.concatenate([_masks(rng, K) for _ in range(args.batch)])
    offsets = np.arange(0, K * args.batch + 1, K, dtype=np.int64)
    frames = rng.integers(0, 256, (args.batch, H, W, 3), dtype=np.uint8)
    kern = {}
    for name, d, fr in (("d5", 5, None), ("d5_anon", 5, frames), ("d101", 101, None)):
        ms = solver.time_dynamic_masks(ins, offsets, (H, W), d, fr, reps=args.reps)
        kern[f"{name}_ms_per_frame"] = ms / args.batch
    out["kernel"] = kern

    tmp = tempfile.mkdtemp()
    try:
        full = os.path.join(tmp, "video", "color_full")
        os.makedirs(full)
        base = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        for i in range(args.frames):
            write_png(os.path.join(full, f"frame_{i:06d}.png"), np.roll(base, 7 * i, axis=1))
        with open(os.path.join(tmp, "video", "frames.txt"), "w") as f:
            f.write(f"{args.frames}\n{W}\n{H}\n" + "".join(f"{i / 30:.6f}\n" for i in range(args.frames)))
        pred = StubPredictor(K)
        pred(base)   # warm-up
        runs = {}
        for anno in (False, True):
            shutil.rmtree(os.path.join(tmp, "video", "dynamic_mask"), ignore_errors=True)
            devnull = open(os.devnull, "w")
            real, sys.stdout = sys.stdout, devnull
            try:
                st = dm.compute_dynamic_mask(os.path.join(tmp, "video"), save_anno=anno, predictor=pred)
            finally:
                sys.stdout = real
                devnull.close()
            runs["save_anno" if anno else "masks"] = {k: st[k] for k in ("total_s", "decode_s", "predict_s", "kernel_s", "write_s", "wait_s")}
        out["call"] = runs

        # the reference's per-frame post-processing on the host, on the same masks
        n = min(args.frames, 30)
        img = base
        m = pred(img)["instances"].get("pred_masks").cpu().numpy()
        classes = np.zeros(K, np.int64)
        t = time.perf_counter()
        for i in range(n):
            mask, _ = ref.reference_frame(img, classes, m, 5, False)
            cv2.imwrite(os.path.join(tmp, "ref.png"), mask)
        out["reference"] = {"ms_per_frame": 1e3 * (time.perf_counter() - t) / n, "frames": n}
        try:
            from detectron2.utils.visualizer import Visualizer
        except ImportError:
            out["reference"]["visualizer"] = "not measured: detectron2 is not installed"
        else:
            t = time.perf_counter()
            for i in range(n):
                Visualizer(img[:, :, ::-1]).overlay_instances(masks=m)
            out["reference"]["visualizer_ms_per_frame"] = 1e3 * (time.perf_counter() - t) / n
    finally:
        shutil.rmtree(tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
