"""Generates tests/golden/flow_masks_golden.npz, the flow-consistency mask fixture, from the reference's own utils/consistency.py
(imported unchanged, nothing copied).  Needs a checkout of facebookresearch/robust_cvd named by ROBUST_CVD_DIR, as the other golden
generators in this directory do.

  ROBUST_CVD_DIR=/path/to/robust_cvd python tests/golden/make_flow_masks_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("ROBUST_CVD_DIR", "")


def flow_mask_case(name):
    """Inputs of one flow-mask golden case: flow_ij, flow_ji [H, W, 2] and colour_i, colour_j [H, W, 3] float32, seeded.  The flows
    mix fractional steps with targets exactly on the image borders and on pixel centres, targets off the image, NaN and inf."""
    H, W, seed = {"12x16": (12, 16, 31), "9x13": (9, 13, 32), "20x20": (20, 20, 33)}[name]
    rng = np.random.default_rng(seed)
    iy, ix = np.mgrid[0:H, 0:W]
    smooth = np.stack((1.3 + 0.8 * np.sin(0.3 * iy), -0.7 + 0.6 * np.cos(0.25 * ix)), axis=-1)
    fij = (smooth + rng.normal(0, 0.05, (H, W, 2))).astype(np.float32)
    k = rng.integers(0, 9, (H, W))
    fij[..., 0] = np.where(k == 0, -ix, fij[..., 0]); fij[..., 0] = np.where(k == 1, W - 1 - ix, fij[..., 0])     # on the x borders
    fij[..., 1] = np.where(k == 2, -iy, fij[..., 1]); fij[..., 1] = np.where(k == 3, H - 1 - iy, fij[..., 1])     # on the y borders
    fij = np.where((k == 4)[..., None], np.round(fij), fij)                                                      # pixel centres
    fij[..., 0] = np.where(k == 5, W - ix + rng.uniform(-0.6, 0.6, (H, W)), fij[..., 0])                        # just off / just in
    fij[..., 1] = np.where(k == 6, -iy - rng.uniform(0, 1e-3, (H, W)), fij[..., 1])                             # just above the image
    fij = fij.astype(np.float32)
    fij[0, 1, 0] = np.nan; fij[1, 2, 1] = np.nan; fij[2, 3] = np.nan; fij[3, 4, 0] = np.inf; fij[4, 5, 1] = -np.inf
    fji = (-smooth + rng.normal(0, 0.3, (H, W, 2))).astype(np.float32)     # roughly consistent backward flow
    fji[5, 6, 0] = np.nan
    base = (0.5 + 0.4 * np.sin(ix * 0.7)[..., None] * np.cos(iy[..., None] * 0.5 + np.arange(3))).astype(np.float32)
    ci = (base + rng.normal(0, 0.15, (H, W, 3))).astype(np.float32)
    cj = (base + rng.normal(0, 0.15, (H, W, 3))).astype(np.float32)
    return fij, fji, ci, cj


FLOW_MASK_CASES = ("12x16", "9x13", "20x20")
FLOW_MASK_THRESHOLDS = ((1, 1), (0.7, 0.7))


def golden_flow_masks():
    """Flow-consistency masks from the reference's own utils/consistency.py (imported unchanged): consistent_flow_masks' masks,
    and for each direction the arrays its consistency_mask compares -- sample() of -flow_tgt and of colour_tgt at pixel + flow_ref,
    and sse() of each check -- for FLOW_MASK_CASES at the thresholds FLOW_MASK_THRESHOLDS."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_consistency", os.path.join(REF, "utils", "consistency.py"))
    cons = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cons)
    out = {}
    for name in FLOW_MASK_CASES:
        fij, fji, ci, cj = flow_mask_case(name)
        H, W = fij.shape[:2]
        out.update({f"{name}/flow_ij": fij, f"{name}/flow_ji": fji, f"{name}/color_i": ci, f"{name}/color_j": cj})
        X, Y = np.meshgrid(np.arange(W), np.arange(H))
        for d, (fr, ft, cr, ct) in enumerate(((fij, fji, ci, cj), (fji, fij, cj, ci))):
            uv = np.stack((fr[..., 0] + X, fr[..., 1] + Y), axis=-1)      # consistency_mask's idx_x, idx_y
            fs, cs = cons.sample(-ft, uv), cons.sample(ct, uv)
            out.update({f"{name}/{d}/flow_sample": fs, f"{name}/{d}/color_sample": cs,
                        f"{name}/{d}/sse_flow": cons.sse(fr, fs), f"{name}/{d}/sse_color": cons.sse(cr, cs)})
        for ft_, ct_ in FLOW_MASK_THRESHOLDS:
            masks = cons.consistent_flow_masks([fij, fji], [ci, cj], ft_, ct_)
            for d in range(2):
                out[f"{name}/{d}/mask_{ft_}_{ct_}"] = np.asarray(masks[d], bool)
    np.savez_compressed(os.path.join(HERE, "flow_masks_golden.npz"), **out)


if __name__ == "__main__":
    if not os.path.isfile(os.path.join(REF, "utils", "consistency.py")):
        sys.exit("set ROBUST_CVD_DIR to a checkout of facebookresearch/robust_cvd")
    golden_flow_masks()
    print("flow-mask golden fixture written")
