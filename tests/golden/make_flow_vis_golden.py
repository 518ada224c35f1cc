"""Generates tests/golden/flow_vis_golden.npz, the flow-visualisation fixture, by running the reference's own Flow.visualize_flow(warp=True)
(flow.py, with utils/flowlib.py, utils/visualization.py and utils/geometry.py imported unchanged, nothing copied) on small seeded working
directories.  flow.py's imports that are not needed here and not installable offline (iopath.common.file_io, optical_flow_homography) go
into sys.modules as stubs.  Without a GPU the reference's torch device is the CPU, so the warps are torch's CPU grid_sample.  Needs a
checkout of facebookresearch/robust_cvd named by ROBUST_CVD_DIR, as the other golden generators in this directory do.

  ROBUST_CVD_DIR=/path/to/robust_cvd python tests/golden/make_flow_vis_golden.py

Stored per case: the inputs (colours, masks and both flows of each pair), the decoded PNGs (cv2.imread, so array channel order), and the
intermediates: flowlib.flow_to_image of each flow, the normalised (u, v) that flowlib.compute_color receives, the float32 warp values of
flow.warp_by_flow, and the dtypes numpy gives the normalisation and the composite (NEP 50 promotion of the installed numpy)."""
import os
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("ROBUST_CVD_DIR", "")

# (H, W, frames, pairs, seed): odd sizes, H != W, non-square; frames shared by several pairs
FLOW_VIS_CASES = {"9x13": (9, 13, 3, [(0, 1), (1, 2), (0, 2)], 41), "11x7": (11, 7, 3, [(2, 0), (1, 2)], 42)}


def flow_vis_case(name):
    """Inputs of one case: colours {frame: [H, W, 3] f32}, flows {(a, b): [H, W, 2] f32} in both directions of every pair, masks
    {(a, b): [H, W] u8}.  The flows of the first pair carry NaN, +-inf, |u| > 1e7 and |u| = 1e7 (not unknown); the second pair's
    forward flow is all zero; the rest are smooth with targets exactly on the borders, off the image and on pixel centres."""
    H, W, F, pairs, seed = FLOW_VIS_CASES[name]
    rng = np.random.default_rng(seed)
    iy, ix = np.mgrid[0:H, 0:W]
    colors = {}
    for f in range(F):
        c = rng.random((H, W, 3)).astype(np.float32)
        c[0, 0] = (-0.01, 1.2, 0.5)                        # saturation at both ends
        c[1, 1] = (0.5 / 255, 1.5 / 255, 254.5 / 255)      # near the half-way points of the rounding
        colors[f] = c
    flows, masks = {}, {}
    for n, (i, j) in enumerate(pairs):
        for d, (a, b) in enumerate(((i, j), (j, i))):
            f = np.stack((rng.normal(0, 2, (H, W)) + 1.5 * np.sin(0.4 * iy), rng.normal(0, 2, (H, W)) - np.cos(0.3 * ix)), axis=-1)
            k = rng.integers(0, 10, (H, W))
            f[..., 0] = np.where(k == 0, -ix, f[..., 0]); f[..., 0] = np.where(k == 1, W - 1 - ix, f[..., 0])     # on the x borders
            f[..., 1] = np.where(k == 2, -iy, f[..., 1]); f[..., 1] = np.where(k == 3, H - 1 - iy, f[..., 1])     # on the y borders
            f = np.where((k == 4)[..., None], np.round(f), f)                                                     # pixel centres
            f[..., 0] = np.where(k == 5, f[..., 0] + 3 * W, f[..., 0])                                            # off the image
            f = f.astype(np.float32)
            if n == 0 and d == 0:
                f[0, 1, 0] = np.nan; f[2, 3] = np.nan; f[3, 4, 0] = np.inf; f[4, 5, 1] = -np.inf
                f[5, 6, 0] = 2e7; f[6, 2, 1] = -1e7
            if n == 0 and d == 1:
                f[1, 2, 0] = 1e7; f[7, 3, 1] = -3e7
            if n == 1 and d == 0:
                f[:] = 0
            flows[(a, b)] = f
            m = np.where(rng.random((H, W)) < 0.6, 255, 0).astype(np.uint8)
            m[0, :3] = (1, 128, 0)                                  # mask > 0, not only 255
            masks[(a, b)] = m
    return colors, flows, masks


def _import_reference():
    """The reference's flow module and flowlib, with the two unavailable imports stubbed."""
    if REF not in sys.path:
        sys.path.insert(0, REF)
    for name in ("iopath", "iopath.common", "iopath.common.file_io"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["iopath.common.file_io"].g_pathmgr = None
    sys.modules.setdefault("optical_flow_homography", types.ModuleType("optical_flow_homography"))
    import flow as ref_flow
    from utils import flowlib
    return ref_flow, flowlib


def golden_flow_vis():
    import cv2
    sys.path.insert(0, ROOT)
    from robust_cvd_b200.synthetic_files import write_raw
    ref_flow, flowlib = _import_reference()
    seen = []
    orig = flowlib.compute_color

    def recording_compute_color(u, v):
        seen.append((u.copy(), v.copy()))
        return orig(u, v)
    flowlib.compute_color = recording_compute_color
    written, imwrite = {}, cv2.imwrite

    def recording_imwrite(fn, img, *a):
        written.setdefault(os.path.basename(os.path.dirname(fn)), set()).add(str(img.dtype))
        return imwrite(fn, img, *a)
    cv2.imwrite = recording_imwrite
    out = {}
    try:
        for name in FLOW_VIS_CASES:
            colors, flows, masks = flow_vis_case(name)
            H, W, F, pairs, _ = FLOW_VIS_CASES[name]
            tmp = tempfile.mkdtemp(prefix="flowvis_")
            try:
                for d in ("flow", "flow_mask", "color_down"):
                    os.makedirs(os.path.join(tmp, d))
                for f, c in colors.items():
                    write_raw(os.path.join(tmp, "color_down", f"frame_{f:06d}.raw"), c)
                    out[f"{name}/color/{f}"] = c
                for (a, b), fl in flows.items():
                    write_raw(os.path.join(tmp, "flow", f"flow_{a:06d}_{b:06d}.raw"), fl)
                    cv2.imwrite(os.path.join(tmp, "flow_mask", f"mask_{a:06d}_{b:06d}.png"), masks[(a, b)])
                    out[f"{name}/flow/{a}_{b}"] = fl
                    out[f"{name}/mask/{a}_{b}"] = masks[(a, b)]
                    seen.clear()
                    out[f"{name}/flow_image/{a}_{b}"] = flowlib.flow_to_image(np.copy(fl))
                    out[f"{name}/u/{a}_{b}"], out[f"{name}/v/{a}_{b}"] = seen[0]
                    out[f"{name}/warp_values/{a}_{b}"] = ref_flow.warp_by_flow(colors[b] * 255, fl)   # colour b sampled at p + flow_ab
                ref_flow.Flow(tmp, tmp).visualize_flow(warp=True)
                for d in ("vis_flow", "vis_flow_warped"):
                    for fn in sorted(os.listdir(os.path.join(tmp, d))):
                        out[f"{name}/{d}/{fn}"] = cv2.imread(os.path.join(tmp, d, fn), cv2.IMREAD_UNCHANGED)
            finally:
                shutil.rmtree(tmp)
        key = f"{pairs[0][0]}_{pairs[0][1]}"
        out["dtype/normalised_uv"] = np.array(str(out[f"{name}/u/{key}"].dtype))
        out["dtype/flow_image"] = np.array(str(out[f"{name}/flow_image/{key}"].dtype))
        out["dtype/warp_values"] = np.array(str(out[f"{name}/warp_values/{key}"].dtype))
        for d, dts in written.items():
            out[f"dtype/{d}"] = np.array(",".join(sorted(dts)))        # what cv2.imwrite was given
        out["numpy_version"] = np.array(np.__version__)
    finally:
        flowlib.compute_color = orig
        cv2.imwrite = imwrite
    np.savez_compressed(os.path.join(HERE, "flow_vis_golden.npz"), **out)


if __name__ == "__main__":
    if not os.path.isfile(os.path.join(REF, "flow.py")):
        sys.exit("set ROBUST_CVD_DIR to a checkout of facebookresearch/robust_cvd")
    golden_flow_vis()
    print("flow-visualisation golden fixture written")
