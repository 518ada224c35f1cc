"""Float32 restatement of the reference's joint depth / colour bilateral filter (TEST INFRASTRUCTURE; checks
robust_cvd_b200/csrc/rcvd_bilateral.cuh through tests/test_bilateral.py, tests/test_gpu_bilateral.py and tools/bench_bilateral.py).

`python tests/bilateral_ref.py` rewrites tests/golden/bilateral_golden.npz, which pins the restatement against silent edits."""
import os
import sys

import numpy as np

f32 = np.float32
# ---------------------------------------------------------------------------------------------------------
# Joint depth / colour bilateral filter: float32 restatement of DepthVideoProcessor::bilateralFilter (reference
# lib/Processor.cpp:183-313).  Vectorised over pixels; the window offsets are visited in the reference's order (frame -> row ->
# column) and every sum is an explicit elementwise accumulation, so each pixel's float32 sums are the reference's.  Arrays use the
# local frame indexing of rcvd_bilateral_filter (include/rcvd.h).
# ---------------------------------------------------------------------------------------------------------
def _bilateral_samples(depth, color, frame, rows, frame_radius, spatial_radius, depth_sigma, color_sigma):
    """Yields (valid [n,w], depth [n,w], weight [n,w]) for every window offset of the output rows `rows`, in window order."""
    F, h, w = depth.shape
    r = spatial_radius
    ys = np.arange(rows.start, rows.stop)[:, None]; xs = np.arange(w)[None, :]
    dref = depth[frame, rows]
    cref = None if color is None else color[frame, rows]
    ds2 = f32(f32(depth_sigma) * f32(depth_sigma)); cs2 = f32(f32(color_sigma) * f32(color_sigma))
    for wf in range(max(0, frame - frame_radius), min(F - 1, frame + frame_radius) + 1):
        for dy in range(-r, r + 1):
            wy = ys + dy
            for dx in range(-r, r + 1):
                wx = xs + dx
                valid = (wy >= 0) & (wy < h) & (wx >= 0) & (wx < w)
                cy = np.clip(wy, 0, h - 1); cx = np.clip(wx, 0, w - 1)
                d = depth[wf][cy, cx]
                e = np.zeros(d.shape, f32)
                with np.errstate(all="ignore"):
                    if depth_sigma > 0:
                        t = (d - dref).astype(f32)
                        e = (e + (-(t * t)) / ds2).astype(f32)
                    if color_sigma > 0:
                        c = color[wf][cy, cx]
                        t = (c - cref).astype(f32)
                        d2 = ((t[..., 0] * t[..., 0] + t[..., 1] * t[..., 1]) + t[..., 2] * t[..., 2]).astype(f32)
                        e = (e + (-d2) / cs2).astype(f32)
                    wt = np.where(e != 0, np.exp(e), f32(1)).astype(f32)
                yield valid, d, wt


def bilateral_filter(depth, out_frames, color=None, frame_radius=2, spatial_radius=0, depth_sigma=0.3, color_sigma=0.0, median=False,
                     retransform=None, max_keys=1 << 23):
    """depth [F,h,w] f32 (transformed depth of stream 0), color [F,h,w,3] f32 BGR (read when color_sigma > 0), out_frames ascending
    local indices -> [num_out,h,w] f32.  retransform(frame, filtered) -> image: in-place filtering (the output goes back into stream
    0); after each output frame its stack slot becomes retransform(frame, filtered), which later windows then read."""
    depth = np.array(depth, f32, copy=True)
    color = None if color is None or not color_sigma > 0 else np.asarray(color, f32)
    F, h, w = depth.shape
    n_off = (2 * spatial_radius + 1) ** 2 * (2 * frame_radius + 1)
    out = np.zeros((len(out_frames), h, w), f32)
    for o, frame in enumerate(out_frames):
        step = h if not median else max(1, min(h, max_keys // max(1, n_off * w)))
        for y0 in range(0, h, step):
            rows = slice(y0, min(h, y0 + step))
            sum_d = np.zeros((rows.stop - y0, w), f32); sum_w = np.zeros_like(sum_d)
            keys = []
            for valid, d, wt in _bilateral_samples(depth, color, frame, rows, frame_radius, spatial_radius, depth_sigma, color_sigma):
                with np.errstate(all="ignore"):
                    if median:
                        keys.append((valid, d, wt))
                    else:
                        sum_d = np.where(valid, sum_d + d * wt, sum_d).astype(f32)
                    sum_w = np.where(valid, sum_w + wt, sum_w).astype(f32)
            with np.errstate(all="ignore"):
                if median:
                    valid = np.stack([k[0] for k in keys]); d = np.stack([k[1] for k in keys]); wt = np.stack([k[2] for k in keys])
                    d = np.where(d == 0, f32(0), d)                       # std::pair compares -0 equal to +0
                    order = np.lexsort((wt, d, ~valid), axis=0)           # valid samples first, then (depth, weight) ascending
                    ds = np.take_along_axis(d, order, 0); ws = np.take_along_axis(wt, order, 0); vs = np.take_along_axis(valid, order, 0)
                    cum = np.add.accumulate(np.where(vs, ws, f32(0)), axis=0, dtype=f32)
                    hit = (cum >= (sum_w / f32(2)).astype(f32)) & vs
                    first = np.argmax(hit, axis=0)
                    res = np.where(hit.any(axis=0), np.take_along_axis(ds, first[None], 0)[0], f32(0))
                else:
                    res = np.where(sum_w > 0, sum_d / sum_w, f32(0))
            out[o, rows] = res.astype(f32)
        if retransform is not None and frame_radius > 0:
            depth[frame] = np.asarray(retransform(frame, out[o]), f32)
    return out


def golden_configs():
    """Settings of tests/golden/bilateral_golden.npz (in_place: retransform with the stored per-frame scales)."""
    return [("mean_r0", dict(frame_radius=2, spatial_radius=0, depth_sigma=0.3)),
            ("mean_r2_color", dict(frame_radius=1, spatial_radius=2, depth_sigma=0.3, color_sigma=0.1)),
            ("median_r1_color", dict(frame_radius=2, spatial_radius=1, depth_sigma=0.3, color_sigma=0.1, median=True)),
            ("median_r2_unit", dict(frame_radius=1, spatial_radius=2, depth_sigma=0.0, median=True)),
            ("mean_in_place", dict(frame_radius=2, spatial_radius=1, depth_sigma=0.3, in_place=True))]


def write_golden(path):
    rng = np.random.default_rng(31)
    F, h, w = 6, 9, 11
    depth = rng.uniform(0.5, 3.0, (F, h, w)).astype(f32)
    depth[2, 4, 3:6] = depth[3, 4, 4]
    color = rng.uniform(0, 1, (F, h, w, 3)).astype(f32)
    scale = rng.uniform(0.7, 1.4, F)
    out_frames = np.array([0, 2, 3, 5], np.int32)
    out = {"depth": depth, "color": color, "scale": scale, "out_frames": out_frames}
    for name, kw in golden_configs():
        if kw.pop("in_place", False):
            kw["retransform"] = lambda f, img: (img.astype(np.float64) * scale[f]).astype(f32)
        out[name] = bilateral_filter(depth, list(out_frames), color, **kw)
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    write_golden(sys.argv[1] if len(sys.argv) > 1 else os.path.join(here, "golden", "bilateral_golden.npz"))
