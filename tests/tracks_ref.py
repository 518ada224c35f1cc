"""Float32 restatement of the reference's long point tracker (TEST INFRASTRUCTURE; checks robust_cvd_b200/csrc/rcvd_tracks.cuh through
tests/test_tracks.py, tests/test_gpu_tracks.py and tools/bench_tracks.py).

`python tests/tracks_ref.py` rewrites tests/golden/tracks_golden.npz, which pins the restatement against silent edits."""
import os
import struct
import sys

import numpy as np

f32 = np.float32
FLT_MAX = f32(3.402823466e+38)
IN_RANGE, HAS_COLOR, FLOW, MASK = 1, 2, 4, 8   # frame flags of rcvd_compute_tracks (include/rcvd.h)


# ---------------------------------------------------------------------------------------------------------
# DepthVideoProcessor::computeTracks (reference lib/Processor.cpp:646-886), statement by statement, one track and one candidate
# at a time.  Arrays use the local frame indexing of rcvd_compute_tracks: local frame 0 is the first frame of the range, the last
# local frame its last one; slot f of flow / flow_mask holds the pair (f-1 -> f).  Where the reference reads outside an image (a
# dynamic-distance lookup at -1, a track row rounded to h) the nearest pixel is read.
# ---------------------------------------------------------------------------------------------------------
def _disk(r):
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    return (x * x + y * y) <= r * r


def _splat(mask, disk, x, y):
    r = disk.shape[0] // 2
    h, w = mask.shape
    x0, x1, y0, y1 = max(0, x - r), min(w - 1, x + r), max(0, y - r), min(h - 1, y + r)
    mask[y0:y1 + 1, x0:x1 + 1] |= disk[y0 - (y - r):y1 - (y - r) + 1, x0 - (x - r):x1 - (x - r) + 1]


def compute_tracks(color, flags, flow=None, flow_mask=None, dyn_masks=None, spawn_distance=20, prune_distance=5, min_dynamic_distance=3,
                   inv_aspect=1.0):
    """Returns (tracks, frames): tracks[id] = list of (local frame, x, y) float32 observations, frames[f] = ascending track ids."""
    import cv2
    F, h, w = color.shape[:3]
    ia = f32(inv_aspect)
    mdd = f32(min_dynamic_distance)
    spawn_disk, prune_disk = _disk(spawn_distance), _disk(prune_distance)
    tracks, frames = [], [[] for _ in range(F)]
    for f in range(F):
        fl = int(flags[f])
        if not (fl & IN_RANGE) or not (fl & HAS_COLOR):
            continue
        if dyn_masks is not None:
            m = np.asarray(dyn_masks[f], np.uint8)
            dist = cv2.distanceTransform(np.where(m < 127, 0, 255).astype(np.uint8), cv2.DIST_L2, 5)
            dh, dw = m.shape
            sx, sy = f32(f32(dw) / f32(w)), f32(f32(dh) / f32(h))
        else:
            dist, dh, dw, sx, sy = None, h, w, f32(1), f32(1)

        def dyn(ys, xs):
            if dist is None:
                return FLT_MAX
            return dist[min(max(ys, 0), dh - 1), min(max(xs, 0), dw - 1)]

        spawn_mask = np.zeros((h, w), bool)
        prune_mask = np.zeros((h, w), bool)
        if f > 0 and (fl & FLOW) and (fl & MASK):
            for tid in frames[f - 1]:
                _, lx, ly = tracks[tid][-1]
                fx0 = f32(lx * f32(w))
                fy0 = f32(f32(ly / ia) * f32(h))
                ix0 = min(max(int(f32(fx0 + f32(0.5))), 0), w - 1)
                iy0 = min(max(int(f32(fy0 + f32(0.5))), 0), h - 1)
                if not flow_mask[f, iy0, ix0]:
                    continue
                fx1 = f32(fx0 + flow[f, iy0, ix0, 0])
                fy1 = f32(fy0 + flow[f, iy0, ix0, 1])
                ix1 = int(f32(fx1 + f32(0.5)))
                iy1 = int(f32(fy1 + f32(0.5)))
                if 0 <= ix1 < w and 0 <= iy1 < h:
                    if not prune_mask[iy1, ix1] and dyn(int(f32(fy1 * sy)), int(f32(fx1 * sx))) >= mdd:
                        tracks[tid].append((f, f32(fx1 / f32(w)), f32(f32(fy1 / f32(h)) * ia)))
                        frames[f].append(tid)
                        _splat(prune_mask, prune_disk, ix1, iy1)
                        _splat(spawn_mask, spawn_disk, ix1, iy1)
        if f < F - 1:
            corner = cv2.cornerMinEigenVal(cv2.cvtColor(np.ascontiguousarray(color[f], f32), cv2.COLOR_BGR2GRAY), 3)
            cand = np.ones((h, w), bool) if not (fl & MASK) else flow_mask[f] != 0
            if dist is not None:
                ys = np.clip((np.arange(h, dtype=f32) * sy).astype(np.int64), 0, dh - 1)
                xs = np.clip((np.arange(w, dtype=f32) * sx).astype(np.int64), 0, dw - 1)
                cand &= dist[ys[:, None], xs[None, :]] > mdd
            idx = np.flatnonzero(cand)
            order = idx[np.argsort(-corner.ravel()[idx], kind="stable")]   # score descending, scan order on ties
            for p in order:
                y, x = divmod(int(p), w)
                px = f32(f32(x) / f32(w))
                py = f32(f32(f32(y) / f32(h)) * ia)
                mx = int(f32(px * f32(w)))
                my = int(f32(f32(py / ia) * f32(h)))
                if spawn_mask[my, mx]:
                    continue
                frames[f].append(len(tracks))
                tracks.append([(f, px, py)])
                _splat(spawn_mask, spawn_disk, mx, my)
    return tracks, frames


def delete_short(tracks, min_track_length):
    """The track table after the final pruning: None for deleted ids."""
    return [t if len(t) >= min_track_length else None for t in tracks]


def frame_lists(table, num_frames):
    """(offsets [F+1], ids, locs [n,2]) of a table, per local frame, ids ascending: the layout rcvd_compute_tracks returns."""
    per = [[] for _ in range(num_frames)]
    for tid, t in enumerate(table):
        if t is not None:
            for f, x, y in t:
                per[f].append((tid, x, y))
    offsets = np.zeros(num_frames + 1, np.int64)
    ids, locs = [], []
    for f in range(num_frames):
        offsets[f + 1] = offsets[f] + len(per[f])
        for tid, x, y in per[f]:
            ids.append(tid); locs.append((x, y))
    return offsets, np.asarray(ids, np.int32), np.asarray(locs, f32).reshape(-1, 2)


def serialize(table, video_frames, first_frame=0):
    """TrackTable::save (lib/core/TrackTable-impl.h:565-636): u64 ids; per id u8 valid, then u64 first frame, u64 length and
    length x (f32 x, f32 y); u64 frame offset (0), u64 frame count.  Frames are absolute: local frame + first_frame."""
    out = [struct.pack("<Q", len(table))]
    for t in table:
        if t is None:
            out.append(b"\x00")
        else:
            out.append(b"\x01" + struct.pack("<QQ", t[0][0] + first_frame, len(t)))
            out.append(np.asarray([(x, y) for _, x, y in t], f32).tobytes())
    out.append(struct.pack("<QQ", 0, video_frames))
    return b"".join(out)


# ---------------------------------------------------------------------------------------------------------
# inputs from a working directory, read the way DepthVideoProcessor::computeTracks reads them
# ---------------------------------------------------------------------------------------------------------
def load_inputs(root, frames, w, h, dynamic=False):
    """Local stacks over the absolute frames [frames[0], frames[-1]] (frames: the sorted frame range)."""
    import cv2
    from robust_cvd_b200 import synthetic_files as sf
    first, last = frames[0], frames[-1]
    F = last - first + 1
    color = np.zeros((F, h, w, 3), f32)
    flow = np.zeros((F, h, w, 2), f32)
    fmask = np.zeros((F, h, w), np.uint8)
    flags = np.zeros(F, np.uint8)
    dyn = None
    for i in range(F):
        a = first + i
        if a in frames:
            flags[i] |= IN_RANGE
        cf = os.path.join(root, "color_down", f"frame_{a:06d}.raw")
        if os.path.exists(cf):
            color[i] = sf.read_raw(cf); flags[i] |= HAS_COLOR
        ff = os.path.join(root, "flow", f"flow_{a - 1:06d}_{a:06d}.raw")
        if a > 0 and os.path.exists(ff):
            fl = sf.read_raw(ff)
            if fl.shape == (h, w, 2):
                flow[i] = fl; flags[i] |= FLOW
        mf = os.path.join(root, "flow_mask", f"mask_{a - 1:06d}_{a:06d}.png")
        if a > 0 and os.path.exists(mf):
            m = cv2.imread(mf, cv2.IMREAD_GRAYSCALE)
            if m.shape == (h, w):
                fmask[i] = m; flags[i] |= MASK
        if dynamic:
            m = cv2.imread(os.path.join(root, "dynamic_mask", f"frame_{a:06d}.png"), cv2.IMREAD_GRAYSCALE)
            if dyn is None:
                dyn = np.full((F,) + m.shape, 255, np.uint8)
            dyn[i] = m
    return color, flags, flow, fmask, dyn


# ---------------------------------------------------------------------------------------------------------
# golden
# ---------------------------------------------------------------------------------------------------------
def golden_inputs():
    """A small seeded clip: 6 frames 40x28, a constant sub-pixel drift, a dynamic mask with a blob, one frame out of range."""
    rng = np.random.default_rng(11)
    F, h, w = 6, 28, 40
    color = rng.uniform(0, 1, (F, h, w, 3)).astype(f32)
    flow = np.empty((F, h, w, 2), f32); flow[..., 0] = f32(1.3); flow[..., 1] = f32(-0.6)
    flow += rng.normal(0, 0.3, flow.shape).astype(f32)
    fmask = (rng.uniform(0, 1, (F, h, w)) > 0.1).astype(np.uint8) * 255
    dyn = np.full((F, 14, 20), 255, np.uint8); dyn[:, 4:9, 6:12] = 0
    flags = np.array([IN_RANGE | HAS_COLOR] + [IN_RANGE | HAS_COLOR | FLOW | MASK] * (F - 1), np.uint8)
    flags[4] = HAS_COLOR | FLOW | MASK
    return color, flags, flow, fmask, dyn


def golden_configs():
    return [("default", dict(spawn_distance=5, prune_distance=2, min_dynamic_distance=1)),
            ("dense", dict(spawn_distance=0, prune_distance=0, min_dynamic_distance=-1)),
            ("dyn", dict(spawn_distance=3, prune_distance=1, min_dynamic_distance=2, dynamic=True))]


def run_golden(name, kw):
    color, flags, flow, fmask, dyn = golden_inputs()
    kw = dict(kw)
    use_dyn = kw.pop("dynamic", False)
    tracks, _ = compute_tracks(color, flags, flow, fmask, dyn if use_dyn else None, inv_aspect=f32(28) / f32(40), **kw)
    return frame_lists(delete_short(tracks, 3), len(flags)), len(tracks)


def write_golden(path):
    out = {}
    for name, kw in golden_configs():
        (off, ids, locs), n = run_golden(name, kw)
        out[f"{name}_offsets"], out[f"{name}_ids"], out[f"{name}_locs"], out[f"{name}_count"] = off, ids, locs, np.int64(n)
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    write_golden(sys.argv[1] if len(sys.argv) > 1 else os.path.join(here, "golden", "tracks_golden.npz"))
