"""Literal numpy transcription of FlowConstraintsCollection::pruneStaticFlag (reference lib/FlowConstraints.cpp:662-748) and of
buildDiskMask, the oracle of the host restatement (robust_cvd_b200/host/constraints.cpp) and of rcvd_prune_static_flags.

Two deliberate differences from the reference, both where it has no defined result:
  - the phase-2 lookups clamp the pixel to the image, where the reference indexes the mask unchecked (a "down" stream whose aspect
    differs from the video's makes int(loc.y * w) reach h);
  - a negative distance changes no flag, where the reference fails in OpenCV's Mat allocation.

pairs:    {(frame0, frame1): (locs [n, 4] float32, isStatic [n] bool)}
triplets: {centre: (locs [n, 6] float32, isStatic [n] bool)}
"""
import numpy as np


def build_disk_mask(distance):
    size = 2 * distance + 1
    mask = np.zeros((size, size), np.uint8)
    for y in range(size):
        for x in range(size):
            rx, ry = x - distance, y - distance
            mask[y, x] = 255 if rx * rx + ry * ry <= distance * distance else 0
    return mask


def end_pixel(loc, w):
    """(int(loc.x * w), int(loc.y * w)): float32 products, truncated toward zero; y is scaled by the WIDTH as in the reference."""
    return int(np.float32(loc[0]) * np.float32(w)), int(np.float32(loc[1]) * np.float32(w))


def prune_static_flag(pairs, triplets, num_frames, h, w, distance):
    """Returns the pruned flags ({key: isStatic [n] bool} for pairs, the same for triplets); the inputs are not modified."""
    out_p = {k: np.array(v[1], bool) for k, v in pairs.items()}
    out_t = {k: np.array(v[1], bool) for k, v in triplets.items()}
    if distance < 0:
        return out_p, out_t
    keys = sorted(pairs)                                   # std::map order
    disk_mask = build_disk_mask(distance)
    masks = [None] * num_frames
    for frame in range(num_frames):
        mask = np.zeros((h, w), np.uint8)
        masks[frame] = mask
        for key in keys:
            if key[0] != frame and key[1] != frame:
                continue
            locs, static = pairs[key]
            for c in range(len(locs)):
                if static[c]:
                    continue
                loc = locs[c, 0:2] if key[0] == frame else locs[c, 2:4]
                x, y = end_pixel(loc, w)
                mx0, mx1 = max(0, x - distance), min(w - 1, x + distance)
                my0, my1 = max(0, y - distance), min(h - 1, y + distance)
                if mx0 > mx1:
                    continue
                for my in range(my0, my1 + 1):
                    dy = my - (y - distance)
                    disk_row = disk_mask[dy, mx0 - (x - distance):mx1 - (x - distance) + 1]     # the mx loop, one row at a time
                    mask[my, mx0:mx1 + 1][disk_row != 0] = 255

    def at(frame, loc):
        x, y = end_pixel(loc, w)
        return masks[frame][min(max(y, 0), h - 1), min(max(x, 0), w - 1)] != 0

    for key in keys:
        locs = pairs[key][0]
        for c in range(len(locs)):
            if at(key[0], locs[c, 0:2]) or at(key[1], locs[c, 2:4]):
                out_p[key][c] = False
    for t in sorted(triplets):
        locs = triplets[t][0]
        for c in range(len(locs)):
            if at(t - 1, locs[c, 0:2]) or at(t, locs[c, 2:4]) or at(t + 1, locs[c, 4:6]):
                out_t[t][c] = False
    return out_p, out_t
