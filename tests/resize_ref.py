"""Plain float32 numpy restatement of cv2.resize(src, (w, h), interpolation=cv2.INTER_AREA) on float32 images (OpenCV 4.13's three
INTER_AREA paths, imgproc/src/resize.cpp), the reference for the k_resize_area kernel (robust_cvd_b200/csrc/rcvd_resize.cuh).

Every channel uses the same arithmetic; every operation is one float32 rounding (numpy never fuses).  The scale of an axis is
s = 1 / (dst / src) in double -- not src / dst, which differs in the last bit (98 -> 20 moves a tap).
  1. integer factors ix, iy >= 1 on both axes (|s - round(s)| < DBL_EPSILON): acc = 0, plus the cell's values in row-major order four
     at a time as acc += ((v0 + v1) + v2) + v3, then one at a time; the result acc * float32(1 / (ix iy)).
  2. other factors, both >= 1: per-axis area tables (weights in double, rounded to float32); each source row is resampled along x as
     buf = buf + v alpha over the x entries in order, each output row as sum = sum + beta buf over the y entries in order.
  3. either axis upscales: per axis two linear taps (i, 1 - f), (min(i + 1, n - 1), f) with i = floor(d s),
     f = float32((d + 1) - (i + 1) inv) (inv = dst / src), f = 0 if f <= 0 else f - floor(f); i >= n - 1 gives f = 0, i = n - 1.
     Horizontal first, v_i (1 - f) + v_i+1 f, then vertical over the horizontal results.  This is path 2's accumulation with two
     entries per output index: (0 + v0 a0) + v1 a1 = v0 a0 + v1 a1 for the non-negative values of an image.
"""
import math
import sys

import numpy as np

DBL_EPSILON = sys.float_info.epsilon


def axis_scale(n_src, n_dst):
    return 1.0 / (n_dst / n_src)


def area_fast_factors(W, H, w, h):
    """(ix, iy) when both axes have integer factors >= 1 (path 1), else None."""
    sx, sy = axis_scale(W, w), axis_scale(H, h)
    ix, iy = int(np.rint(sx)), int(np.rint(sy))
    if sx >= 1 and sy >= 1 and abs(sx - ix) < DBL_EPSILON and abs(sy - iy) < DBL_EPSILON:
        return ix, iy
    return None


def resize_path(W, H, w, h):
    """'integer', 'area' or 'linear': the INTER_AREA path cv2 takes for W x H -> w x h."""
    if area_fast_factors(W, H, w, h):
        return "integer"
    return "area" if axis_scale(W, w) >= 1 and axis_scale(H, h) >= 1 else "linear"


def area_taps(n, m):
    """computeResizeAreaTab: per output index the list of (source index, float32 weight)."""
    s = axis_scale(n, m)
    taps = []
    for d in range(m):
        f1 = d * s
        f2 = f1 + s
        cw = min(s, n - f1)
        i1, i2 = math.ceil(f1), math.floor(f2)
        i2 = min(i2, n - 1)
        i1 = min(i1, i2)
        t = []
        if i1 - f1 > 1e-3:
            t.append((i1 - 1, np.float32((i1 - f1) / cw)))
        for k in range(i1, i2):
            t.append((k, np.float32(1.0 / cw)))
        if f2 - i2 > 1e-3:
            t.append((i2, np.float32(min(min(f2 - i2, 1.0), cw) / cw)))
        taps.append(t)
    return taps


def linear_taps(n, m):
    """The upscale path's two taps per output index."""
    s, inv = axis_scale(n, m), m / n
    taps = []
    for d in range(m):
        i = math.floor(d * s)
        f = np.float32((d + 1) - (i + 1) * inv)
        f = np.float32(0) if f <= 0 else np.float32(f - np.float32(math.floor(f)))
        if i >= n - 1:
            f, i = np.float32(0), n - 1
        taps.append([(i, np.float32(1) - f), (min(i + 1, n - 1), f)])
    return taps


def _accumulate(img, taps, axis):
    """acc = acc + v * weight over each output index's taps in order, along `axis` (0 rows, 1 columns), starting from 0."""
    img = np.moveaxis(img, axis, 0)
    out = np.zeros((len(taps),) + img.shape[1:], np.float32)
    for slot in range(max(len(t) for t in taps)):
        d = np.array([k for k, t in enumerate(taps) if len(t) > slot], np.int64)
        src = np.array([taps[k][slot][0] for k in d], np.int64)
        wt = np.array([taps[k][slot][1] for k in d], np.float32).reshape((-1,) + (1,) * (img.ndim - 1))
        out[d] = out[d] + img[src] * wt
    return np.moveaxis(out, 0, axis)


def resize_area(img, w, h):
    """cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA) for a float32 [H, W, C] image."""
    img = np.asarray(img, np.float32)
    H, W = img.shape[:2]
    fast = area_fast_factors(W, H, w, h)
    if fast:
        ix, iy = fast
        cells = img[:h * iy, :w * ix].reshape(h, iy, w, ix, -1).transpose(0, 2, 1, 3, 4).reshape(h, w, iy * ix, -1)
        n = ix * iy
        acc = np.zeros((h, w, cells.shape[-1]), np.float32)
        k = 0
        while k + 4 <= n:
            acc = acc + (((cells[:, :, k] + cells[:, :, k + 1]) + cells[:, :, k + 2]) + cells[:, :, k + 3])
            k += 4
        for k in range(k, n):
            acc = acc + cells[:, :, k]
        return acc * (np.float32(1) / np.float32(n))
    taps = area_taps if resize_path(W, H, w, h) == "area" else linear_taps
    return _accumulate(_accumulate(img, taps(W, w), 1), taps(H, h), 0)


def to_float(u8):
    """np.float32(img) / 255.0: one float32 division."""
    return np.float32(u8) / np.float32(255.0)


def to_png_u8(img):
    """cv2.imwrite(fn, img * 255)'s pixels: float32 x * 255, rounded half to even and saturated to u8."""
    return np.clip(np.rint(np.asarray(img, np.float32) * np.float32(255)), 0, 255).astype(np.uint8)
