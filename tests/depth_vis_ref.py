"""numpy restatement of the reference's depth visualisation (utils/visualization.py:53-134) for the tests: the range of
visualize_depth_dir (np.percentile of each frame's finite values, Python's min / max from sys.float_info.max and sys.float_info.min), the
u8 index of visualize_depth, cv2.applyColorMap's gray conversion of a 3-channel index, and the colour table after it.  It uses numpy
only, so the tests can compare against it where the reference tree and cv2 are absent."""
import sys

import numpy as np


def frame_range(frames, min_percentile, max_percentile):
    """(d_min, d_max) of visualize_depth_dir over `frames` (each a float32 [h, w] or u8 [h, w, 3] array, in file order), as the numpy
    scalars or Python floats the reference holds."""
    d_min = sys.float_info.max
    d_max = sys.float_info.min
    for d in frames:
        ix = np.isfinite(d)
        if np.sum(ix) == 0:
            continue
        valid = d[ix]
        d_min = min(d_min, np.percentile(valid, min_percentile))
        d_max = max(d_max, np.percentile(valid, max_percentile))
    return d_min, d_max


def gray(bgr):
    """cv::cvtColor(COLOR_BGR2GRAY) of 8-bit B, G, R values (15-bit fixed point, equal to cv2 over all 2^24 colours)."""
    b, g, r = (bgr[..., c].astype(np.int64) for c in range(3))
    return ((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15).astype(np.uint8)


def index(depth, depth_min, depth_max):
    """The u8 colormap index of visualize_depth: np.uint8(((depth - depth_min) / (depth_max - depth_min)) ** 0.5 * 255), converted to
    gray for a 3-channel image."""
    with np.errstate(all="ignore"):
        s = (depth - depth_min) / (depth_max - depth_min)
        s = s ** 0.5
        idx = np.uint8(s * 255)
    return gray(idx) if idx.ndim == 3 else idx


def tables(lut):
    """(float64 [256, 3] B, G, R: ((lut / 255) ** 2.2) * 255, u8 [256, 3] R, G, B: cv2.imwrite's pixels of it)."""
    f64 = ((np.asarray(lut, np.uint8).reshape(256, 3) / 255) ** 2.2) * 255
    return f64, np.clip(np.rint(f64), 0, 255).astype(np.uint8)[:, ::-1]


def visualize_dir(frames, min_percentile, max_percentile, lut):
    """(d_min, d_max, [R, G, B u8 [h, w, 3] per frame]) of visualize_depth_dir with force."""
    d_min, d_max = frame_range(frames, min_percentile, max_percentile)
    _, rgb = tables(lut)
    return d_min, d_max, [rgb[index(d, d_min, d_max)] for d in frames]
