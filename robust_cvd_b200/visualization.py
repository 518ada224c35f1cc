"""Depth visualisations of a robust_cvd working directory, rendered on the GPU.

Drop-in for the reference's visualization.visualize_depth_dir and visualize_depth (utils/visualization.py:53-134), which
DepthFineTuner.save_depth runs with --save_depth_visualization (depth/frame_*.png next to the .raw disparities) and the fine-tuning
evaluation runs on each saved disparity.  The percentile range of every frame is a radix select on the GPU and the colouring one
thread per pixel (rcvd_depth_visualize, include/rcvd.h); the host keeps numpy's arithmetic where it decides a value: np.percentile's
linear interpolation from the selected order statistics, Python's min / max over the frames, NEP 50's weak Python scalars.  Frames are
read on a thread pool in chunks, kept in memory between the two passes while they fit, and the PNGs are encoded on another pool.

After the u8 index, the reference's chain cv2.applyColorMap(index, colormap), ((c / 255) ** 2.2) * 255 and cv2.imwrite (round half to
even, saturate, B, G, R stored as R, G, B) is a 256 x 3 table; it is computed with numpy from the colormap at call time.

Deviations: a .raw that is not single-channel float32, and an image the project's PNG decoder cannot read (anything but an 8-bit,
non-interlaced PNG), are refused before anything is written; the reference crashes part-way.  A missing dst_dir is created.
Percentiles are taken as Python floats.  visualize_depth takes float32 [h, w] or u8 [h, w, 3] frames, with bounds that keep numpy's
arithmetic in float32 and float64 respectively, and refuses other types.

There is no CPU fallback: without librcvd_b200.so or a usable CUDA device both functions raise RuntimeError.
"""
import logging
import os
import os.path as osp
import struct
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import solver
from .png import png_header, write_png
from .synthetic_files import read_raw
from .video import _decode_png


def resolve_colormap(colormap=None):
    """The colormap as a [256, 3] u8 table of cv2.applyColorMap's user-colormap contract (entry k holds the B, G, R of index k).
    colormap: None (the reference's utils.colormaps.cm_magma, imported from the caller's path), a 256-entry 3-channel u8 array, or a
    cv2 colormap id (cv2.COLORMAP_*)."""
    if colormap is None:
        try:
            from utils import colormaps
            colormap = colormaps.cm_magma
        except (ImportError, AttributeError) as e:
            raise RuntimeError("the default colormap is the reference's utils.colormaps.cm_magma, which could not be imported "
                               f"({e}); pass colormap= (a 256-entry B, G, R u8 array or a cv2 colormap id)") from e
    if isinstance(colormap, (int, np.integer)):
        import cv2
        return cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), int(colormap)).reshape(256, 3)
    table = np.asarray(colormap)
    if table.dtype != np.uint8 or table.size != 256 * 3 or table.shape[-1] != 3:
        raise ValueError(f"colormap of shape {table.shape} and type {table.dtype}: need 256 B, G, R entries of type uint8")
    return np.ascontiguousarray(table.reshape(256, 3))


def color_tables(table):
    """(float64 [256, 3] B, G, R: visualize_depth's values ((c / 255) ** 2.2) * 255 per index, u8 [256, 3] R, G, B: the pixels
    cv2.imwrite stores for them, rounded half to even and saturated)."""
    f64 = ((table / 255) ** 2.2) * 255
    return f64, np.ascontiguousarray(np.clip(np.rint(f64), 0, 255).astype(np.uint8)[:, ::-1])


def quantile(p, dtype):
    """np.percentile's quantile p / 100 for an array of `dtype`: float32 division for a float32 array, float64 otherwise."""
    dtype = np.dtype(dtype)
    return np.asanyarray(np.true_divide(float(p), dtype.type(100) if dtype.kind == "f" else 100))


def _virtual_index(n, qf):
    """numpy's linear method for n sorted values: (previous rank, next rank, gamma), as _quantile / _get_indexes / _get_gamma compute
    them (v = (n - 1) q in q's type; both ranks n - 1 when v >= n - 1, where gamma is v + 1 and does not matter)."""
    v = np.asanyarray((n - 1) * qf)
    prev = np.asanyarray(np.floor(v))
    nxt = np.asanyarray(prev + 1)
    if v >= n - 1:
        prev[...] = -1
        nxt[...] = -1
    prev, nxt = prev.astype(np.intp), nxt.astype(np.intp)
    gamma = np.asanyarray(np.asanyarray(v - prev), dtype=v.dtype)
    return int(prev) % n, int(nxt) % n, gamma


def percentile_from_ranks(n, qf, prev_value, next_value, dtype):
    """np.percentile(values, p) of n values of `dtype` from the order statistics at _virtual_index(n, qf)'s ranks (qf =
    quantile(p, dtype)): numpy's _lerp on the values as numpy scalars of `dtype`."""
    a, b = np.dtype(dtype).type(prev_value), np.dtype(dtype).type(next_value)
    t = _virtual_index(n, qf)[2]
    diff = np.subtract(b, a)
    lerp = np.asanyarray(np.add(a, diff * t))
    np.subtract(b, diff * (1 - t), out=lerp, where=t >= 0.5, casting="unsafe", dtype=type(lerp.dtype))
    return lerp[()]


def colour_bounds(dtype, depth_min, depth_max):
    """(kind, offset, scale) of the colour pass for frames of `dtype` with bounds (depth_min, depth_max): the float type numpy computes
    (depth - depth_min) / (depth_max - depth_min) in, and both bounds as that type sees them.  float32 frames need that arithmetic in
    float32 and u8 images in float64; other combinations are refused."""
    dtype = np.dtype(dtype)
    with np.errstate(all="ignore"):
        num = np.empty(0, dtype) - depth_min
        den = depth_max - depth_min
        res = num / den
        if dtype == np.float32 and num.dtype == res.dtype == np.float32:
            return 0, float(np.float32(depth_min)), float(np.float32(den))
        if dtype == np.uint8 and num.dtype == res.dtype == np.float64:
            return 1, float(depth_min), float(den)
    raise ValueError(f"{dtype} frames with bounds of type {type(depth_min).__name__} and {type(depth_max).__name__} compute in "
                     f"{num.dtype} / {res.dtype}: need float32 frames computed in float32 or u8 images computed in float64")


def visualize_depth(depth, depth_min=None, depth_max=None, colormap=None, device=None):
    """The reference's visualize_depth: depth rescaled so that depth_min and depth_max map to 0 and 1 (np.nanmin / np.nanmax when
    None, so +-inf included), square-rooted, cast to u8 and coloured, as the float64 [h, w, 3] B, G, R array the reference returns.
    depth: float32 [h, w] or u8 [h, w, 3] (B, G, R, converted to gray after the index)."""
    depth = np.asarray(depth)
    if not ((depth.dtype == np.float32 and depth.ndim == 2) or (depth.dtype == np.uint8 and depth.ndim == 3 and depth.shape[2] == 3)):
        raise ValueError(f"depth of shape {depth.shape} and type {depth.dtype}: need float32 [h, w] or u8 [h, w, 3]")
    table64, _ = color_tables(resolve_colormap(colormap))
    if depth_min is None:
        depth_min = np.nanmin(depth)
    if depth_max is None:
        depth_max = np.nanmax(depth)
    _, offset, scale = colour_bounds(depth.dtype, depth_min, depth_max)
    _, idx = solver.depth_colorize(depth[None], offset, scale, index=True, device=_device(device))
    return table64[idx[0]]


def _device(device):
    dev = solver.lib().rcvd_current_device() if device is None else int(device)
    if dev < 0:
        raise RuntimeError("rcvd error 5: no usable CUDA device for the depth visualisation; this library has no CPU fallback")
    return dev


def _frame_bytes(fn, raw):
    """Bytes of a frame as read, after checking that it can be read: a .raw must be single-channel float32, an image an 8-bit,
    non-interlaced PNG (the project's decoder)."""
    if raw:
        with open(fn, "rb") as f:
            head = f.read(20)
        if len(head) < 20:
            raise ValueError(f"{fn}: not a .raw image")
        rows, cols, typ, _ = struct.unpack("<iiiQ", head)
        if typ != 5:
            raise ValueError(f"{fn}: a .raw of type {typ & 7} with {(typ >> 3) + 1} channels; depth must be single-channel float32")
        return rows * cols * 4
    try:
        hd = png_header(fn)
    except ValueError as e:
        raise ValueError(f"{fn} cannot be read: {e}; images are read by the project's PNG decoder") from e
    if hd["bit_depth"] != 8 or hd["interlace"]:
        raise ValueError(f"{fn} cannot be read: a {hd['bit_depth']}-bit{' interlaced' if hd['interlace'] else ''} PNG; the "
                         "project's PNG decoder reads 8-bit, non-interlaced PNGs")
    return hd["height"] * hd["width"] * 3


def _read_frame(fn, raw):
    if raw:
        return read_raw(fn)
    try:
        return _decode_png(fn)
    except RuntimeError as e:
        raise ValueError(f"{fn} cannot be read: {e}") from e


def _read_chunk(src_dir, names, raw, files):
    t = time.perf_counter()
    frames = list(files.map(lambda n: _read_frame(osp.join(src_dir, n), raw), names))
    return frames, time.perf_counter() - t


def _chunks(items, sizes, chunk_bytes):
    """Consecutive groups of items whose sizes sum to at most chunk_bytes (at least one item each)."""
    out, cur, total = [], [], 0
    for it, s in zip(items, sizes):
        if cur and total + s > chunk_bytes:
            out.append(cur)
            cur, total = [], 0
        cur.append(it)
        total += s
    if cur:
        out.append(cur)
    return out


def _by_shape(frames):
    """{shape: indices into frames} in first-seen order: one GPU call per frame size."""
    groups = {}
    for k, f in enumerate(frames):
        groups.setdefault(f.shape, []).append(k)
    return groups


def _chunk_stream(src_dir, chunks, names, raw, reader, files):
    """Yields (chunk, frames, read seconds) for each chunk of indices into names, reading the next chunk while the caller works."""
    nxt = reader.submit(_read_chunk, src_dir, [names[i] for i in chunks[0]], raw, files) if chunks else None
    for k, chunk in enumerate(chunks):
        frames, rs = nxt.result()
        if k + 1 < len(chunks):
            nxt = reader.submit(_read_chunk, src_dir, [names[i] for i in chunks[k + 1]], raw, files)
        yield chunk, frames, rs


def visualize_depth_dir(src_dir, dst_dir, force=False, extension=".raw", min_percentile=0, max_percentile=100, colormap=None,
                        device=None, chunk_bytes=256 << 20, resident_bytes=2 << 30, workers=None):
    """The reference's visualize_depth_dir: every file of src_dir whose lower-cased extension is `extension`, in sorted order, written
    as dst_dir/<base>.png through visualize_depth with one range over all of them: the smallest min_percentile and the largest
    max_percentile of each frame's finite values (Python's min and max, from sys.float_info.max and sys.float_info.min; a frame with
    none logs a warning, takes no part and is still written).  Returns at once when nothing matches, or when every output exists and
    force is false; otherwise, without force, each existing output is skipped.  .raw files are float32 disparities; other extensions
    are read as cv2.imread's 3-channel B, G, R images.  Frames are read in chunks of at most chunk_bytes, kept in memory for the second
    pass when all of them take at most resident_bytes, else read again.  Returns timings: {"frames", "written", "read_s",
    "compute_s", "write_s" (summed over threads), "resident", "total_s"}; None where the reference returns early."""
    t0 = time.perf_counter()
    src_files, dst_files = [], []
    for file in sorted(os.listdir(src_dir)):
        base, ext = osp.splitext(file)
        if ext.lower() == extension:
            src_files.append(file)
            dst_files.append(f"{base}.png")
    if len(src_files) == 0:
        return None
    if not force and all(osp.exists(osp.join(dst_dir, f)) for f in dst_files):
        return None
    if not (0 <= float(min_percentile) <= 100 and 0 <= float(max_percentile) <= 100):
        raise ValueError("Percentiles must be in the range [0, 100]")
    raw = extension == ".raw"
    dtype = np.float32 if raw else np.uint8
    qs = (quantile(min_percentile, dtype), quantile(max_percentile, dtype))
    workers = workers or min(8, os.cpu_count() or 1)
    stats = {"frames": len(src_files), "written": 0, "read_s": 0.0, "compute_s": 0.0, "write_s": 0.0, "resident": False,
             "total_s": 0.0}
    with ThreadPoolExecutor(1) as reader, ThreadPoolExecutor(workers) as files, ThreadPoolExecutor(workers) as writers:
        sizes = list(files.map(lambda n: _frame_bytes(osp.join(src_dir, n), raw), src_files))
        table = resolve_colormap(colormap)
        dev = _device(device)
        _, lut = color_tables(table)
        resident = sum(sizes) <= resident_bytes
        stats["resident"] = resident
        kept = [None] * len(src_files)
        d_min = sys.float_info.max
        d_max = sys.float_info.min
        chunks = _chunks(range(len(src_files)), sizes, chunk_bytes)
        for chunk, frames, rs in _chunk_stream(src_dir, chunks, src_files, raw, reader, files):
            stats["read_s"] += rs
            t = time.perf_counter()
            counts, order = np.empty(len(chunk), np.int64), np.empty((len(chunk), 4))
            for ks in _by_shape(frames).values():
                counts[ks], order[ks] = solver.depth_range(np.stack([frames[k] for k in ks]), [float(q) for q in qs], device=dev)
            stats["compute_s"] += time.perf_counter() - t
            for k, i in enumerate(chunk):
                print("reading '%s'." % src_files[i])
                n = int(counts[k])
                if n == 0:
                    logging.warning(f"{src_files[i]} has 0 valid depth")
                    continue
                d_min = min(d_min, percentile_from_ranks(n, qs[0], order[k, 0], order[k, 1], dtype))
                d_max = max(d_max, percentile_from_ranks(n, qs[1], order[k, 2], order[k, 3], dtype))
            if resident:
                for k, i in enumerate(chunk):
                    kept[i] = frames[k]
            del frames
        _, offset, scale = colour_bounds(dtype, d_min, d_max)
        os.makedirs(dst_dir, exist_ok=True)
        todo = [i for i in range(len(src_files)) if force or not osp.exists(osp.join(dst_dir, dst_files[i]))]
        done = set(todo)
        if resident:
            chunks2 = [(c, [kept[i] for i in c], 0.0) for c in _chunks(todo, [sizes[i] for i in todo], chunk_bytes)]
        else:
            chunks2 = _chunk_stream(src_dir, _chunks(todo, [sizes[i] for i in todo], chunk_bytes), src_files, raw, reader, files)
        pending, shown = [], 0
        for chunk, frames, rs in chunks2:
            stats["read_s"] += rs
            t = time.perf_counter()
            rgb = [None] * len(chunk)
            for ks in _by_shape(frames).values():
                out = solver.depth_colorize(np.stack([frames[k] for k in ks]), offset, scale, lut, device=dev)
                for j, k in enumerate(ks):
                    rgb[k] = out[j]
            stats["compute_s"] += time.perf_counter() - t
            stats["write_s"] += sum(f.result() for f in pending)   # at most one chunk of outputs waits for its files
            pending = []
            for k, i in enumerate(chunk):
                while shown <= i:   # the reference's messages, in file order
                    print(f"reading '{src_files[shown]}'.")
                    print(f"writing '{dst_files[shown]}'." if shown in done else f"skipping existing file '{dst_files[shown]}'.")
                    shown += 1
                pending.append(writers.submit(write_png, osp.join(dst_dir, dst_files[i]), rgb[k]))
            del frames, rgb
        stats["write_s"] += sum(f.result() for f in pending)
        for s in range(shown, len(src_files)):
            print(f"reading '{src_files[s]}'.")
            print(f"skipping existing file '{dst_files[s]}'.")
        stats["written"] = len(todo)
    stats["total_s"] = time.perf_counter() - t0
    return stats
