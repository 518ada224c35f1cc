"""Flow-consistency masks and pair mask ratios of a robust_cvd working directory, with the mask arithmetic on the GPU.

Drop-in for the reference's Flow.compute_flow_masks and Flow.compute_flow_pair_stats (flow.py:44-74, :180-209), which process.py runs
after RAFT: it reads flow/flow_%06d_%06d.raw and color_down/frame_%06d.raw and writes flow_mask/mask_%06d_%06d.png (8-bit, 0 / 255)
and flow_list.json, the files the constraint builder, static flags, tracks and filters read.  The per-pixel test is rcvd_flow_masks
(include/rcvd.h); the files are read with numpy, and the PNGs are encoded on a thread pool while the next chunk of pairs computes.

There is no CPU fallback: without librcvd_b200.so or a usable CUDA device compute_flow_masks raises RuntimeError.
"""
import json
import os
import re
import struct
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import solver
from .synthetic_files import read_raw

FLOW_FMT = os.path.join("flow", "flow_{:06d}_{:06d}.raw")
MASK_FMT = os.path.join("flow_mask", "mask_{:06d}_{:06d}.png")
COLOR_FMT = os.path.join("color_down", "frame_{:06d}.raw")
_FLOW_NAME = re.compile(r"^flow_(\d+)_(\d+)\.raw$")


def pairs_to_compute(path):
    """The pairs (i, j) whose two masks compute_flow_masks writes, in the order of the flow/ listing.  The reference walks that listing
    and skips a flow whose own mask exists; otherwise it computes and writes both masks of the pair, so the reverse flow is skipped
    later.  The net effect: a pair is computed once, from the first of its flows listed, when either of its masks is missing."""
    done = set()
    out = []
    for name in os.listdir(os.path.join(path, "flow")):
        m = _FLOW_NAME.match(name)
        if not m:
            continue
        i, j = int(m.group(1)), int(m.group(2))
        if (i, j) in done or os.path.isfile(os.path.join(path, MASK_FMT.format(i, j))):
            continue
        out.append((i, j))
        done.update(((i, j), (j, i)))
    return out


def _raw_shape(fn):
    """(rows, cols, channels) from the 20-byte header of a .raw file (lib/core/CvUtil.cpp)."""
    with open(fn, "rb") as f:
        head = f.read(20)
    if len(head) < 20:
        raise ValueError(f"{fn}: not a .raw image")
    rows, cols, typ, _ = struct.unpack("<iiiQ", head)
    return rows, cols, (typ >> 3) + 1


def _check_inputs(path, pairs):
    """Every file a pair reads exists, and each flow has its colour images' size: refused before any mask is written."""
    for i, j in pairs:
        for a, b in ((i, j), (j, i)):
            fn = os.path.join(path, FLOW_FMT.format(a, b))
            if not os.path.isfile(fn):
                raise FileNotFoundError(f"flow {a} -> {b} is missing ({fn}): the masks of a pair need both of its flows")
        shapes = {}
        for fn in (FLOW_FMT.format(i, j), FLOW_FMT.format(j, i), COLOR_FMT.format(i), COLOR_FMT.format(j)):
            full = os.path.join(path, fn)
            if not os.path.isfile(full):
                raise FileNotFoundError(f"{full} is missing")
            shapes[fn] = _raw_shape(full)
        sizes = {s[:2] for s in shapes.values()}
        chans = [s[2] for s in shapes.values()]
        if len(sizes) != 1 or chans != [2, 2, 3, 3]:
            raise ValueError(f"pair ({i}, {j}): flow and colour images differ in size or channels: {shapes}")


def png_gray_bytes(img, level=1):
    """An 8-bit grayscale PNG of img [h, w] u8 (filter type 0 on every row, one zlib IDAT)."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    raw = np.zeros((h, w + 1), np.uint8)
    raw[:, 1:] = img

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(raw.tobytes(), level)) + chunk(b"IEND", b""))


def _write_png(fn, img):
    t = time.perf_counter()
    data = png_gray_bytes(img)
    with open(fn, "wb") as f:
        f.write(data)
    return time.perf_counter() - t


def _chunks(pairs, plane_bytes, chunk_bytes):
    """Consecutive groups of pairs whose flows and colours take at most chunk_bytes of host memory (at least one pair each)."""
    out, cur, frames = [], [], set()
    for p in pairs:
        new = frames | set(p)
        if cur and (len(cur) + 1) * 16 * plane_bytes + len(new) * 12 * plane_bytes > chunk_bytes:
            out.append(cur)
            cur, new = [], set(p)
        cur.append(p)
        frames = new
    if cur:
        out.append(cur)
    return out


def _read_chunk(path, chunk, files):
    """The colours and both flows of a chunk of pairs, read by the `files` thread pool (file reads release the GIL)."""
    t = time.perf_counter()
    frames = sorted({f for p in chunk for f in p})
    local = {f: k for k, f in enumerate(frames)}

    def stack(fmt, keys):
        return np.stack(list(files.map(lambda k: read_raw(os.path.join(path, fmt.format(*k))), keys)))
    colors = stack(COLOR_FMT, [(f,) for f in frames])
    fij = stack(FLOW_FMT, chunk)
    fji = stack(FLOW_FMT, [(j, i) for i, j in chunk])
    pf = np.array([[local[i], local[j]] for i, j in chunk], np.int32)
    return colors, pf, fij, fji, time.perf_counter() - t


def compute_flow_masks(path, flow_thresh=1, color_thresh=1, device=None, chunk_bytes=256 << 20, workers=None):
    """Flow.compute_flow_masks on the GPU: writes flow_mask/mask_i_j.png and mask_j_i.png for every pair of pairs_to_compute(path).
    flow_thresh / color_thresh as in the reference (thresholds float32(flow_thresh^2) and float32(3 color_thresh^2)).  Pairs are
    processed in chunks of at most chunk_bytes of flows and colours; PNGs are encoded by `workers` threads while the next chunk reads
    and computes.  A missing reverse flow or colour image, or a flow whose size differs from its colours, raises before anything is
    written.  Returns timings: {"pairs", "read_s", "compute_s", "png_s" (encode + write, summed over threads), "wait_s" (the caller's
    thread blocked on reads and writes), "total_s"}."""
    t0 = time.perf_counter()
    L = solver.lib()
    dev = L.rcvd_current_device() if device is None else int(device)
    if dev < 0:
        raise RuntimeError("rcvd error 5: no usable CUDA device for the flow masks; this library has no CPU fallback")
    os.makedirs(os.path.join(path, "flow_mask"), exist_ok=True)
    pairs = pairs_to_compute(path)
    stats = {"pairs": len(pairs), "read_s": 0.0, "compute_s": 0.0, "png_s": 0.0, "wait_s": 0.0, "total_s": 0.0}
    if not pairs:
        stats["total_s"] = time.perf_counter() - t0
        return stats
    _check_inputs(path, pairs)
    rows, cols, _ = _raw_shape(os.path.join(path, COLOR_FMT.format(pairs[0][0])))
    fsq = np.float32(flow_thresh ** 2)
    csq = np.float32(3 * color_thresh ** 2)
    chunks = _chunks(pairs, rows * cols, chunk_bytes)
    workers = workers or min(8, os.cpu_count() or 1)
    with ThreadPoolExecutor(1) as reader, ThreadPoolExecutor(4) as files, ThreadPoolExecutor(workers) as writers:
        pending = []
        nxt = reader.submit(_read_chunk, path, chunks[0], files)
        for k, chunk in enumerate(chunks):
            t = time.perf_counter()
            colors, pf, fij, fji, rs = nxt.result()
            stats["wait_s"] += time.perf_counter() - t
            stats["read_s"] += rs
            if k + 1 < len(chunks):
                nxt = reader.submit(_read_chunk, path, chunks[k + 1], files)
            t = time.perf_counter()
            mij, mji, _ = solver.flow_masks(colors, pf, fij, fji, fsq, csq, device=dev)
            stats["compute_s"] += time.perf_counter() - t
            del colors, fij, fji
            t = time.perf_counter()
            stats["png_s"] += sum(f.result() for f in pending)   # at most one chunk of masks waits for its PNGs
            stats["wait_s"] += time.perf_counter() - t
            pending = []
            for n, (i, j) in enumerate(chunk):
                pending.append(writers.submit(_write_png, os.path.join(path, MASK_FMT.format(i, j)), mij[n]))
                pending.append(writers.submit(_write_png, os.path.join(path, MASK_FMT.format(j, i)), mji[n]))
        t = time.perf_counter()
        stats["png_s"] += sum(f.result() for f in pending)
        stats["wait_s"] += time.perf_counter() - t
    stats["total_s"] = time.perf_counter() - t0
    return stats


def _read_mask(fn):
    """A mask PNG through the project's PNG decoder (lib_python._imreadPng, the cv::imread subset the C++ readers use)."""
    host = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host")
    if host not in sys.path:
        sys.path.insert(0, host)
    import lib_python
    if not os.path.isfile(fn):
        raise FileNotFoundError(f"{fn} is missing")
    return lib_python._imreadPng(fn, True)


def compute_flow_pair_stats(path, frame_pairs):
    """Flow.compute_flow_pair_stats: returns the path of flow_list.json if it exists, untouched.  Otherwise, for each pair of
    frame_pairs not seen before in either direction (the caller's order), r = min over its two masks of (non-zero pixels) / (h w), and
    the rows [a, b, r], [b, a, r] follow the header ["frame0", "frame1", "mask_ratio"] in the json.dump the reference writes.  Like the
    reference, returns None after writing."""
    flow_list_path = os.path.join(path, "flow_list.json")
    if os.path.isfile(flow_list_path):
        return flow_list_path
    results = [["frame0", "frame1", "mask_ratio"]]
    checked = set()
    for pair in frame_pairs:
        key = tuple(pair)
        if key in checked:
            continue
        checked.update((key, key[::-1]))
        ratios = []
        for a, b in (key, key[::-1]):
            m = _read_mask(os.path.join(path, MASK_FMT.format(a, b)))
            ratios.append(np.count_nonzero(m) / (m.shape[0] * m.shape[1]))
        r = min(ratios)
        results.append([pair[0], pair[1], r])
        results.append([pair[1], pair[0], r])
        print(f"Frames {pair[0]} <-> {pair[1]}: mask_ratio = {r*100:04.1f}%")
    with open(flow_list_path, "w") as f:
        json.dump(list(results), f)


class Flow:
    """The mask and pair-statistics stages of the reference's Flow class (flow.py), on the GPU: a caller of
    Flow(path, out_path).compute_flow_masks() / .compute_flow_pair_stats(frame_pairs) switches by importing this class instead.  RAFT
    (compute_flow) and the visualisation are not part of it."""

    def __init__(self, path, out_path):
        self.path = path
        self.out_path = out_path

    @staticmethod
    def max_size():
        return 1024

    def compute_flow_masks(self, flow_thresh=1, color_thresh=1):
        compute_flow_masks(self.path, flow_thresh, color_thresh)

    def compute_flow_pair_stats(self, frame_pairs):
        return compute_flow_pair_stats(self.path, frame_pairs)
