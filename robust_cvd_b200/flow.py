"""Homography-registered optical flows, flow-consistency masks, pair mask ratios and flow visualisations of a robust_cvd working
directory, with the per-pixel work on the GPU.

Drop-in for the reference's Flow class (flow.py): compute_flow (flow.py:84-126, optical_flow_homography.py) reads color_flow/frame_%06d.png
and writes flow/flow_%06d_%06d.raw; compute_flow_masks, compute_flow_pair_stats and visualize_flow (flow.py:44-74, :128-209), which
process.py runs after it, read flow/flow_%06d_%06d.raw and color_down/frame_%06d.raw and write flow_mask/mask_%06d_%06d.png (8-bit,
0 / 255) and flow_list.json, the files the constraint builder, static flags, tracks and filters read; with --vis_flow they also write
vis_flow/frame_%06d_%06d.png and vis_flow_warped/frame_%06d_%06d_warped.png.  The per-pixel work is rcvd_homography_warp,
rcvd_flow_unregister, rcvd_flow_masks and rcvd_flow_visualize (include/rcvd.h); the files are read with numpy, and the outputs are
written on a thread pool while the next pairs compute.  The optical-flow model (RAFT) and the feature detector (SURF) are the caller's.

There is no CPU fallback: without librcvd_b200.so or a usable CUDA device these functions raise RuntimeError.
"""
import json
import os
import re
import struct
import sys
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import solver
from .png import png_gray_bytes, png_header, png_rgb_bytes, write_png  # noqa: F401  (png_*_bytes: part of this module's interface)
from .synthetic_files import read_raw, write_raw

FLOW_FMT = os.path.join("flow", "flow_{:06d}_{:06d}.raw")
MASK_FMT = os.path.join("flow_mask", "mask_{:06d}_{:06d}.png")
COLOR_FMT = os.path.join("color_down", "frame_{:06d}.raw")
VIS_FMT = os.path.join("vis_flow", "frame_{:06d}_{:06d}.png")
WARP_FMT = os.path.join("vis_flow_warped", "frame_{:06d}_{:06d}_warped.png")
FRAME_FMT = os.path.join("color_flow", "frame_{:06d}.png")
RAFT_MODEL_PATH = os.path.join("models", "raft-things.pth")
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


def _chunks(pairs, plane_bytes, chunk_bytes, pair_bytes=16):
    """Consecutive groups of pairs whose per-pair arrays (pair_bytes per pixel: both flows, and whatever else a pair reads or writes)
    and colours take at most chunk_bytes of host memory (at least one pair each)."""
    out, cur, frames = [], [], set()
    for p in pairs:
        new = frames | set(p)
        if cur and (len(cur) + 1) * pair_bytes * plane_bytes + len(new) * 12 * plane_bytes > chunk_bytes:
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
                pending.append(writers.submit(write_png, os.path.join(path, MASK_FMT.format(i, j)), mij[n]))
                pending.append(writers.submit(write_png, os.path.join(path, MASK_FMT.format(j, i)), mji[n]))
        t = time.perf_counter()
        stats["png_s"] += sum(f.result() for f in pending)
        stats["wait_s"] += time.perf_counter() - t
    stats["total_s"] = time.perf_counter() - t0
    return stats


IDENTITY = np.array([1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0]).reshape(3, 3)


def cv_invert3(H):
    """cv::invert(H, DECOMP_LU) of a 3 x 3 double matrix, the map cv2.warpPerspective applies: its closed form (cofactors times 1 / det,
    det expanded along row 0, every product rounded); a zero det gives the zero matrix, as cv::invert leaves it."""
    m = np.asarray(H, np.float64).reshape(3, 3).tolist()
    (a, b, c), (d, e, f), (g, h, i) = m
    det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g)
    if det == 0:
        return np.zeros((3, 3))
    r = 1.0 / det
    return np.array([[(e * i - f * h) * r, (c * h - b * i) * r, (b * f - c * e) * r],
                     [(f * g - d * i) * r, (a * i - c * g) * r, (c * d - a * f) * r],
                     [(d * h - e * g) * r, (b * g - a * h) * r, (a * e - b * d) * r]])


def frame_features(img, detector):
    """detectAndDescribe: the keypoint positions float32 [n, 2] and the descriptors (None without keypoints) of detector.detectAndCompute."""
    kps, des = detector.detectAndCompute(img, None)
    return np.float32([kp.pt for kp in kps]), des


def homography(feat1, feat2, ratio=0.75, reproj_thresh=4.0):
    """getimage's H_BA, which maps frame 2 onto frame 1, from the frame_features of both frames: frame 2's descriptors matched to frame
    1's (BruteForce knnMatch, k = 2), the matches that pass Lowe's ratio test, and findHomography(RANSAC, reproj_thresh) of more than 4
    of them.  The identity when anything fails, as the reference's fallbacks give: no descriptors (knnMatch raises), at most 4 matches,
    findHomography raising or returning None, or a matrix np.linalg.inv refuses."""
    import cv2
    (kps1, des1), (kps2, des2) = feat1, feat2
    try:
        knn = cv2.DescriptorMatcher_create("BruteForce").knnMatch(des2, des1, 2)
        good = [(m[0].queryIdx, m[0].trainIdx) for m in knn if len(m) == 2 and m[0].distance < m[1].distance * ratio]
        if len(good) <= 4:
            return IDENTITY.copy()
        H, _ = cv2.findHomography(np.float32([kps2[q] for q, _ in good]), np.float32([kps1[t] for _, t in good]), cv2.RANSAC,
                                  reproj_thresh)
    except Exception:
        return IDENTITY.copy()
    if H is None:
        return IDENTITY.copy()
    try:
        np.linalg.inv(H)
    except np.linalg.LinAlgError:
        return IDENTITY.copy()
    return H


class _Args(dict):
    """The reference's argument record (a dict read by attribute, None when absent), which RAFT's constructor reads."""
    __getattr__ = dict.get


def _default_model(path_pairs, size, device):
    """The reference's RAFT, imported from the caller's path and built as optical_flow_homography.process builds it."""
    try:
        import torch
        from raft.core.raft import RAFT
        im1, im2, out = path_pairs
        args = _Args(model="raft", pretrained_weights=RAFT_MODEL_PATH, im1=im1, im2=im2, out=out, size=size, fp16=False, homography=True,
                     rgb_max=255.0, visualize=False)
        model = torch.nn.DataParallel(RAFT(args))
        model.load_state_dict(torch.load(args.pretrained_weights, map_location=device))
        model = model.module
        model.to(device)
        model.eval()
        return model
    except Exception as e:
        raise RuntimeError(f"the default flow model is the reference's RAFT (raft.core.raft, weights {RAFT_MODEL_PATH}), which could not be "
                           f"loaded ({type(e).__name__}: {e}); pass model= (a module called as model(img1, img2, iters=20, "
                           "test_mode=True))") from e


def _default_features():
    import cv2
    try:
        return cv2.xfeatures2d.SURF_create
    except AttributeError as e:
        raise RuntimeError("the default feature detector is SURF (cv2.xfeatures2d.SURF_create), which this cv2 lacks (it is in the "
                           "opencv-contrib build); pass features= (a callable returning a detector with detectAndCompute)") from e


def flow_pairs_to_compute(path, index_pairs):
    """The pairs (i, j) of index_pairs, first occurrence first, whose flow/flow_i_j.raw is missing: none when every file exists."""
    out, seen = [], set()
    for i, j in index_pairs:
        p = (int(i), int(j))
        if p not in seen and not os.path.isfile(os.path.join(path, FLOW_FMT.format(*p))):
            out.append(p)
        seen.add(p)
    return out


def _check_flow_inputs(path, pairs):
    """Every frame of the pairs is an 8-bit RGB PNG of color_flow/frame_000000.png's size, and color_down/frame_000000.raw exists: refused
    before anything is written.  Returns ((H, W) of the frames, (w, h) of color_down)."""
    frames = sorted({0} | {f for p in pairs for f in p})
    size = None
    for f in frames:
        fn = os.path.join(path, FRAME_FMT.format(f))
        if not os.path.isfile(fn):
            raise FileNotFoundError(f"{fn} is missing")
        hd = png_header(fn)
        if hd["bit_depth"] != 8 or hd["color_type"] != 2 or hd["interlace"]:
            raise ValueError(f"{fn}: a {hd['bit_depth']}-bit PNG of colour type {hd['color_type']} (interlace {hd['interlace']}); the frames "
                             "must be 8-bit RGB, not interlaced")
        size = size or (hd["height"], hd["width"])
        if (hd["height"], hd["width"]) != size:
            raise ValueError(f"{fn}: {hd['width']} x {hd['height']} pixels, but frame 0 has {size[1]} x {size[0]}")
    down = os.path.join(path, COLOR_FMT.format(0))
    if not os.path.isfile(down):
        raise FileNotFoundError(f"{down} is missing: the flows are resized to the color_down frames' size")
    rows, cols, _ = _raw_shape(down)
    return size, (cols, rows)


def compute_flow(path, index_pairs, flow_model="raft", model=None, features=None, device=None, workers=None, batch=16):
    """Flow.compute_flow with the per-pixel work on the GPU: writes flow/flow_i_j.raw for every pair of index_pairs whose file is
    missing (nothing runs when all exist), as optical_flow_homography.process computes it: H_BA from the features of both color_flow
    frames, frame j registered by cv2.warpPerspective (rcvd_homography_warp), the model's flow_up[0] of (frame i, registered frame j),
    un-registered through np.linalg.inv(H_BA) and resized to color_down's size by resize_flow (rcvd_flow_unregister).

    model: the flow network, called once per pair as model(img1, img2, iters=20, test_mode=True) on float32 [1, 3, H, W] BGR tensors
    under no_grad; None builds the reference's RAFT from the caller's path.  features: a callable returning a detector with
    detectAndCompute (one per worker thread); None is cv2.xfeatures2d.SURF_create.  Each frame is decoded and its features computed once,
    on `workers` threads, which also match the pairs and write the files while the model runs.  A flow_model other than "raft" raises
    ValueError; a missing model or detector raises RuntimeError, and a missing or odd frame or a missing color_down/frame_000000.raw
    raises, all before anything is written.  Returns timings: {"pairs", "model_s", "kernel_s", "wait_s" (the caller's thread blocked on
    decoding, features and matching), "total_s"}."""
    import torch
    from .video import _decode_png   # video imports this module
    t0 = time.perf_counter()
    if flow_model != "raft":
        raise ValueError(f"flow model {flow_model!r}: only 'raft' is supported")
    pairs = flow_pairs_to_compute(path, index_pairs)
    stats = {"pairs": len(pairs), "model_s": 0.0, "kernel_s": 0.0, "wait_s": 0.0, "total_s": 0.0}
    if not pairs:
        os.makedirs(os.path.join(path, "flow"), exist_ok=True)
        stats["total_s"] = time.perf_counter() - t0
        return stats
    factory = features or _default_features()
    (H, W), size = _check_flow_inputs(path, pairs)
    tdev = torch.device("cuda") if device is None else torch.device("cuda", int(device))
    if model is None:
        model = _default_model(([os.path.join(path, FRAME_FMT.format(i)) for i, _ in pairs],
                                [os.path.join(path, FRAME_FMT.format(j)) for _, j in pairs],
                                [os.path.join(path, FLOW_FMT.format(i, j)) for i, j in pairs]), size, tdev)
    dev = solver.lib().rcvd_current_device() if device is None else int(device)
    if dev < 0:
        raise RuntimeError("rcvd error 5: no usable CUDA device for the flows; this library has no CPU fallback")
    os.makedirs(os.path.join(path, "flow"), exist_ok=True)
    print("Resizing flow to", size)
    local = threading.local()

    def load(f):
        img = _decode_png(os.path.join(path, FRAME_FMT.format(f)))
        if not hasattr(local, "detector"):
            local.detector = factory()
        return img, frame_features(img, local.detector)

    workers = workers or min(8, os.cpu_count() or 1)
    with ThreadPoolExecutor(workers) as pool:
        frames = {f: pool.submit(load, f) for f in sorted({f for p in pairs for f in p})}
        # every frame's job is queued before any pair's, so a pair's job never waits on a job queued behind it
        hs = [pool.submit(lambda i, j: homography(frames[i].result()[1], frames[j].result()[1]), i, j) for i, j in pairs]
        pending = []
        for b0 in range(0, len(pairs), batch):
            chunk = pairs[b0:b0 + batch]
            t = time.perf_counter()
            H_BA = [h.result() for h in hs[b0:b0 + batch]]
            js = sorted({j for _, j in chunk})
            src = np.stack([frames[j].result()[0] for j in js])
            stats["wait_s"] += time.perf_counter() - t
            t = time.perf_counter()
            reg = solver.homography_warp(src, [js.index(j) for _, j in chunk], [cv_invert3(h) for h in H_BA], device=dev)
            stats["kernel_s"] += time.perf_counter() - t
            t = time.perf_counter()
            flows = []
            with torch.no_grad():
                for n, (i, _) in enumerate(chunk):
                    img1 = torch.from_numpy(frames[i].result()[0]).to(tdev).permute(2, 0, 1).contiguous().float()[None]
                    img2 = torch.from_numpy(reg[n]).to(tdev).permute(2, 0, 1).contiguous().float()[None]
                    _, flow_up = model(img1, img2, iters=20, test_mode=True)
                    flows.append(flow_up[0].permute(1, 2, 0).cpu().numpy())
            stats["model_s"] += time.perf_counter() - t
            t = time.perf_counter()
            out = solver.flow_unregister(np.stack(flows), [np.linalg.inv(h) for h in H_BA], size, device=dev)
            stats["kernel_s"] += time.perf_counter() - t
            pending += [pool.submit(write_raw, os.path.join(path, FLOW_FMT.format(i, j)), out[n]) for n, (i, j) in enumerate(chunk)]
        for f in pending:
            f.result()
    stats["total_s"] = time.perf_counter() - t0
    return stats


def _flow_name_pair(name):
    """The reference's get_indices for visualize_flow: the integers after the first '_' of the name without its extension, sorted.  A
    name that does not give exactly two integers is refused (the reference crashes on it part-way)."""
    parts = os.path.splitext(name)[0].split("_")[1:]
    try:
        idx = sorted(int(s) for s in parts)
    except ValueError:
        idx = []
    if len(idx) != 2:
        raise ValueError(f"flow/{name}: not a flow_<i>_<j> file name")
    return tuple(idx)


def vis_pairs_to_compute(path, warp=False):
    """The sorted pairs (i, j), i <= j, that visualize_flow writes: every entry of flow/ parsed as the reference does, a pair skipped when
    its vis_flow PNG exists and, with warp, its vis_flow_warped/frame_i_j_warped.png (sorted indices) too."""
    pairs = sorted({_flow_name_pair(n) for n in os.listdir(os.path.join(path, "flow"))})
    return [(i, j) for i, j in pairs if not (os.path.isfile(os.path.join(path, VIS_FMT.format(i, j))) and
                                             (not warp or os.path.isfile(os.path.join(path, WARP_FMT.format(i, j)))))]


def _png_size(fn):
    """(rows, cols) from a PNG's IHDR."""
    with open(fn, "rb") as f:
        head = f.read(24)
    if len(head) < 24 or head[:8] != b"\x89PNG\r\n\x1a\n" or head[12:16] != b"IHDR":
        raise ValueError(f"{fn}: not a PNG file")
    w, h = struct.unpack(">II", head[16:24])
    return h, w


def _check_vis_inputs(path, pairs):
    """Both flows and masks and both colours of every pair exist and have one size of at least 2 x 2: refused before anything is
    written."""
    for i, j in pairs:
        shapes = {}
        for fn, size in ((FLOW_FMT.format(i, j), _raw_shape), (FLOW_FMT.format(j, i), _raw_shape), (MASK_FMT.format(i, j), _png_size),
                         (MASK_FMT.format(j, i), _png_size), (COLOR_FMT.format(i), _raw_shape), (COLOR_FMT.format(j), _raw_shape)):
            full = os.path.join(path, fn)
            if not os.path.isfile(full):
                raise FileNotFoundError(f"{full} is missing: the visualisation of pair ({i}, {j}) needs both flows, both masks and both colours")
            shapes[fn] = size(full)
        sizes = {s[:2] for s in shapes.values()}
        chans = [s[2] for s in shapes.values() if len(s) == 3]
        if len(sizes) != 1 or chans != [2, 2, 3, 3]:
            raise ValueError(f"pair ({i}, {j}): flows, masks and colours differ in size or channels: {shapes}")
        h, w = sizes.pop()
        if h < 2 or w < 2:
            raise ValueError(f"pair ({i}, {j}): images of {h} x {w} pixels; the warp's grid divides by width - 1 and height - 1")


def _read_vis_chunk(path, chunk, files):
    """_read_chunk plus both masks of every pair, decoded by the `files` pool."""
    colors, pf, fij, fji, rs = _read_chunk(path, chunk, files)
    t = time.perf_counter()
    masks = list(files.map(lambda k: _read_mask(os.path.join(path, MASK_FMT.format(*k))), [p for i, j in chunk for p in ((i, j), (j, i))]))
    mij, mji = np.stack(masks[0::2]), np.stack(masks[1::2])
    return colors, pf, fij, fji, mij, mji, rs + time.perf_counter() - t


def visualize_flow(path, warp=False, device=None, chunk_bytes=256 << 20, workers=None):
    """Flow.visualize_flow on the GPU: for every pair of vis_pairs_to_compute(path, warp) writes vis_flow/frame_i_j.png (the flow
    colours and masks composite) and, with warp, vis_flow_warped/frame_i_j_warped.png (colour j warped by flow i -> j) and
    frame_j_i_warped.png, both rewritten when the pair runs.  Both output directories are always created.  Pairs are processed in chunks
    of at most chunk_bytes of inputs and outputs; PNGs are encoded by `workers` threads while the next chunk reads and computes.  A name
    in flow/ that does not parse, a missing flow, mask or colour of a pair, or a size mismatch raises before anything is written.
    Returns timings as compute_flow_masks does."""
    t0 = time.perf_counter()
    L = solver.lib()
    dev = L.rcvd_current_device() if device is None else int(device)
    if dev < 0:
        raise RuntimeError("rcvd error 5: no usable CUDA device for the flow visualisation; this library has no CPU fallback")
    pairs = vis_pairs_to_compute(path, warp)
    _check_vis_inputs(path, pairs)
    for d in (VIS_FMT, WARP_FMT):
        os.makedirs(os.path.join(path, os.path.dirname(d)), exist_ok=True)
    stats = {"pairs": len(pairs), "read_s": 0.0, "compute_s": 0.0, "png_s": 0.0, "wait_s": 0.0, "total_s": 0.0}
    if not pairs:
        stats["total_s"] = time.perf_counter() - t0
        return stats
    rows, cols, _ = _raw_shape(os.path.join(path, COLOR_FMT.format(pairs[0][0])))
    # per pair and pixel: flows 16 B, masks 2 B, composite 24 B, warps 6 B
    chunks = _chunks(pairs, rows * cols, chunk_bytes, pair_bytes=48)
    workers = workers or min(8, os.cpu_count() or 1)
    with ThreadPoolExecutor(1) as reader, ThreadPoolExecutor(4) as files, ThreadPoolExecutor(workers) as writers:
        pending = []
        nxt = reader.submit(_read_vis_chunk, path, chunks[0], files)
        for k, chunk in enumerate(chunks):
            t = time.perf_counter()
            colors, pf, fij, fji, mij, mji, rs = nxt.result()
            stats["wait_s"] += time.perf_counter() - t
            stats["read_s"] += rs
            if k + 1 < len(chunks):
                nxt = reader.submit(_read_vis_chunk, path, chunks[k + 1], files)
            t = time.perf_counter()
            vis, wij, wji = solver.flow_visualize(colors, pf, fij, fji, mij, mji, warp=warp, device=dev)
            stats["compute_s"] += time.perf_counter() - t
            del colors, fij, fji, mij, mji
            t = time.perf_counter()
            stats["png_s"] += sum(f.result() for f in pending)   # at most one chunk of images waits for its PNGs
            stats["wait_s"] += time.perf_counter() - t
            pending = []
            for n, (i, j) in enumerate(chunk):
                pending.append(writers.submit(write_png, os.path.join(path, VIS_FMT.format(i, j)), vis[n]))
                if warp:
                    pending.append(writers.submit(write_png, os.path.join(path, WARP_FMT.format(i, j)), wij[n]))
                    pending.append(writers.submit(write_png, os.path.join(path, WARP_FMT.format(j, i)), wji[n]))
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
    """The reference's Flow class (flow.py) on the GPU: a caller of Flow(path, out_path).compute_flow(index_pairs, flow_model) /
    .compute_flow_masks() / .compute_flow_pair_stats(frame_pairs) / .visualize_flow(warp) switches by importing this class instead.
    compute_flow builds the reference's RAFT and SURF, as the reference does; compute_flow(path, ..., model=, features=) takes others."""

    def __init__(self, path, out_path):
        self.path = path
        self.out_path = out_path

    @staticmethod
    def max_size():
        return 1024

    def check_flow_files(self, index_pairs):
        return all(os.path.exists(os.path.join(self.path, FLOW_FMT.format(i, j))) for i, j in index_pairs)

    def compute_flow(self, index_pairs, flow_model):
        compute_flow(self.path, index_pairs, flow_model)

    def compute_flow_masks(self, flow_thresh=1, color_thresh=1):
        compute_flow_masks(self.path, flow_thresh, color_thresh)

    def compute_flow_pair_stats(self, frame_pairs):
        return compute_flow_pair_stats(self.path, frame_pairs)

    def visualize_flow(self, warp=False):
        visualize_flow(self.path, warp)
