"""Downscaled colour frames of a robust_cvd working directory, with the resize on the GPU.

Drop-in for the reference's Video.downscale_frames (video.py:154-182) and DatasetProcessor.downscale_frames (process.py:99-113), the
stage after frame extraction: it reads color_full/frame_%06d.png (8-bit RGB, as ffmpeg's rgb24 writes them) and writes the streams every
later stage reads: color_down/frame_%06d.raw (float32 B, G, R, the "down" stream), color_down_png/frame_%06d.png and
color_flow/frame_%06d.png (RAFT's input).  Each frame is np.float32(img) / 255.0 resized by cv2.resize(INTER_AREA), bit for bit
(rcvd_resize_area, include/rcvd.h).  Frames are decoded once for every output directory, by the project's PNG decoder on a thread pool,
in chunks read while the previous chunk computes; the outputs are written by another thread pool.

Deviation: a frame carrying an eXIf chunk is refused.  The reference rotates such a frame by its orientation tag through Pillow;
ffmpeg never writes one.  Frames that are not 8-bit RGB are refused too: on gray, palette and RGBA frames the reference writes streams
lib_python cannot read (a mirrored gray image, 4-channel raws).

There is no CPU fallback: without librcvd_b200.so or a usable CUDA device downscale_all and Video.downscale_frames raise RuntimeError.
"""
import os
import os.path as osp
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import solver
from .flow import Flow
from .png import png_header, write_png
from .synthetic_files import write_raw

FRAME_FMT = "frame_{:06d}.{}"


def target_size(H, W, max_size, align=1, short_side_target=False):
    """(height, width) of a W x H frame after the reference's resize_to_target (utils/image_io.py:26-52), with its Python float
    operations: scale = min(1, max_size / float(max(W, H))) (min(W, H) with short_side_target), int(side * scale), and a side that is
    not a multiple of align becomes align * round(side / align) -- Python's round, half to even (208 at align 32 gives 192)."""
    target_side = float(min(W, H)) if short_side_target else float(max(W, H))
    scale = min(1.0, max_size / target_side)
    h, w = int(H * scale), int(W * scale)
    if w % align != 0:
        w = align * round(w / align)
    if h % align != 0:
        h = align * round(h / align)
    return h, w


def _decode_png(fn):
    """A frame as [h, w, 3] u8 in B, G, R order through the project's PNG decoder (lib_python._imreadPng, the cv::imread subset the C++
    readers use; it decodes without the GIL)."""
    host = osp.join(osp.dirname(osp.abspath(__file__)), "host")
    if host not in sys.path:
        sys.path.insert(0, host)
    import lib_python
    img = lib_python._imreadPng(fn, False)
    if img is None:
        raise ValueError(f"{fn}: could not be decoded")
    return img


def check_frame_header(fn, hd):
    """Refuses a frame whose png_header `hd` the project's decoder does not read as ffmpeg's frames: not 8-bit RGB (colour type 2),
    interlaced, or carrying an eXIf chunk."""
    if hd["bit_depth"] != 8 or hd["color_type"] != 2:
        raise ValueError(f"{fn}: a {hd['bit_depth']}-bit PNG of colour type {hd['color_type']}; the frames must be 8-bit RGB "
                         "(colour type 2), as ffmpeg's rgb24 writes them")
    if hd["interlace"]:
        raise ValueError(f"{fn}: an interlaced PNG; the frames must not be interlaced")
    if hd["exif"]:
        raise ValueError(f"{fn}: carries an eXIf chunk; a frame's EXIF orientation is not applied, so such frames are refused")


def _check_full_frames(full_dir, count, files):
    """(height, width) of the frames color_full/frame_%06d.png, 0 <= i < count, after checking each one's header on the `files` pool:
    present, 8-bit RGB (colour type 2), not interlaced, no eXIf chunk, frame 0's size."""
    def header(i):
        fn = osp.join(full_dir, FRAME_FMT.format(i, "png"))
        if not osp.isfile(fn):
            raise FileNotFoundError(f"{fn} is missing: expected {count} frames (frames.txt)")
        return fn, png_header(fn)
    heads = list(files.map(header, range(count)))
    size = (heads[0][1]["height"], heads[0][1]["width"])
    for fn, hd in heads:
        check_frame_header(fn, hd)
        if (hd["height"], hd["width"]) != size:
            raise ValueError(f"{fn}: {hd['width']} x {hd['height']} pixels, but frame 0 has {size[1]} x {size[0]}")
    return size


def _read_frames(full_dir, frames, shape, files):
    """Frames [len(frames), H, W, 3] u8 (B, G, R), decoded by the `files` pool."""
    t = time.perf_counter()
    out = np.empty((len(frames),) + shape + (3,), np.uint8)

    def one(k):
        out[k] = _decode_png(osp.join(full_dir, FRAME_FMT.format(frames[k], "png")))
    list(files.map(one, range(len(frames))))
    return out, time.perf_counter() - t


def _write_raw(fn, img):
    t = time.perf_counter()
    write_raw(fn, img)
    return time.perf_counter() - t


def _downscale(video, outputs, full_subdir="color_full", device=None, chunk_bytes=256 << 20, workers=None):
    """Writes every output (subdir, max_size, ext, align, short_side_target) of `video` that does not pass check_frames, decoding each
    frame once for all of them.  Every refusal happens before anything is written; each written directory is checked again after.
    Returns timings: {"frames", "outputs" (the subdirs written), "read_s", "compute_s", "write_s" (summed over threads), "wait_s" (the
    caller's thread blocked on reads and writes), "total_s"}."""
    t0 = time.perf_counter()
    if getattr(video, "frame_count", None) is None and not video.check_extracted_pts():
        raise FileNotFoundError(f"{osp.join(video.path, 'frames.txt')} is missing: the frame count comes from it")
    count = video.frame_count
    todo = [o for o in outputs if not video.check_frames(osp.join(video.path, o[0]), o[2])]
    stats = {"frames": count, "outputs": [o[0] for o in todo], "read_s": 0.0, "compute_s": 0.0, "write_s": 0.0, "wait_s": 0.0,
             "total_s": 0.0}
    if not todo or count == 0:
        for o in todo:
            os.makedirs(osp.join(video.path, o[0]), exist_ok=True)
        stats["total_s"] = time.perf_counter() - t0
        return stats
    full_dir = osp.join(video.path, full_subdir)
    workers = workers or min(8, os.cpu_count() or 1)
    with ThreadPoolExecutor(1) as reader, ThreadPoolExecutor(workers) as files, ThreadPoolExecutor(workers) as writers:
        H, W = _check_full_frames(full_dir, count, files)
        sizes = []
        for subdir, max_size, ext, align, short_side in todo:
            h, w = target_size(H, W, max_size, align, short_side)
            if h <= 0 or w <= 0:
                raise ValueError(f"{subdir}: a {W} x {H} frame at max_size {max_size}, align {align} gives {w} x {h} pixels")
            if ext not in ("raw", "png"):
                raise ValueError(f"{subdir}: extension {ext!r}; the frames are written as raw or png")
            sizes.append((h, w, ext))
        L = solver.lib()
        dev = L.rcvd_current_device() if device is None else int(device)
        if dev < 0:
            raise RuntimeError("rcvd error 5: no usable CUDA device for the frame downscaling; this library has no CPU fallback")
        print(f"Original size: {W} x {H}")
        for (subdir, *_), (h, w, _) in zip(todo, sizes):
            print(f"Resized: {w} x {h} ({subdir})")
            os.makedirs(osp.join(video.path, subdir), exist_ok=True)
        per_frame = H * W * 3 + sum(h * w * (12 if ext == "raw" else 3) for h, w, ext in sizes)
        step = max(1, chunk_bytes // per_frame)
        chunks = [list(range(s, min(s + step, count))) for s in range(0, count, step)]
        pending = []
        nxt = reader.submit(_read_frames, full_dir, chunks[0], (H, W), files)
        for k, chunk in enumerate(chunks):
            t = time.perf_counter()
            frames, rs = nxt.result()
            stats["wait_s"] += time.perf_counter() - t
            stats["read_s"] += rs
            if k + 1 < len(chunks):
                nxt = reader.submit(_read_frames, full_dir, chunks[k + 1], (H, W), files)
            t = time.perf_counter()
            outs = solver.resize_area(frames, sizes, device=dev)
            stats["compute_s"] += time.perf_counter() - t
            del frames
            t = time.perf_counter()
            stats["write_s"] += sum(f.result() for f in pending)   # at most one chunk of outputs waits for its files
            stats["wait_s"] += time.perf_counter() - t
            pending = []
            for (subdir, _, ext, _, _), out in zip(todo, outs):
                write = _write_raw if ext == "raw" else write_png
                for n, i in enumerate(chunk):
                    pending.append(writers.submit(write, osp.join(video.path, subdir, FRAME_FMT.format(i, ext)), out[n]))
        t = time.perf_counter()
        stats["write_s"] += sum(f.result() for f in pending)
        stats["wait_s"] += time.perf_counter() - t
    for subdir, _, ext, _, _ in todo:
        video.check_frames(osp.join(video.path, subdir), ext)
    stats["total_s"] = time.perf_counter() - t0
    return stats


class Video:
    """The reference's Video class (video.py) for the stages after extraction: check_extracted_pts, check_frames and downscale_frames,
    with the reference's signatures, messages and exits.  extract_pts and extract_frames (ffmpeg) are not provided."""

    def __init__(self, path, video_file=None):
        self.path = path
        self.video_file = video_file

    def check_extracted_pts(self):
        """Reads the frame count from frames.txt line 1; False when the file is missing, sys.exit when its line count is not
        count + 3."""
        pts_file = osp.join(self.path, "frames.txt")
        if not os.path.exists(pts_file):
            return False
        with open(pts_file, "r") as file:
            lines = file.readlines()
            self.frame_count = int(lines[0])
            width = int(lines[1])
            height = int(lines[2])
            print("%d frames detected (%d x %d)." % (self.frame_count, width, height))
            if len(lines) != self.frame_count + 3:
                sys.exit("frames.txt has wrong number of lines")
            print("frames.txt exists, checked OK.")
            return True

    def check_frames(self, frame_dir, extension, frames=None):
        """False when frame_dir holds no file ending in extension; sys.exit when the count of those files differs from the frame count
        or a frame_%06d.<extension> is missing; True otherwise."""
        if not os.path.isdir(frame_dir):
            return False
        files = [n for n in os.listdir(frame_dir) if n.endswith(extension)]
        if len(files) == 0:
            return False
        if frames is None:
            frames = range(self.frame_count)
        if len(files) != len(frames):
            sys.exit("ERROR: expected to find %d files but found %d in '%s'" % (self.frame_count, len(files), frame_dir))
        for i in frames:
            frame_file = "%s/frame_%06d.%s" % (frame_dir, i, extension)
            if not os.path.exists(frame_file):
                sys.exit("ERROR: did not find expected file '%s'" % frame_file)
        print("Frames found, checked OK.")
        return True

    def downscale_frames(self, subdir, max_size, ext, align=32, full_subdir="color_full", short_side_target=False):
        """Writes subdir/frame_%06d.<ext> (ext "raw" or "png") from full_subdir/frame_%06d.png resized to target_size(..., max_size,
        align, short_side_target), unless subdir already passes check_frames.  Returns timings as downscale_all does."""
        return _downscale(self, [(subdir, max_size, ext, align, short_side_target)], full_subdir)


def downscale_all(path, size=384, align=32, short_side_target=False, device=None, chunk_bytes=256 << 20, workers=None):
    """DatasetProcessor.downscale_frames: color_down (.raw) and color_down_png (.png) at (size, align, short_side_target), and
    color_flow (.png) at Flow.max_size() = 1024, align 64.  Each frame is decoded once for every output that does not pass
    check_frames.  Frames are processed in chunks of at most chunk_bytes of frames and outputs; `workers` threads decode and write.
    Returns timings: {"frames", "outputs", "read_s", "compute_s", "write_s", "wait_s", "total_s"}."""
    outputs = [("color_down", size, "raw", align, short_side_target), ("color_down_png", size, "png", align, short_side_target),
               ("color_flow", Flow.max_size(), "png", 64, False)]
    return _downscale(Video(path), outputs, device=device, chunk_bytes=chunk_bytes, workers=workers)
