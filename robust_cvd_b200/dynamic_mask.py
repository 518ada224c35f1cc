"""Dynamic-object masks of a robust_cvd working directory, with the per-pixel work on the GPU.

Drop-in for the reference's dynamic_mask_generation (dynamic_mask_generation.py:107-182) and DatasetProcessor.compute_dynamic_mask
(process.py:147-165), the stage between the flows and fine-tuning that writes dynamic_mask/frame_%06d.png: 0 where an instance of a
dynamic COCO class (people, vehicles, animals) lies, dilated by d x d, and 255 elsewhere.  setStaticFlagFromDynamicMask, the constraint
builder, computeTracks, pruneStaticFlag and the adaptive smoothness read those files.

The instance-segmentation model stays the caller's (by default the reference's Mask R-CNN through detectron2).  Around it, frames are
decoded ahead by the project's PNG decoder on a thread pool, the model runs on the calling thread, the class ids are selected on the
host and only the dynamic instances' masks are copied, and one rcvd_dynamic_masks call (include/rcvd.h) per chunk of frames (at
most chunk_bytes of inputs, outputs and device buffers) forms the union, the cv2.dilate-equal dilation, the inversion and the
--save_anno image.  The PNGs are encoded on another thread pool.  The
reference also draws a detectron2 Visualizer image for every frame and discards it; that is not done here.

The predictor is called as predictor(frame) with the frame [h, w, 3] u8 in B, G, R order, and returns {"instances": obj}; obj supports
len() and obj.get("pred_classes") ([K] class ids) and obj.get("pred_masks") ([K, h, w] bool), as torch tensors on any device or numpy
arrays.

Deviations: frames the project's decoder cannot read as ffmpeg writes them (not 8-bit RGB, interlaced, or with an eXIf chunk) are
refused before anything is written, as are a negative dilation_factor and, while predicting, masks that are not bool (on a uint8 mask
the reference's indexing writes whole rows) or whose shape is not the frame's.  --webcam, --video_input and a missing --output (the
reference opens windows and writes visualisation videos there) are refused with ValueError.  No tqdm progress bar is drawn.

There is no CPU fallback: without librcvd_b200.so or a usable CUDA device both functions raise RuntimeError.
"""
import glob
import os
import os.path as osp
import time
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import numpy as np

from . import solver
from .png import png_header, write_png
from .video import Video, _decode_png, check_frame_header

# the reference's dynamic class ids (MSCOCO person, vehicles and animals)
DYNAMIC_OBJECT_CATEGORIES = list(range(0, 8)) + list(range(13, 23))
DEFAULT_MASK_RCNN_MODEL_PATH = "models/mask_rcnn_R_50_FPN_3x.pkl"
DEFAULT_MASK_RCNN_CONFIG_PATH = "configs/mask_rcnn_R_50_FPN_3x.yaml"


def default_predictor(args):
    """The reference's predictor: its setup_cfg(args) (imported from the caller's path, where process.py runs) with MODEL.WEIGHTS =
    models/mask_rcnn_R_50_FPN_3x.pkl, frozen, in detectron2's DefaultPredictor."""
    try:
        from dynamic_mask_generation import setup_cfg
        from detectron2.engine import DefaultPredictor
        cfg = setup_cfg(args)
        cfg.merge_from_list(["MODEL.WEIGHTS", DEFAULT_MASK_RCNN_MODEL_PATH])
        cfg.freeze()
        return DefaultPredictor(cfg)
    except Exception as e:
        raise RuntimeError("the default predictor is the reference's Mask R-CNN (dynamic_mask_generation.setup_cfg and detectron2's "
                           f"DefaultPredictor with {DEFAULT_MASK_RCNN_MODEL_PATH}), which could not be built ({e!r}); pass predictor=") from e


def _numpy(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def dynamic_instances(instances, shape, path):
    """The masks [n, h, w] bool of the instances whose class is dynamic, copied from the predictor's output; only those are copied.
    Refuses masks that are not bool or not [len(instances), h, w] with shape = (h, w)."""
    classes = _numpy(instances.get("pred_classes")).reshape(-1)
    masks = instances.get("pred_masks")
    dtype = str(masks.dtype)
    if dtype not in ("bool", "torch.bool"):
        raise ValueError(f"{path}: pred_masks of type {dtype}; the masks must be bool (the reference's indexing writes whole rows for "
                         "integer masks)")
    if tuple(masks.shape) != (len(classes),) + tuple(shape):
        raise ValueError(f"{path}: pred_masks of shape {tuple(masks.shape)} for {len(classes)} classes and a {shape[1]} x {shape[0]} "
                         "frame")
    sel = np.flatnonzero(np.isin(classes, DYNAMIC_OBJECT_CATEGORIES))
    if hasattr(masks, "detach"):
        import torch
        return masks[torch.as_tensor(sel, dtype=torch.long, device=masks.device)].cpu().numpy()
    return np.asarray(masks)[sel]


def call_bytes(instances, shape, save_anno):
    """The bytes one frame adds to a rcvd_dynamic_masks call, on the host and on the device alike: its dynamic instances, the union and
    the mask, and with save_anno the frame and the anonymised frame."""
    return instances.nbytes + shape[0] * shape[1] * (2 + (6 if save_anno else 0))


def _device(device):
    dev = solver.lib().rcvd_current_device() if device is None else int(device)
    if dev < 0:
        raise RuntimeError("rcvd error 5: no usable CUDA device for the dynamic masks; this library has no CPU fallback")
    return dev


def _decode(path):
    t = time.perf_counter()
    img = _decode_png(path)
    return img, time.perf_counter() - t


def dynamic_mask_generation(args, predictor=None, device=None, workers=None, chunk_bytes=256 << 20):
    """The reference's dynamic_mask_generation(args) for --input: every file of glob.glob(expanduser(args.input[0])) (an empty match
    raises AssertionError), in that order, gets <output>/<base>.png = cv2.bitwise_not(cv2.dilate(union of its dynamic instances,
    np.ones((args.dilation_factor,) * 2))), and with args.save_anno also <output>/<base>_anon.png, the frame with the undilated union
    set to white.  An existing output file takes exactly one input and names the outputs' prefix; a missing output directory is
    created.  Prints "{path}: detected {n} instances in {t:.2f}s" per frame (n counts every instance).  Reads args.input, output,
    dilation_factor, save_anno, webcam and video_input, and config_file, opts and confidence_threshold for the default predictor.
    One GPU call handles a chunk of consecutive frames of one size that together need at most chunk_bytes (call_bytes: instances,
    union and mask, and with save_anno frame and anonymised frame), or a single frame that needs more; a chunk's files are written
    while the predictor works on the next chunk.  Returns timings: {"frames", "instances" (dynamic instances passed to the GPU), "decode_s", "predict_s", "kernel_s", "write_s" (decode and
    write summed over threads), "wait_s" (the calling thread blocked on decodes and writes), "total_s"}."""
    t0 = time.perf_counter()
    if getattr(args, "webcam", False) or getattr(args, "video_input", None):
        raise ValueError("--webcam and --video_input are not supported: they show windows and write visualisation videos")
    if not getattr(args, "input", None):
        raise ValueError("--input is needed: a glob pattern of the frames")
    if not getattr(args, "output", None):
        raise ValueError("--output is needed: without it the reference shows every frame in a window")
    d = int(args.dilation_factor)
    if d < 0:
        raise ValueError(f"dilation_factor {d}: must be >= 0 (0 dilates by 3 x 3, as OpenCV does)")
    print(f"dynamic frames input paths: {args.input}")
    paths = glob.glob(osp.expanduser(args.input[0]))
    if not paths:
        raise AssertionError("The input path(s) was not found")
    out = args.output
    to_file = osp.isfile(out)
    if to_file and len(paths) != 1:
        raise AssertionError("Please specify a *directory* with args.output")
    prefixes = [osp.splitext(out if to_file else osp.join(out, osp.basename(p)))[0] for p in paths]
    workers = workers or min(8, os.cpu_count() or 1)
    stats = {"frames": len(paths), "instances": 0, "decode_s": 0.0, "predict_s": 0.0, "kernel_s": 0.0, "write_s": 0.0, "wait_s": 0.0,
             "total_s": 0.0}
    with ThreadPoolExecutor(workers) as files, ThreadPoolExecutor(workers) as writers:
        for p in files.map(lambda p: (p, png_header(p)), paths):
            check_frame_header(*p)
        if predictor is None:
            predictor = default_predictor(args)
        if not to_file:
            os.makedirs(out, exist_ok=True)
        dev = None
        chunk, chunk_size, pending = [], 0, []

        def flush():
            nonlocal dev, pending
            if dev is None:
                dev = _device(device)
            shape = chunk[0][1]
            offsets = np.cumsum([0] + [len(s) for _, _, s, _ in chunk])
            instances = np.concatenate([s for _, _, s, _ in chunk]) if offsets[-1] else np.zeros((0,) + shape, np.uint8)
            frames = np.stack([img for _, _, _, img in chunk]) if args.save_anno else None
            t = time.perf_counter()
            masks, anon = solver.dynamic_masks(instances, offsets, shape, d, frames, device=dev)
            stats["kernel_s"] += time.perf_counter() - t
            stats["instances"] += int(offsets[-1])
            t = time.perf_counter()
            stats["write_s"] += sum(f.result() for f in pending)   # at most one chunk of outputs waits for its files
            stats["wait_s"] += time.perf_counter() - t
            pending = [writers.submit(write_png, prefixes[i] + ".png", masks[k]) for k, (i, _, _, _) in enumerate(chunk)]
            if anon is not None:
                pending += [writers.submit(write_png, prefixes[i] + "_anon.png", anon[k]) for k, (i, _, _, _) in enumerate(chunk)]
            chunk.clear()

        ahead = 2 * workers
        decoding = {i: files.submit(_decode, paths[i]) for i in range(min(ahead, len(paths)))}
        for i, path in enumerate(paths):
            t = time.perf_counter()
            img, ds = decoding.pop(i).result()
            stats["wait_s"] += time.perf_counter() - t
            stats["decode_s"] += ds
            if i + ahead < len(paths):
                decoding[i + ahead] = files.submit(_decode, paths[i + ahead])
            start = time.time()
            predictions = predictor(img)
            elapsed = time.time() - start
            stats["predict_s"] += elapsed
            instances = predictions["instances"]
            print("{}: detected {} instances in {:.2f}s".format(path, len(instances), elapsed))
            sel = dynamic_instances(instances, img.shape[:2], path)
            size = call_bytes(sel, img.shape[:2], args.save_anno)
            if chunk and (img.shape[:2] != chunk[0][1] or chunk_size + size > chunk_bytes):
                flush()
                chunk_size = 0
            chunk.append((i, img.shape[:2], sel, img if args.save_anno else None))
            chunk_size += size
        flush()
        t = time.perf_counter()
        stats["write_s"] += sum(f.result() for f in pending)
        stats["wait_s"] += time.perf_counter() - t
    stats["total_s"] = time.perf_counter() - t0
    return stats


def compute_dynamic_mask(path, dilation_factor=5, save_anno=False, confidence_threshold=0.5, config_file=DEFAULT_MASK_RCNN_CONFIG_PATH,
                         opts=(), predictor=None, device=None, workers=None, chunk_bytes=256 << 20):
    """DatasetProcessor.compute_dynamic_mask: dynamic_mask/ from color_full/*.png, skipped with "Dynamic masks exist, checked OK." (and
    None returned) when Video.check_frames(<path>/dynamic_mask, "png") passes for the frame count of frames.txt; like it, exits on a
    partial directory.  The keyword arguments are the reference's command-line options.  Returns dynamic_mask_generation's timings.
    Deviation: an error is raised; the reference logs it and goes on without masks.  A missing frames.txt raises FileNotFoundError."""
    video = Video(path)
    if not video.check_extracted_pts():
        raise FileNotFoundError(f"{osp.join(path, 'frames.txt')} is missing: the frame count comes from it")
    mask_dir = osp.join(path, "dynamic_mask")
    if video.check_frames(mask_dir, "png"):
        print("Dynamic masks exist, checked OK.")
        return None
    args = SimpleNamespace(input=[osp.join(path, "color_full") + "/*.png"], output=mask_dir, config_file=config_file, opts=list(opts),
                           confidence_threshold=confidence_threshold, dilation_factor=dilation_factor, save_anno=save_anno,
                           webcam=False, video_input=None)
    return dynamic_mask_generation(args, predictor=predictor, device=device, workers=workers, chunk_bytes=chunk_bytes)
