"""Generates tests/golden/downscale_golden.npz, the frame-downscaling fixture, by running the reference's own video.Video(path)
.downscale_frames(...) and utils/image_io.resize_to_target (imported unchanged, nothing copied; they need cv2, Pillow and six) on small
seeded working directories.  Needs a checkout of facebookresearch/robust_cvd named by ROBUST_CVD_DIR, as the other golden generators in
this directory do.

  ROBUST_CVD_DIR=/path/to/robust_cvd python tests/golden/make_downscale_golden.py

Every directory holds FRAMES seeded 8-bit RGB frames of an odd-sized (or, for a factor of 2, one even side), non-square size.  The calls
cover each INTER_AREA path: integer factors 5 / 3 / 2 with equal and unequal x and y factors, area tables, upscaling on both axes and on
one (mixed), a half-to-even tie of the align rounding, short_side_target, a color_flow-like call with a small max_size and align 16 in
place of 1024 / 64, and the three calls of process.py's DatasetProcessor.downscale_frames at their defaults.

Stored: "<dir>/frames" [F, H, W, 3] u8 (R, G, B, the PNG's channels); per call "<dir>/<subdir>/args" (max_size, align,
short_side_target), "<dir>/<subdir>/ext", and "<dir>/<subdir>" the output: the .raw files' float32 arrays (B, G, R) or the PNGs as
cv2.imread decodes them (B, G, R u8); "target_cases" [n, 5] (H, W, max_size, align, short_side_target) with "target_sizes" [n, 2] the
(height, width) resize_to_target produced, -1 where cv2.resize refused the size."""
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("ROBUST_CVD_DIR", "")
FRAMES = 2
FLOW_MAX_SIZE = 1024   # the reference's Flow.max_size(); flow.py itself imports RAFT

# directory: (W, H, seed, [(subdir, max_size, ext, align, short_side_target)])
DOWNSCALE_CASES = {
    "75x45": (75, 45, 51, [("int5", 15, "raw", 1, False), ("int3", 25, "png", 1, False), ("area", 19, "raw", 1, False)]),
    "21x35": (21, 35, 52, [("int3x5", 7, "raw", 7, False)]),
    "45x18": (45, 18, 53, [("int5x2", 13, "raw", 9, False), ("int5x2_png", 13, "png", 9, False)]),
    "97x61": (97, 61, 54, [("area", 40, "raw", 1, False), ("area_png", 40, "png", 1, False), ("short", 20, "raw", 1, True),
                           ("flow", 48, "png", 16, False)]),
    "37x21": (37, 21, 55, [("up", 64, "raw", 8, False), ("up_png", 64, "png", 8, False)]),
    "41x23": (41, 23, 56, [("mixed", 64, "raw", 8, False)]),
    "45x20": (45, 20, 57, [("tie", 64, "raw", 8, False)]),
    "45x33": (45, 33, 58, [("color_down", 384, "raw", 32, False), ("color_down_png", 384, "png", 32, False),
                           ("color_flow", FLOW_MAX_SIZE, "png", 64, False)]),
}


def frames_of(name):
    """The seeded frames of a directory, [FRAMES, H, W, 3] u8 in R, G, B order: smooth gradients plus noise, with 0 and 255 present."""
    W, H, seed, _ = DOWNSCALE_CASES[name]
    rng = np.random.default_rng(seed)
    iy, ix = np.mgrid[0:H, 0:W]
    out = []
    for _ in range(FRAMES):
        base = np.stack([ix * 255.0 / W, iy * 255.0 / H, (ix + iy) * 127.0 / (W + H)], axis=-1)
        f = np.clip(base + rng.normal(0, 40, (H, W, 3)), 0, 255).astype(np.uint8)
        f[0, 0], f[-1, -1] = 0, 255
        out.append(f)
    return np.stack(out)


def target_cases():
    """(H, W, max_size, align, short_side_target) rows: the production frame sizes at process.py's settings, the issue's half-even ties
    (a side of 208 or 216 at align 32), sides that round to 0, and seeded small sizes."""
    rows = []
    for H, W in ((1080, 1920), (720, 1280), (480, 853), (360, 640), (2160, 3840), (1920, 1080), (1040, 1920), (1080, 1080)):
        for ms, al, sst in ((384, 32, 0), (384, 32, 1), (FLOW_MAX_SIZE, 64, 0), (384, 1, 0)):
            rows.append((H, W, ms, al, sst))
    rows += [(208, 300, 384, 32, 0), (216, 300, 384, 32, 0), (300, 208, 384, 32, 0), (10, 40, 384, 32, 0), (5, 200, 20, 1, 0)]
    rng = np.random.default_rng(59)
    for _ in range(200):
        rows.append((int(rng.integers(1, 400)), int(rng.integers(1, 400)), int(rng.integers(1, 500)), int(rng.integers(1, 70)),
                     int(rng.integers(0, 2))))
    return np.array(rows, np.int64)


def main():
    if not REF or not os.path.isfile(os.path.join(REF, "video.py")):
        sys.exit("set ROBUST_CVD_DIR to a checkout of facebookresearch/robust_cvd")
    sys.path.insert(0, REF)
    import cv2
    import video
    from utils import image_io

    out = {}
    tmp = tempfile.mkdtemp()
    try:
        for name, (W, H, _, calls) in DOWNSCALE_CASES.items():
            root = os.path.join(tmp, name)
            os.makedirs(os.path.join(root, "color_full"))
            frames = frames_of(name)
            for i, f in enumerate(frames):
                assert cv2.imwrite(os.path.join(root, "color_full", f"frame_{i:06d}.png"), f[..., ::-1])
            with open(os.path.join(root, "frames.txt"), "w") as fh:
                fh.write(f"{FRAMES}\n{W}\n{H}\n" + "".join(f"{i / 30.0:.6f}\n" for i in range(FRAMES)))
            out[f"{name}/frames"] = frames
            v = video.Video(root)
            assert v.check_extracted_pts()
            for subdir, ms, ext, al, sst in calls:
                v.downscale_frames(subdir, ms, ext, align=al, short_side_target=sst)
                files = [os.path.join(root, subdir, f"frame_{i:06d}.{ext}") for i in range(FRAMES)]
                imgs = [image_io.load_raw_float32_image(fn) if ext == "raw" else cv2.imread(fn, cv2.IMREAD_UNCHANGED) for fn in files]
                out[f"{name}/{subdir}"] = np.stack(imgs)
                out[f"{name}/{subdir}/args"] = np.array([ms, al, int(sst)], np.int64)
                out[f"{name}/{subdir}/ext"] = np.array(ext)
        rows = target_cases()
        sizes = []
        for H, W, ms, al, sst in rows:
            try:
                img = image_io.resize_to_target(np.zeros((H, W), np.uint8), int(ms), align=int(al), suppress_messages=True,
                                                short_side_target=bool(sst))
                sizes.append(img.shape[:2])
            except cv2.error:
                sizes.append((-1, -1))
        out["target_cases"] = rows
        out["target_sizes"] = np.array(sizes, np.int64)
    finally:
        shutil.rmtree(tmp)
    out["numpy_version"] = np.array(np.__version__)
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(os.path.join(HERE, "downscale_golden.npz"), **out)
    print(f"wrote {len(out)} arrays to {os.path.join(HERE, 'downscale_golden.npz')}")


if __name__ == "__main__":
    main()
