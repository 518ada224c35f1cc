"""Generates tests/golden/depth_vis_golden.npz, the depth-visualisation fixture, by running the reference's own
utils/visualization.visualize_depth_dir and visualize_depth (imported unchanged, nothing copied; they need cv2) on small seeded
directories.  Needs a checkout of facebookresearch/robust_cvd named by ROBUST_CVD_DIR, as the other golden generators in this directory
do.

  ROBUST_CVD_DIR=/path/to/robust_cvd python tests/golden/make_depth_vis_golden.py

Cases: NaN and +-inf pixels, a frame without a finite value, negative values and an all-negative directory, a constant directory,
percentiles 0 / 100, 2 / 98 and 37.5 / 62.5 (values outside the range wrap), odd and mixed frame sizes with an upper-case .RAW and a file
of another extension, the .png branch, and the evaluation's visualize_depth(d, 0, float32 max).

Stored: "lut" [256, 3] u8, the reference's colormaps.cm_magma (B, G, R); per directory "<dir>/ext" and "<dir>/names" (the file names,
sorted), "<dir>/in_<k>" the k-th file's array (float32 [h, w] or the B, G, R u8 image cv2.imread gives); per call "<dir>/<call>/args"
(min_percentile, max_percentile), "<dir>/<call>/d_min" and "/d_max" (float64) with "/bounds_type" their Python type names ("float"
where a bound is still Python's start value), "<dir>/<call>/vis_<k>" visualize_depth's float64 array and "<dir>/<call>/png_<k>" the
written PNG as cv2.imread decodes it (B, G, R u8); "eval/depth", "eval/vis" for visualize_depth(depth, 0, depth.max())."""
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("ROBUST_CVD_DIR", "")


def _disp(rng, h, w, lo=0.05, hi=2.0):
    return rng.uniform(lo, hi, (h, w)).astype(np.float32)


def cases():
    """{dir: (extension, [(file name, array)], [(call name, min_percentile, max_percentile)])}"""
    rng = np.random.default_rng(71)
    a = _disp(rng, 17, 23)
    a[0, 0], a[1, 1], a[2, 2], a[3, 3] = np.nan, np.inf, -np.inf, -0.0
    b = np.full((17, 23), np.nan, np.float32)
    b[::2, ::3] = np.inf
    c = _disp(rng, 17, 23, -1.0, 1.0)
    c[5, 5] = 0.0
    neg = [_disp(rng, 9, 11, -3.0, -0.5) for _ in range(2)]
    const = [np.full((8, 10), 0.5, np.float32) for _ in range(2)]
    mixed = [_disp(rng, 31, 17), _disp(rng, 9, 16, 0.0, 5.0), _disp(rng, 31, 17, 0.5, 1.0)]
    mixed[1][3, 4] = 1e10
    imgs = [rng.integers(0, 256, (13, 19, 3), dtype=np.uint8), rng.integers(40, 200, (13, 19, 3), dtype=np.uint8),
            rng.integers(0, 256, (7, 5, 3), dtype=np.uint8)]
    pct = [("p0_100", 0, 100), ("p2_98", 2, 98), ("p37_62", 37.5, 62.5)]
    return {
        "nonfinite": (".raw", [("frame_000000.raw", a), ("frame_000001.raw", b), ("frame_000002.raw", c)], pct),
        "negative": (".raw", [("frame_000000.raw", neg[0]), ("frame_000001.raw", neg[1])], pct[:2]),
        "constant": (".raw", [("frame_000000.raw", const[0]), ("frame_000001.raw", const[1])], pct[:1]),
        "mixed": (".raw", [("frame_000000.raw", mixed[0]), ("frame_000001.RAW", mixed[1]), ("frame_000002.raw", mixed[2])], pct),
        "png": (".png", [("img_a.png", imgs[0]), ("img_b.png", imgs[1]), ("img_c.png", imgs[2])], pct),
    }


def main():
    if not REF or not os.path.isfile(os.path.join(REF, "utils", "visualization.py")):
        sys.exit("set ROBUST_CVD_DIR to a checkout of facebookresearch/robust_cvd")
    sys.path.insert(0, REF)
    import cv2
    from utils import colormaps, image_io, visualization

    original = visualization.visualize_depth
    seen = []

    def recorder(depth, depth_min=None, depth_max=None):
        out = original(depth, depth_min, depth_max)
        seen.append((depth_min, depth_max, out))
        return out
    visualization.visualize_depth = recorder

    out = {"lut": np.ascontiguousarray(colormaps.cm_magma.reshape(256, 3))}
    tmp = tempfile.mkdtemp()
    try:
        for name, (ext, files, calls) in cases().items():
            src = os.path.join(tmp, name)
            os.makedirs(src)
            for fn, arr in files:
                if ext == ".raw":
                    image_io.save_raw_float32_image(os.path.join(src, fn), arr)
                else:
                    assert cv2.imwrite(os.path.join(src, fn), arr)
            with open(os.path.join(src, "notes.txt"), "w") as fh:
                fh.write("not a frame\n")
            names = sorted(fn for fn, _ in files)
            out[f"{name}/ext"] = np.array(ext)
            out[f"{name}/names"] = np.array(names)
            for k, fn in enumerate(names):
                out[f"{name}/in_{k}"] = (image_io.load_raw_float32_image(os.path.join(src, fn)) if ext == ".raw"
                                         else cv2.imread(os.path.join(src, fn)))
            for call, lo, hi in calls:
                dst = os.path.join(tmp, f"{name}_{call}")
                os.makedirs(dst)
                seen.clear()
                visualization.visualize_depth_dir(src, dst, force=True, extension=ext, min_percentile=lo, max_percentile=hi)
                assert len(seen) == len(names)
                d_min, d_max = seen[0][0], seen[0][1]
                out[f"{name}/{call}/args"] = np.array([lo, hi], np.float64)
                out[f"{name}/{call}/d_min"] = np.float64(d_min)
                out[f"{name}/{call}/d_max"] = np.float64(d_max)
                out[f"{name}/{call}/bounds_type"] = np.array([type(d_min).__name__, type(d_max).__name__])
                for k, fn in enumerate(names):
                    out[f"{name}/{call}/vis_{k}"] = seen[k][2]
                    out[f"{name}/{call}/png_{k}"] = cv2.imread(os.path.join(dst, os.path.splitext(fn)[0] + ".png"))
        rng = np.random.default_rng(72)
        depth = _disp(rng, 12, 14)
        out["eval/depth"] = depth
        out["eval/vis"] = original(depth, depth_min=0, depth_max=depth.max())
    finally:
        shutil.rmtree(tmp)
        visualization.visualize_depth = original
    out["numpy_version"] = np.array(np.__version__)
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(os.path.join(HERE, "depth_vis_golden.npz"), **out)
    print(f"wrote {len(out)} arrays to {os.path.join(HERE, 'depth_vis_golden.npz')}")


if __name__ == "__main__":
    main()
