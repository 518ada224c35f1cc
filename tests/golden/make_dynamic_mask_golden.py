"""Generates tests/golden/dynamic_mask_golden.npz, the dynamic-mask fixture, by running the reference's own
dynamic_mask_generation.dynamic_mask_generation (imported unchanged, nothing copied; it needs cv2, torch, tqdm and PIL) on small seeded
directories.  detectron2 and utils.predictor are stubbed in sys.modules: the configuration is inert, read_image decodes with PIL as
detectron2's does for these EXIF-free 8-bit RGB PNGs, and the predictor returns the seeded instances stored for each frame (torch
tensors: int64 classes, bool masks).  Needs a checkout of facebookresearch/robust_cvd named by ROBUST_CVD_DIR, as the other golden
generators in this directory do.

  ROBUST_CVD_DIR=/path/to/robust_cvd python tests/golden/make_dynamic_mask_golden.py

Cases: classes at the category edges (7, 8, 12, 13, 22, 23, 79); frames without instances and with only non-dynamic ones; overlapping
instances and instances touching every border under d = 0, 1, 2, 3, 4, 5, 8 and 45 (larger than the image); odd and mixed frame
sizes in one directory, down to one row and one column; --save_anno on and off.

Stored per case: "<case>/d", "<case>/anno", "<case>/names" (input file names, sorted), "<case>/written" (the names the reference wrote,
sorted); per input k: "<case>/in_<k>" the frame (B, G, R u8), "<case>/classes_<k>" [K] int64, "<case>/masks_<k>" [K, h, w] bool,
"<case>/mask_<k>" the written <base>.png as cv2.imread(IMREAD_UNCHANGED) decodes it, and with anno "<case>/anon_<k>" the written
<base>_anon.png as cv2.imread decodes it (B, G, R)."""
import hashlib
import os
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("ROBUST_CVD_DIR", "")


def _blob(rng, h, w):
    m = np.zeros((h, w), bool)
    y0, x0 = rng.integers(0, h), rng.integers(0, w)
    m[y0:y0 + rng.integers(1, max(2, h // 2)), x0:x0 + rng.integers(1, max(2, w // 2))] = True
    m |= rng.random((h, w)) < 0.01
    return m


def _border(h, w, side):
    m = np.zeros((h, w), bool)
    {"top": lambda: m.__setitem__((0, slice(w // 3, w // 3 + 2)), True),
     "bottom": lambda: m.__setitem__((h - 1, slice(0, 1)), True),
     "left": lambda: m.__setitem__((slice(h // 2, h // 2 + 1), 0), True),
     "right": lambda: m.__setitem__((slice(h - 2, h), w - 1), True)}[side]()
    return m


def _frame(rng, h, w, classes, masks):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8), np.asarray(classes, np.int64).reshape(-1), np.asarray(masks, bool).reshape((-1, h, w))


def cases():
    """{case: (d, save_anno, [(name, frame B, G, R, classes, masks)])}"""
    rng = np.random.default_rng(2024)
    out = {}
    edges = [7, 8, 12, 13, 22, 23, 79]
    out["class_edges"] = (5, True, [(f"frame_{i:06d}.png",) + _frame(rng, 23, 31, edges, [_blob(rng, 23, 31) for _ in edges]) for i in range(2)])
    out["no_dynamic"] = (5, True, [("frame_000000.png",) + _frame(rng, 17, 13, [], np.zeros((0, 17, 13), bool)),
                                   ("frame_000001.png",) + _frame(rng, 17, 13, [8, 12, 23, 50, 79], [_blob(rng, 17, 13) for _ in range(5)])])
    for d, anno in ((0, True), (1, False), (2, True), (3, False), (4, True), (5, True), (8, False), (45, True)):
        frames = []
        for i in range(3):
            h, w = 19, 27
            ms = [_blob(rng, h, w) for _ in range(3)]
            ms[1] = ms[0] | _blob(rng, h, w)   # overlaps the first
            ms += [_border(h, w, s) for s in ("top", "bottom", "left", "right")]
            cls = [0, 2, 16, 5, 14, 1, 20] if i != 1 else [0, 2, 9, 5, 30, 1, 20]
            frames.append((f"frame_{i:06d}.png",) + _frame(rng, h, w, cls, ms))
        out[f"overlap_border_d{d}"] = (d, anno, frames)
    mixed = []
    for i, (h, w) in enumerate(((11, 1), (1, 9), (25, 16), (2, 2))):
        ms = [_blob(rng, h, w) for _ in range(2)]
        mixed.append((f"img_{i}.png",) + _frame(rng, h, w, [3, 18], ms))
    out["mixed_sizes"] = (4, True, mixed)
    return out


def _stub_modules(lookup):
    import torch
    from PIL import Image

    class Node:
        def __getattr__(self, k):
            v = Node()
            object.__setattr__(self, k, v)
            return v

    class Cfg(Node):
        def merge_from_file(self, fn): pass
        def merge_from_list(self, items): pass
        def freeze(self): pass

    class Instances:
        def __init__(self, classes, masks):
            self.fields = {"pred_classes": torch.as_tensor(classes), "pred_masks": torch.as_tensor(masks)}
        def __len__(self): return len(self.fields["pred_classes"])
        def get(self, k): return self.fields[k]

    class VisualizationDemo:
        def __init__(self, cfg): pass
        def run_on_image(self, img):
            classes, masks = lookup[hashlib.sha1(np.ascontiguousarray(img).tobytes()).hexdigest()]
            return {"instances": Instances(classes, masks)}, None

    def read_image(path, format=None):
        assert format == "BGR"
        return np.asarray(Image.open(path).convert("RGB"))[:, :, ::-1]

    d2 = types.ModuleType("detectron2")
    mods = {"detectron2": d2, "detectron2.config": types.ModuleType("detectron2.config"),
            "detectron2.data": types.ModuleType("detectron2.data"),
            "detectron2.data.detection_utils": types.ModuleType("detectron2.data.detection_utils"),
            "utils.predictor": types.ModuleType("utils.predictor")}
    mods["detectron2.config"].get_cfg = Cfg
    mods["detectron2.data.detection_utils"].read_image = read_image
    mods["utils.predictor"].VisualizationDemo = VisualizationDemo
    sys.modules.update(mods)


def main():
    if not REF or not os.path.isfile(os.path.join(REF, "dynamic_mask_generation.py")):
        sys.exit("set ROBUST_CVD_DIR to a checkout of facebookresearch/robust_cvd")
    sys.path.insert(0, REF)
    sys.path.insert(0, ROOT)
    import cv2
    from robust_cvd_b200.png import write_png
    lookup = {}
    _stub_modules(lookup)
    import dynamic_mask_generation as dmg

    out = {}
    tmp = tempfile.mkdtemp()
    try:
        for case, (d, anno, frames) in cases().items():
            src, dst = os.path.join(tmp, case, "in"), os.path.join(tmp, case, "out")
            os.makedirs(src)
            names = sorted(f[0] for f in frames)
            for name, img, classes, masks in frames:
                write_png(os.path.join(src, name), img[:, :, ::-1])
                lookup[hashlib.sha1(np.ascontiguousarray(img).tobytes()).hexdigest()] = (classes, masks)
            args = types.SimpleNamespace(input=[src + "/*.png"], output=dst, config_file="unused.yaml", opts=[], confidence_threshold=0.5,
                                         dilation_factor=d, save_anno=anno, webcam=False, video_input=None)
            dmg.dynamic_mask_generation(args)
            out[f"{case}/d"], out[f"{case}/anno"] = np.int64(d), np.bool_(anno)
            out[f"{case}/names"] = np.array(names)
            out[f"{case}/written"] = np.array(sorted(os.listdir(dst)))
            by_name = {f[0]: f for f in frames}
            for k, name in enumerate(names):
                _, img, classes, masks = by_name[name]
                base = os.path.splitext(name)[0]
                out[f"{case}/in_{k}"], out[f"{case}/classes_{k}"], out[f"{case}/masks_{k}"] = img, classes, masks
                out[f"{case}/mask_{k}"] = cv2.imread(os.path.join(dst, base + ".png"), cv2.IMREAD_UNCHANGED)
                if anno:
                    out[f"{case}/anon_{k}"] = cv2.imread(os.path.join(dst, base + "_anon.png"), cv2.IMREAD_UNCHANGED)
    finally:
        shutil.rmtree(tmp)
    np.savez_compressed(os.path.join(HERE, "dynamic_mask_golden.npz"), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == "__main__":
    main()
