"""Dynamic masks without a GPU: the numpy restatement tests/dynamic_mask_ref.py against the reference's own files in
tests/golden/dynamic_mask_golden.npz, the Python pipeline of robust_cvd_b200.dynamic_mask (input, output, message and skip rules) with
a fake predictor and the restatement standing in for the GPU call, and the refusals, raised before any device call."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from tests import dynamic_mask_ref as ref
from robust_cvd_b200 import abi, dynamic_mask as dm, solver
from robust_cvd_b200.png import png_gray_bytes, write_png
from robust_cvd_b200.video import _decode_png

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "dynamic_mask_golden.npz")


def golden_cases():
    g = np.load(GOLDEN)
    cases = sorted({k.split("/")[0] for k in g.files})
    out = {}
    for c in cases:
        names = list(g[f"{c}/names"])
        anno = bool(g[f"{c}/anno"])
        frames = [dict(name=n, img=g[f"{c}/in_{k}"], classes=g[f"{c}/classes_{k}"], masks=g[f"{c}/masks_{k}"], mask=g[f"{c}/mask_{k}"],
                       anon=g[f"{c}/anon_{k}"] if anno else None) for k, n in enumerate(names)]
        out[c] = dict(d=int(g[f"{c}/d"]), anno=anno, frames=frames, written=list(g[f"{c}/written"]))
    return out


class FakeInstances:
    def __init__(self, classes, masks):
        self.f = {"pred_classes": classes, "pred_masks": masks}

    def __len__(self):
        return len(self.f["pred_classes"])

    def get(self, k):
        return self.f[k]


class TablePredictor:
    """Returns the stored instances of each frame, found by its pixels."""
    def __init__(self, frames, convert=lambda a: a):
        self.table = {f["img"].tobytes(): (f["classes"], f["masks"]) for f in frames}
        self.convert = convert
        self.calls = 0

    def __call__(self, img):
        self.calls += 1
        classes, masks = self.table[np.ascontiguousarray(img).tobytes()]
        return {"instances": FakeInstances(self.convert(classes), self.convert(masks))}


def restated_dynamic_masks(instances, offsets, shape, dilation=5, frames=None, device=0):
    """solver.dynamic_masks restated in numpy (the instances are already the dynamic ones)."""
    masks, anon = [], []
    for f in range(len(offsets) - 1):
        u = ref.union(instances[offsets[f]:offsets[f + 1]], shape)
        masks.append(255 - ref.dilate(u, dilation))
        if frames is not None:
            a = frames[f][:, :, ::-1].copy()
            a[u != 0] = 255
            anon.append(a)
    return np.stack(masks), (np.stack(anon) if frames is not None else None)


@pytest.fixture
def no_gpu(monkeypatch):
    """The restatement stands in for the GPU call; calls are counted."""
    calls = []

    def fake(*a, **k):
        calls.append(len(a[1]) - 1)
        return restated_dynamic_masks(*a, **k)
    monkeypatch.setattr(solver, "dynamic_masks", fake)
    monkeypatch.setattr(dm, "_device", lambda device: 0)
    return calls


@pytest.fixture
def no_device_call(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a device call was made")
    monkeypatch.setattr(solver, "dynamic_masks", refuse)
    monkeypatch.setattr(dm, "_device", refuse)


def write_inputs(dirname, frames):
    os.makedirs(dirname, exist_ok=True)
    for f in frames:
        write_png(os.path.join(dirname, f["name"]), f["img"][:, :, ::-1])


def args_for(src, dst, d=5, anno=False, pattern="*.png", **kw):
    from types import SimpleNamespace
    a = SimpleNamespace(input=[os.path.join(src, pattern)], output=dst, dilation_factor=d, save_anno=anno, config_file="unused.yaml", opts=[],
                        confidence_threshold=0.5, webcam=False, video_input=None)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_restatement_equals_reference_golden():
    n = 0
    for c, case in golden_cases().items():
        for f in case["frames"]:
            mask, anon = ref.frame_outputs(f["img"], f["classes"], f["masks"], case["d"], case["anno"])
            np.testing.assert_array_equal(mask, f["mask"], err_msg=f"{c}/{f['name']}")
            rmask, ranon = ref.reference_frame(f["img"], f["classes"], f["masks"], case["d"], case["anno"])
            np.testing.assert_array_equal(rmask, f["mask"], err_msg=f"{c}/{f['name']}")
            if case["anno"]:
                np.testing.assert_array_equal(anon, f["anon"][:, :, ::-1], err_msg=f"{c}/{f['name']}")
                np.testing.assert_array_equal(ranon, f["anon"], err_msg=f"{c}/{f['name']}")
            n += 1
    assert n >= 30


def test_dilation_restatement_equals_cv2():
    import cv2
    rng = np.random.default_rng(5)
    for _ in range(300):
        h, w = (int(v) for v in rng.integers(1, 45, 2))
        d = int(rng.choice([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 60]))
        u = ((rng.random((h, w)) < rng.choice([0.005, 0.05, 0.4])) * 255).astype(np.uint8)
        np.testing.assert_array_equal(ref.dilate(u, d), cv2.dilate(u, np.ones((d, d), np.uint8), iterations=1), err_msg=f"{h}x{w} d={d}")


@pytest.mark.parametrize("chunk_bytes", [256 << 20, 1])
def test_pipeline_writes_the_golden_files(tmp_path, no_gpu, chunk_bytes):
    for c, case in golden_cases().items():
        src, dst = str(tmp_path / c / "in"), str(tmp_path / c / "out")
        write_inputs(src, case["frames"])
        stats = dm.dynamic_mask_generation(args_for(src, dst, case["d"], case["anno"]), predictor=TablePredictor(case["frames"]), workers=2,
                                           chunk_bytes=chunk_bytes)
        assert sorted(os.listdir(dst)) == case["written"], c
        assert stats["frames"] == len(case["frames"])
        for f in case["frames"]:
            base = os.path.join(dst, os.path.splitext(f["name"])[0])
            np.testing.assert_array_equal(_decode_png(base + ".png")[:, :, 0], f["mask"], err_msg=c)
            if case["anno"]:
                np.testing.assert_array_equal(_decode_png(base + "_anon.png"), f["anon"], err_msg=c)
    frames = sum(len(case["frames"]) for case in golden_cases().values())
    assert sum(no_gpu) == frames
    if chunk_bytes == 1:   # every frame is a call of its own, with or without dynamic instances
        assert len(no_gpu) == frames


@pytest.mark.parametrize("anno", [False, True])
def test_frames_without_instances_are_split_by_chunk_bytes(tmp_path, no_gpu, anno):
    """A static video (no dynamic instance anywhere) still goes to the GPU in chunks of at most chunk_bytes: each frame counts its
    union and mask, and with save_anno its frame and anonymised frame."""
    rng = np.random.default_rng(3)
    h, w = 12, 10
    frames = [dict(name=f"frame_{i:06d}.png", img=rng.integers(0, 256, (h, w, 3), dtype=np.uint8), classes=np.array([9, 40]),
                   masks=rng.random((2, h, w)) < 0.3) for i in range(7)]
    src, dst = str(tmp_path / "in"), str(tmp_path / "out")
    write_inputs(src, frames)
    per_frame = dm.call_bytes(np.zeros((0, h, w), bool), (h, w), anno)
    assert per_frame == h * w * (8 if anno else 2)
    dm.dynamic_mask_generation(args_for(src, dst, 3, anno), predictor=TablePredictor(frames), chunk_bytes=2 * per_frame)
    assert sorted(no_gpu) == [1, 2, 2, 2]
    assert len(os.listdir(dst)) == (14 if anno else 7)
    for f in frames:
        np.testing.assert_array_equal(_decode_png(os.path.join(dst, f["name"]))[:, :, 0], np.full((h, w), 255, np.uint8))


def test_messages_and_output_rules(tmp_path, no_gpu, capsys):
    case = golden_cases()["class_edges"]
    src = str(tmp_path / "in")
    write_inputs(src, case["frames"])
    dst = str(tmp_path / "a" / "b")   # missing directories are created
    dm.dynamic_mask_generation(args_for(src, dst), predictor=TablePredictor(case["frames"]))
    out = capsys.readouterr().out.splitlines()
    assert out[0] == f"dynamic frames input paths: {[os.path.join(src, '*.png')]}"
    assert sorted(out[1:]) == sorted(f"{os.path.join(src, f['name'])}: detected 7 instances in 0.00s" for f in case["frames"])
    assert sorted(os.listdir(dst)) == ["frame_000000.png", "frame_000001.png"]
    # an existing output file takes exactly one input, and names the prefix of the outputs
    target = str(tmp_path / "single.png")
    open(target, "wb").close()
    with pytest.raises(AssertionError, match="directory"):
        dm.dynamic_mask_generation(args_for(src, target), predictor=TablePredictor(case["frames"]))
    dm.dynamic_mask_generation(args_for(src, target, anno=True, pattern="frame_000001.png"), predictor=TablePredictor(case["frames"]))
    np.testing.assert_array_equal(_decode_png(target)[:, :, 0], case["frames"][1]["mask"])
    assert os.path.isfile(str(tmp_path / "single_anon.png"))
    with pytest.raises(AssertionError, match="not found"):
        dm.dynamic_mask_generation(args_for(src, dst, pattern="*.jpg"), predictor=TablePredictor(case["frames"]))


def test_torch_and_numpy_predictor_outputs_write_equal_files(tmp_path, no_gpu):
    torch = pytest.importorskip("torch")
    case = golden_cases()["overlap_border_d4"]
    src = str(tmp_path / "in")
    write_inputs(src, case["frames"])
    dm.dynamic_mask_generation(args_for(src, str(tmp_path / "np"), 4, True), predictor=TablePredictor(case["frames"]))
    dm.dynamic_mask_generation(args_for(src, str(tmp_path / "pt"), 4, True), predictor=TablePredictor(case["frames"], torch.as_tensor))
    for n in sorted(os.listdir(str(tmp_path / "np"))):
        assert open(str(tmp_path / "np" / n), "rb").read() == open(str(tmp_path / "pt" / n), "rb").read(), n


def _video_dir(tmp_path, frames):
    root = str(tmp_path / "video")
    write_inputs(os.path.join(root, "color_full"), frames)
    h, w = frames[0]["img"].shape[:2]
    with open(os.path.join(root, "frames.txt"), "w") as f:
        f.write(f"{len(frames)}\n{w}\n{h}\n" + "".join(f"{i / 30:.6f}\n" for i in range(len(frames))))
    return root


def test_compute_dynamic_mask_stage_and_skip_rule(tmp_path, no_gpu, capsys):
    case = golden_cases()["overlap_border_d5"]
    root = _video_dir(tmp_path, case["frames"])
    pred = TablePredictor(case["frames"])
    stats = dm.compute_dynamic_mask(root, dilation_factor=5, predictor=pred)
    assert stats["frames"] == 3 and pred.calls == 3
    for k, f in enumerate(case["frames"]):
        np.testing.assert_array_equal(_decode_png(os.path.join(root, "dynamic_mask", f["name"]))[:, :, 0], f["mask"])
    capsys.readouterr()
    assert dm.compute_dynamic_mask(root, predictor=pred) is None and pred.calls == 3
    assert "Dynamic masks exist, checked OK." in capsys.readouterr().out
    # a partial directory makes the check exit, as the reference's does
    os.remove(os.path.join(root, "dynamic_mask", "frame_000002.png"))
    with pytest.raises(SystemExit):
        dm.compute_dynamic_mask(root, predictor=pred)
    # --save_anno leaves 2N files, so the next run's check exits too, as the reference's does
    shutil.rmtree(os.path.join(root, "dynamic_mask"))
    assert dm.compute_dynamic_mask(root, save_anno=True, predictor=pred)["frames"] == 3
    assert len(os.listdir(os.path.join(root, "dynamic_mask"))) == 6
    calls = pred.calls
    with pytest.raises(SystemExit):
        dm.compute_dynamic_mask(root, save_anno=True, predictor=pred)
    assert pred.calls == calls
    os.remove(os.path.join(root, "frames.txt"))
    with pytest.raises(FileNotFoundError):
        dm.compute_dynamic_mask(root, predictor=pred)


def _bad_mask_predictor(case, which):
    def pred(img):
        f = next(f for f in case["frames"] if f["img"].tobytes() == np.ascontiguousarray(img).tobytes())
        masks = f["masks"].astype(np.uint8) if which == "u8" else f["masks"][:, :-1]
        return {"instances": FakeInstances(f["classes"], masks)}
    return pred


@pytest.mark.parametrize("which", ["u8", "shape"])
def test_bad_masks_refused_before_any_device_call(tmp_path, no_device_call, which):
    case = golden_cases()["class_edges"]
    src, dst = str(tmp_path / "in"), str(tmp_path / "out")
    write_inputs(src, case["frames"])
    with pytest.raises(ValueError, match="bool" if which == "u8" else "shape"):
        dm.dynamic_mask_generation(args_for(src, dst), predictor=_bad_mask_predictor(case, which))
    assert os.listdir(dst) == []


def test_argument_and_frame_refusals_before_anything_is_written(tmp_path, no_device_call):
    case = golden_cases()["class_edges"]
    src, dst = str(tmp_path / "in"), str(tmp_path / "out")
    write_inputs(src, case["frames"])
    pred = TablePredictor(case["frames"])
    with pytest.raises(ValueError, match="dilation_factor"):
        dm.dynamic_mask_generation(args_for(src, dst, d=-1), predictor=pred)
    for kw in ({"webcam": True}, {"video_input": "v.mp4"}, {"output": None}):
        with pytest.raises(ValueError):
            dm.dynamic_mask_generation(args_for(src, dst, **kw), predictor=pred)
    with open(os.path.join(src, "frame_000009.png"), "wb") as f:   # a gray frame
        f.write(png_gray_bytes(np.zeros((23, 31), np.uint8)))
    with pytest.raises(ValueError, match="8-bit RGB"):
        dm.dynamic_mask_generation(args_for(src, dst), predictor=pred)
    assert pred.calls == 0 and not os.path.exists(dst)


def test_default_predictor_failure_names_the_argument(tmp_path, no_device_call):
    case = golden_cases()["class_edges"]
    src, dst = str(tmp_path / "in"), str(tmp_path / "out")
    write_inputs(src, case["frames"])
    with pytest.raises(RuntimeError, match="predictor="):
        dm.dynamic_mask_generation(args_for(src, dst))
    assert not os.path.exists(dst)


def test_c_entry_refusals():
    L = solver.lib()
    h, w = 4, 5
    off = np.array([0, 1, 1], np.int64)
    ins = np.zeros((1, h, w), np.uint8)
    fr = np.zeros((2, h, w, 3), np.uint8)
    masks = np.zeros((2, h, w), np.uint8)
    anon = np.zeros((2, h, w, 3), np.uint8)
    P = lambda a, t=C.c_uint8: a.ctypes.data_as(C.POINTER(t))   # noqa: E731

    def call(prm, off=off, frames=fr, an=None):
        return L.rcvd_dynamic_masks(prm if prm is None else C.byref(prm), C.c_int32(0), P(off, C.c_int64), P(ins), None if frames is None else P(frames),
                                    P(masks), None if an is None else P(an))
    ok = dict(width=w, height=h, num_frames=2, dilation=5)
    assert call(None) == abi.ERR_INVALID
    for bad in (dict(width=0), dict(height=-1), dict(width=65536, height=10923), dict(num_frames=-1), dict(dilation=-1)):
        assert call(abi.DynamicMaskParams(**{**ok, **bad})) == abi.ERR_INVALID, bad
    assert call(abi.DynamicMaskParams(**ok), off=np.array([0, 1, 0], np.int64)) == abi.ERR_INVALID
    assert call(abi.DynamicMaskParams(**ok), off=np.array([1, 1, 1], np.int64)) == abi.ERR_INVALID
    assert call(abi.DynamicMaskParams(**ok), frames=None, an=anon) == abi.ERR_INVALID
    assert call(abi.DynamicMaskParams(**{**ok, "num_frames": 0})) == abi.OK
