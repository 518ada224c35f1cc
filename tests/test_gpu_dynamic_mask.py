"""Dynamic masks on the GPU: rcvd_dynamic_masks against the numpy restatement tests/dynamic_mask_ref.py bit for bit (seeded cases up
to 1920 x 1080 and d = 2500 (reaches across many 64-row column segments, and past the image), planes with and without 16-byte vectors, more than 2^31 bytes of instances in one call),
dynamic_mask_generation against the reference's own files in tests/golden/dynamic_mask_golden.npz by decoded pixels, CUDA-tensor and
numpy predictor outputs, the check_frames skip, and the written masks read back through lib_python as the dynamic_mask stream by
setStaticFlagFromDynamicMask."""
import os
import sys

import numpy as np
import pytest

from tests import dynamic_mask_ref as ref
from tests.test_dynamic_mask import TablePredictor, args_for, golden_cases, write_inputs
from robust_cvd_b200 import dynamic_mask as dm, solver, synthetic, synthetic_files
from robust_cvd_b200.video import _decode_png

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CV_32FC3, CV_8UC1 = 21, 0


def _restated(instances, offsets, shape, d, frames):
    masks, anon = [], []
    for f in range(len(offsets) - 1):
        u = ref.union(instances[offsets[f]:offsets[f + 1]], shape)
        masks.append(255 - ref.dilate(u, d))
        if frames is not None:
            a = frames[f][:, :, ::-1].copy()
            a[u != 0] = 255
            anon.append(a)
    return np.stack(masks), (np.stack(anon) if frames is not None else None)


def _random_case(rng, F, h, w, kmax=4):
    counts = rng.integers(0, kmax + 1, F)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    ins = np.zeros((int(offsets[-1]), h, w), bool)
    for k in range(len(ins)):
        y0, x0 = rng.integers(0, h), rng.integers(0, w)
        ins[k, y0:y0 + rng.integers(1, h // 3 + 2), x0:x0 + rng.integers(1, w // 3 + 2)] = True
        ins[k] |= rng.random((h, w)) < rng.choice([0.0, 1e-4, 0.01])
        if k % 5 == 0:   # touching the borders
            ins[k, 0, rng.integers(0, w)] = ins[k, -1, rng.integers(0, w)] = ins[k, rng.integers(0, h), 0] = ins[k, rng.integers(0, h), -1] = True
    return ins, offsets, rng.integers(0, 256, (F, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("F,h,w,ds", [(5, 23, 31, (0, 1, 2, 3, 4, 5, 8, 40)), (3, 1, 17, (0, 2, 5)), (3, 19, 1, (3, 4, 30)),
                                      (4, 64, 48, (5, 6, 17, 101)), (3, 1080, 1920, (5, 8, 101, 300)),
                                      (2, 1081, 1919, (5, 64, 129, 2500)), (2, 700, 3, (0, 65, 128, 129, 1401))])
def test_entry_equals_restatement(F, h, w, ds):
    rng = np.random.default_rng(F * 1000 + h + w)
    ins, offsets, frames = _random_case(rng, F, h, w)
    for d in ds:
        l0 = solver.lib().rcvd_dynamic_mask_launch_count()
        masks, anon = solver.dynamic_masks(ins, offsets, (h, w), d, frames)
        assert solver.lib().rcvd_dynamic_mask_launch_count() > l0
        want_m, want_a = _restated(ins, offsets, (h, w), d, frames)
        np.testing.assert_array_equal(masks, want_m, err_msg=f"{h}x{w} d={d}")
        np.testing.assert_array_equal(anon, want_a, err_msg=f"{h}x{w} d={d}")
        masks2, none = solver.dynamic_masks(ins.astype(np.uint8) * 7, offsets, (h, w), d)
        assert none is None
        np.testing.assert_array_equal(masks2, want_m)


def test_instance_buffer_over_2gb_in_one_call():
    h, w = 1080, 1920
    total = (1 << 31) // (h * w) + 4          # > 2^31 bytes of instances
    F = 3
    offsets = np.array([0, 1, total - 2, total], np.int64)
    ins = np.zeros((total, h, w), np.uint8)
    ins[0, 5:9, 7:12] = 1
    ins[total - 1, h - 3:, w - 50:w - 40] = 1   # past byte 2^31 of the buffer
    ins[total - 2, 0, 0] = 1
    ins[total // 2, 500:510, 900:905] = 1      # frame 1
    masks, _ = solver.dynamic_masks(ins, offsets, (h, w), 7)
    for f in range(F):
        want = 255 - ref.dilate(ref.union(ins[offsets[f]:offsets[f + 1]], (h, w)), 7)
        np.testing.assert_array_equal(masks[f], want, err_msg=f"frame {f}")
    assert (masks[2] == 0).sum() > 0 and masks[2][h - 1, w - 45] == 0


def test_generation_equals_reference_golden(tmp_path):
    l0 = solver.lib().rcvd_dynamic_mask_launch_count()
    for c, case in golden_cases().items():
        src, dst = str(tmp_path / c / "in"), str(tmp_path / c / "out")
        write_inputs(src, case["frames"])
        dm.dynamic_mask_generation(args_for(src, dst, case["d"], case["anno"]), predictor=TablePredictor(case["frames"]))
        assert sorted(os.listdir(dst)) == case["written"], c
        for f in case["frames"]:
            base = os.path.join(dst, os.path.splitext(f["name"])[0])
            np.testing.assert_array_equal(_decode_png(base + ".png")[:, :, 0], f["mask"], err_msg=c)
            if case["anno"]:
                np.testing.assert_array_equal(_decode_png(base + "_anon.png"), f["anon"], err_msg=c)
    assert solver.lib().rcvd_dynamic_mask_launch_count() > l0


def test_cuda_tensor_and_numpy_predictors_write_equal_files(tmp_path):
    torch = pytest.importorskip("torch")
    case = golden_cases()["overlap_border_d8"]
    src = str(tmp_path / "in")
    write_inputs(src, case["frames"])
    dm.dynamic_mask_generation(args_for(src, str(tmp_path / "np"), 8, True), predictor=TablePredictor(case["frames"]))
    dm.dynamic_mask_generation(args_for(src, str(tmp_path / "cuda"), 8, True),
                               predictor=TablePredictor(case["frames"], lambda a: torch.as_tensor(a).cuda()))
    names = sorted(os.listdir(str(tmp_path / "np")))
    assert names == sorted(os.listdir(str(tmp_path / "cuda"))) and len(names) == 6
    for n in names:
        assert open(str(tmp_path / "np" / n), "rb").read() == open(str(tmp_path / "cuda" / n), "rb").read(), n


def _frames_for(scene, rng):
    """The scene's frames as color_full PNG inputs (B, G, R), and seeded instances per frame."""
    frames = []
    for i in range(scene.N):
        img = (synthetic_files.texture(scene, i) * 255).astype(np.uint8)
        ms = []
        for _ in range(2):
            m = np.zeros((scene.h, scene.w), bool)
            cy, cx = rng.integers(10, scene.h - 10), rng.integers(10, scene.w - 10)
            m[cy - 6:cy + 6, cx - 8:cx + 8] = True
            ms.append(m)
        frames.append(dict(name=f"frame_{i:06d}.png", img=img, classes=np.array([0, 9]), masks=np.stack(ms)))
    return frames


def test_masks_feed_lib_python_static_flags_and_skip(tmp_path, capsys):
    sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))
    import lib_python as lp
    sc = synthetic.Scene(6, 96, 64, seed=11, motion=0.04, rot_deg=0.5)
    frames = _frames_for(sc, np.random.default_rng(11))
    want = [ref.frame_outputs(f["img"], f["classes"], f["masks"], 5, False)[0] for f in frames]
    roots = {}
    for which in ("gpu", "restated"):
        root = str(tmp_path / which)
        synthetic_files.write_scene(sc, root, dynamic_masks=want if which == "restated" else None)
        roots[which] = root
    write_inputs(os.path.join(roots["gpu"], "color_full"), frames)
    pred = TablePredictor(frames)
    stats = dm.compute_dynamic_mask(roots["gpu"], dilation_factor=5, predictor=pred)
    assert stats["frames"] == 6 and stats["instances"] == 6 and pred.calls == 6
    capsys.readouterr()
    assert dm.compute_dynamic_mask(roots["gpu"], predictor=pred) is None and pred.calls == 6
    assert "Dynamic masks exist, checked OK." in capsys.readouterr().out

    def flags(root):
        v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
        v.createColorStream("down", "color_down", ".raw", CV_32FC3); v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
        v.createDepthStream("depth_midas2", "depth_midas2", [-1, -1])
        for i in range(sc.N):
            np.testing.assert_array_equal(v.colorStream("dynamic_mask").frame(i).image(), want[i])
        fp = lp.FlowConstraintsParams(); fp.frameRange.resolve(v.numFrames(), True); fp.doNotUseCache = True
        fc = lp.FlowConstraintsCollection(v, fp)
        fc.setStaticFlagFromDynamicMask(8)
        return {k: np.asarray(x[1]) for k, x in fc._pairs().items()}
    got, ref_flags = flags(roots["gpu"]), flags(roots["restated"])
    assert got.keys() == ref_flags.keys()
    n_dyn = 0
    for k in got:
        np.testing.assert_array_equal(got[k], ref_flags[k], err_msg=f"pair {k}")
        n_dyn += int((~got[k].astype(bool)).sum())
    assert n_dyn > 0
