"""Frame downscaling without a GPU: the float32 restatement tests/resize_ref.py against cv2.resize(INTER_AREA) bit for bit and against
the reference's own outputs (tests/golden/downscale_golden.npz, written by tests/golden/make_downscale_golden.py from the reference's
Video.downscale_frames), the size rule against the reference's resize_to_target, the reference's skip rule and exits, every refusal of
robust_cvd_b200.video (all before anything is written) and the refusals of rcvd_resize_area, which need no device."""
import ctypes as C
import os
import struct
import zlib

import numpy as np
import pytest

from tests import resize_ref as ref
from robust_cvd_b200 import abi, png, solver, video

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "downscale_golden.npz")
PRODUCTION = [((1920, 1080), (384, 224)), ((1920, 1080), (1024, 576)), ((1920, 1080), (384, 216)), ((1280, 720), (384, 224)),
              ((853, 480), (384, 224)), ((640, 360), (640, 384))]


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def golden_calls(g):
    """(directory, subdir, ext, max_size, align, short_side_target) of every call in the fixture."""
    for key in g.files:
        if key.endswith("/ext"):
            name, subdir = key.split("/")[:2]
            ms, al, sst = (int(v) for v in g[f"{name}/{subdir}/args"])
            yield name, subdir, str(g[key]), ms, al, bool(sst)


def sweep_cases():
    """Seeded (W, H, w, h): 98 -> 20, random sizes from 1 to 200 (downscale, upscale and mixed), integer factors 1 .. 6 per axis."""
    rng = np.random.default_rng(2024)
    cases = [(98, 10, 20, 31), (98, 98, 20, 20)]
    cases += [tuple(int(v) for v in rng.integers(1, 201, 4)) for _ in range(400)]
    cases += [(7 * ix, 5 * iy, 7, 5) for ix in range(1, 7) for iy in range(1, 7)]
    return cases


def test_restatement_is_cv2_resize_inter_area():
    import cv2
    rng = np.random.default_rng(5)
    paths = {}
    for W, H, w, h in sweep_cases():
        img = ref.to_float(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        want = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)
        assert bits_equal(ref.resize_area(img, w, h), want), (W, H, w, h)
        paths[ref.resize_path(W, H, w, h)] = paths.get(ref.resize_path(W, H, w, h), 0) + 1
    assert min(paths.get(p, 0) for p in ("integer", "area", "linear")) >= 30, paths


def test_restatement_is_cv2_at_production_shapes():
    import cv2
    rng = np.random.default_rng(6)
    for (W, H), (w, h) in PRODUCTION:
        img = ref.to_float(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        assert bits_equal(ref.resize_area(img, w, h), cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)), (W, H, w, h)


def test_scale_is_one_over_the_inverse():
    """1 / (w / W) and W / w differ in the last bit at 98 -> 20; where that axis takes the upscale path's taps (the other axis
    upscales), output 10 then reads source 48 instead of 49 and 50.  The sweep's (98, 10) -> (20, 31) checks the result against cv2."""
    assert ref.axis_scale(98, 20) != 98 / 20
    taps = ref.linear_taps(98, 20)
    assert [k for k, _ in taps[10]] == [48, 49]
    assert np.floor(10 * (98 / 20)) == 49


def test_to_float_and_png_conversion_match_numpy_and_cv2(tmp_path):
    import cv2
    u = np.arange(256, dtype=np.uint8)
    assert bits_equal(ref.to_float(u), np.float32(u) / 255.0)
    vals = np.array([0.5, 1.5, 2.5, 127.5, 254.5, 255.4, 255.6, 0.0, 1.0, -0.2], np.float32) / np.float32(255)
    img = np.repeat(vals[None, :, None], 3, axis=2)
    fn = str(tmp_path / "v.png")
    assert cv2.imwrite(fn, img * 255)
    np.testing.assert_array_equal(cv2.imread(fn, cv2.IMREAD_UNCHANGED), ref.to_png_u8(img))


def test_restatement_matches_reference_golden():
    """Every call of the fixture: the target size, then the .raw floats bit for bit and the decoded PNG pixels exactly."""
    g = np.load(GOLDEN)
    for name, subdir, ext, ms, al, sst in golden_calls(g):
        frames = g[f"{name}/frames"]
        H, W = frames.shape[1:3]
        h, w = video.target_size(H, W, ms, al, sst)
        want = g[f"{name}/{subdir}"]
        assert want.shape[1:3] == (h, w), (name, subdir)
        for f, out in zip(frames, want):
            got = ref.resize_area(ref.to_float(f[..., ::-1]), w, h)          # the reference swaps to B, G, R after the resize
            if ext == "raw":
                assert bits_equal(got, out), (name, subdir)
            else:
                np.testing.assert_array_equal(ref.to_png_u8(got), out, err_msg=f"{name}/{subdir}")


def test_golden_covers_every_path():
    g = np.load(GOLDEN)
    seen = set()
    for name, subdir, ext, ms, al, sst in golden_calls(g):
        H, W = g[f"{name}/frames"].shape[1:3]
        h, w = video.target_size(H, W, ms, al, sst)
        fast = ref.area_fast_factors(W, H, w, h)
        if fast:
            seen.add(("integer", fast))
        else:
            seen.add((ref.resize_path(W, H, w, h), "up" if w > W and h > H else "mixed" if w > W or h > H else "down"))
        seen.add(("ext", ext))
        if sst:
            seen.add("short_side_target")
        if al > 1 and (int(H * min(1.0, ms / max(W, H))) / al) % 1 == 0.5:
            seen.add("tie")
    factors = {s[1] for s in seen if s[0] == "integer"}
    assert {5, 3, 2} <= {f for fx in factors for f in fx} and any(fx != fy for fx, fy in factors)
    assert {("area", "down"), ("linear", "up"), ("linear", "mixed"), ("ext", "raw"), ("ext", "png"), "short_side_target", "tie"} <= seen


def test_target_size_matches_resize_to_target():
    g = np.load(GOLDEN)
    for (H, W, ms, al, sst), want in zip(g["target_cases"], g["target_sizes"]):
        h, w = video.target_size(int(H), int(W), int(ms), int(al), bool(sst))
        if want[0] < 0:
            assert h <= 0 or w <= 0, (H, W, ms, al, sst)
        else:
            assert (h, w) == tuple(want), (H, W, ms, al, sst)
    assert video.target_size(208, 300, 384, 32) == (192, 288) and video.target_size(216, 300, 384, 32) == (224, 288)


# ---- working directories ----

def _chunk(t, d):
    return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)


def png_file(img, color_type=2, bit_depth=8, interlace=0, extra=b""):
    """PNG bytes with any header and extra chunks after IHDR (the pixel data is only right for 8-bit types)."""
    raw = png.png_rgb_bytes(img) if color_type == 2 and img.ndim == 3 else png.png_gray_bytes(img.reshape(img.shape[0], -1))
    ihdr = _chunk(b"IHDR", struct.pack(">IIBBBBB", img.shape[1], img.shape[0], bit_depth, color_type, 0, 0, interlace))
    return raw[:8] + ihdr + extra + raw[33:]


def write_dir(root, frames, count=None, lines=None):
    """color_full/frame_%06d.png from [F, H, W, 3] u8 (R, G, B) frames, and frames.txt."""
    os.makedirs(os.path.join(root, "color_full"), exist_ok=True)
    for i, f in enumerate(frames):
        with open(os.path.join(root, "color_full", f"frame_{i:06d}.png"), "wb") as fh:
            fh.write(png.png_rgb_bytes(f))
    n = len(frames) if count is None else count
    H, W = frames.shape[1:3]
    with open(os.path.join(root, "frames.txt"), "w") as fh:
        fh.write(f"{n}\n{W}\n{H}\n" + "".join(f"{i / 30.0:.6f}\n" for i in range(n if lines is None else lines)))


def frames_rgb(n=3, H=21, W=37, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


def test_png_header(tmp_path):
    """The header fields, and an eXIf chunk found before or after the image data."""
    img = frames_rgb(1)[0]
    plain = png.png_rgb_bytes(img)
    with_exif = png_file(img, extra=_chunk(b"eXIf", b"MM\x00*\x00\x00\x00\x08\x00\x00"))
    late_exif = plain[:-12] + _chunk(b"eXIf", b"MM") + plain[-12:]
    for k, (data, exif) in enumerate(((plain, False), (with_exif, True), (late_exif, True))):
        fn = str(tmp_path / f"{k}.png")
        open(fn, "wb").write(data)
        assert png.png_header(fn) == {"height": 21, "width": 37, "bit_depth": 8, "color_type": 2, "interlace": 0, "exif": exif}
    fn = str(tmp_path / "cut.png")
    open(fn, "wb").write(plain[:-12])
    with pytest.raises(ValueError, match="truncated"):
        png.png_header(fn)
    open(fn, "wb").write(b"GIF89a" + bytes(40))
    with pytest.raises(ValueError, match="not a PNG"):
        png.png_header(fn)


def test_check_extracted_pts(tmp_path, capsys):
    v = video.Video(str(tmp_path))
    assert v.check_extracted_pts() is False
    write_dir(str(tmp_path), frames_rgb(3))
    assert v.check_extracted_pts() is True and v.frame_count == 3
    assert "3 frames detected (37 x 21)." in capsys.readouterr().out
    write_dir(str(tmp_path), frames_rgb(3), lines=2)
    with pytest.raises(SystemExit, match="^frames.txt has wrong number of lines$"):
        v.check_extracted_pts()


def test_skip_rule_and_exits(tmp_path):
    """check_frames: a missing or extension-less directory is not OK; a count that differs from the frame count, or a missing
    frame_%06d.<ext>, exits with the reference's messages; a complete directory is OK (and its outputs are skipped)."""
    root = str(tmp_path)
    write_dir(root, frames_rgb(3))
    v = video.Video(root)
    v.check_extracted_pts()
    d = os.path.join(root, "color_down")
    assert v.check_frames(d, "raw") is False
    os.makedirs(d)
    open(os.path.join(d, "notes.txt"), "w").close()
    assert v.check_frames(d, "raw") is False
    for i in (0, 1):
        open(os.path.join(d, f"frame_{i:06d}.raw"), "wb").close()
    with pytest.raises(SystemExit, match=rf"^ERROR: expected to find 3 files but found 2 in '{d}'$"):
        v.check_frames(d, "raw")
    with pytest.raises(SystemExit, match="expected to find 3 files but found 2"):
        video.downscale_all(root)
    open(os.path.join(d, "frame_000007.raw"), "wb").close()
    with pytest.raises(SystemExit, match=rf"^ERROR: did not find expected file '{d}/frame_000002.raw'$"):
        v.check_frames(d, "raw")
    os.rename(os.path.join(d, "frame_000007.raw"), os.path.join(d, "frame_000002.raw"))
    assert v.check_frames(d, "raw") is True
    assert v.check_frames(d, "raw", frames=[0, 1, 2]) is True
    # every output complete: nothing to do, no device needed
    for sub, ext in (("color_down_png", "png"), ("color_flow", "png")):
        os.makedirs(os.path.join(root, sub))
        for i in range(3):
            open(os.path.join(root, sub, f"frame_{i:06d}.{ext}"), "wb").close()
    stats = video.downscale_all(root)
    assert stats["outputs"] == [] and os.path.getsize(os.path.join(d, "frame_000000.raw")) == 0


def _outputs_absent(root):
    return not any(os.path.exists(os.path.join(root, d)) for d in ("color_down", "color_down_png", "color_flow"))


def test_refusals_before_anything_is_written(tmp_path):
    base = frames_rgb(3)

    def fresh(name):
        root = str(tmp_path / name)
        write_dir(root, base)
        return root
    # no frames.txt
    root = fresh("no_pts")
    os.remove(os.path.join(root, "frames.txt"))
    with pytest.raises(FileNotFoundError, match="frames.txt is missing"):
        video.downscale_all(root)
    with pytest.raises(FileNotFoundError, match="frames.txt is missing"):
        video.Video(root).downscale_frames("color_down", 384, "raw")
    # a missing frame (frames.txt counts 4)
    root = fresh("missing")
    write_dir(root, base, count=4)
    with pytest.raises(FileNotFoundError, match="frame_000003.png is missing"):
        video.downscale_all(root)
    # a frame of another size
    root = fresh("size")
    open(os.path.join(root, "color_full", "frame_000001.png"), "wb").write(png.png_rgb_bytes(base[1][:, :-1]))
    with pytest.raises(ValueError, match="but frame 0 has 37 x 21"):
        video.downscale_all(root)
    # frames that are not 8-bit RGB, interlaced or carry EXIF
    for name, data, msg in (
            ("gray", png_file(base[1][..., 0], color_type=0), "colour type 0"),
            ("palette", png_file(base[1][..., 0], color_type=3), "colour type 3"),
            ("rgba", png_file(base[1], color_type=6), "colour type 6"),
            ("gray_alpha", png_file(base[1][..., 0], color_type=4), "colour type 4"),
            ("rgb16", png_file(base[1], bit_depth=16), "16-bit"),
            ("interlaced", png_file(base[1], interlace=1), "interlaced"),
            ("exif", png_file(base[1], extra=_chunk(b"eXIf", b"MM\x00*")), "eXIf")):
        root = fresh(name)
        open(os.path.join(root, "color_full", "frame_000001.png"), "wb").write(data)
        with pytest.raises(ValueError, match=msg):
            video.downscale_all(root)
        assert _outputs_absent(root), name
    # a target side that rounds to 0: 37 x 21 at max_size 10 gives 10 x 5, then align 16 rounds 5 to 0
    root = fresh("zero")
    with pytest.raises(ValueError, match="gives 16 x 0 pixels"):
        video.Video(root).downscale_frames("color_down", 10, "raw", align=16)
    with pytest.raises(ValueError, match="gives 0 x 0 pixels"):
        video.Video(root).downscale_frames("color_down", 0, "raw", align=1)
    for name in ("no_pts", "missing", "size", "zero"):
        assert _outputs_absent(str(tmp_path / name)), name


def test_the_three_outputs_of_process_py(tmp_path):
    """downscale_all is DatasetProcessor.downscale_frames: color_down (.raw) and color_down_png at (size, align, short_side_target),
    color_flow at Flow.max_size() = 1024, align 64; one output that checks OK is skipped on its own."""
    calls = []
    real = video._downscale

    def spy(v, outputs, *a, **k):
        calls.append(outputs)
        return {"outputs": []}
    video._downscale = spy
    try:
        video.downscale_all(str(tmp_path), size=200, align=16, short_side_target=True)
        video.Video(str(tmp_path)).downscale_frames("x", 50, "png", align=8, full_subdir="full", short_side_target=True)
    finally:
        video._downscale = real
    assert calls[0] == [("color_down", 200, "raw", 16, True), ("color_down_png", 200, "png", 16, True), ("color_flow", 1024, "png", 64, False)]
    assert calls[1] == [("x", 50, "png", 8, True)]


def test_no_device_fails_loudly(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    root = str(tmp_path)
    write_dir(root, frames_rgb(2, H=33, W=45))
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        video.downscale_all(root)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        video.Video(root).downscale_frames("color_down", 384, "raw")
    assert _outputs_absent(root)


def test_abi_refusals_need_no_device():
    """Every refusal of rcvd_resize_area happens on the host: on a machine without a GPU it still returns RCVD_ERR_INVALID (not
    RCVD_ERR_NO_DEVICE), and zero frames return RCVD_OK."""
    L = solver.lib()
    fr = np.zeros((2, 5, 7, 3), np.uint8)
    a = np.full((2, 3, 4, 3), 7, np.float32)
    b = np.full((2, 2, 3, 3), 7, np.uint8)
    bufs = (C.c_void_p * 2)(a.ctypes.data, b.ctypes.data)

    def prm(**over):
        q = dict(width=7, height=5, num_frames=2, num_outputs=2)
        outs = over.pop("outs", [(4, 3, abi.RESIZE_RAW), (3, 2, abi.RESIZE_PNG)])
        q.update(over)
        p = abi.ResizeParams(**q)
        for k, (w, h, kind) in enumerate(outs):
            p.outputs[k] = abi.ResizeOutput(width=w, height=h, kind=kind)
        return C.byref(p)
    frp = fr.ctypes.data_as(C.POINTER(C.c_uint8))
    bad = [dict(width=0), dict(height=-1), dict(width=1 << 16, height=1 << 15), dict(num_frames=-1), dict(num_outputs=0),
           dict(num_outputs=4), dict(outs=[(0, 3, 0), (3, 2, 1)]), dict(outs=[(4, 3, 0), (3, -2, 1)]), dict(outs=[(4, 3, 2), (3, 2, 1)]),
           dict(outs=[(4, 3, 0), (1 << 16, 1 << 15, 1)])]
    for over in bad:
        assert L.rcvd_resize_area(prm(**over), 0, frp, bufs) == abi.ERR_INVALID, over
    assert L.rcvd_resize_area(None, 0, frp, bufs) == abi.ERR_INVALID
    assert L.rcvd_resize_area(prm(), 0, None, bufs) == abi.ERR_INVALID
    assert L.rcvd_resize_area(prm(), 0, frp, None) == abi.ERR_INVALID
    for k in range(2):
        nb = (C.c_void_p * 2)(a.ctypes.data, b.ctypes.data)
        nb[k] = None
        assert L.rcvd_resize_area(prm(), 0, frp, nb) == abi.ERR_INVALID, k
    assert np.all(a == 7) and np.all(b == 7)
    assert L.rcvd_resize_area(prm(num_frames=0), 0, None, None) == abi.OK
    ms = C.c_double()
    assert L.rcvd_debug_time_resize_area(prm(num_outputs=0), 0, frp, 1, C.byref(ms)) == abi.ERR_INVALID
    assert L.rcvd_debug_time_resize_area(prm(), 0, frp, 0, C.byref(ms)) == abi.ERR_INVALID
    with pytest.raises(ValueError):
        solver.resize_area(fr[..., :2], [(3, 4, "raw")])
    with pytest.raises(ValueError):
        solver.resize_area(fr, [(3, 4, "raw")] * 4)
