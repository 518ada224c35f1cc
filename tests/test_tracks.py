"""Long point tracks on the CPU: the sequential float32 restatement (tests/tracks_ref.py) against its committed golden and against
hand-built cases that each exercise one rule of the reference loop (lib/Processor.cpp:646-886), the DepthVideoTrackTable file format,
and the host-side checks of DepthVideoProcessor::computeTracks, which all happen before any device work."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import tracks_ref  # noqa: E402
from tests.tracks_ref import FLOW, HAS_COLOR, IN_RANGE, MASK  # noqa: E402
from robust_cvd_b200 import synthetic, synthetic_files  # noqa: E402

f32 = np.float32
CV_8UC1, CV_8UC3, CV_32FC3 = 0, 16, 21
ALL = IN_RANGE | HAS_COLOR | FLOW | MASK


def mapped_row(y, h, ia):
    """The row the reference checks and stamps a spawn candidate of row y at: int(float(float(y / h) * ia) / ia * h)."""
    return int(f32(f32(f32(f32(y) / f32(h)) * ia) / ia) * f32(h))


def clip(F, h, w, seed=0):
    """Random colour, zero flow, full masks, every frame in range."""
    rng = np.random.default_rng(seed)
    color = rng.uniform(0, 1, (F, h, w, 3)).astype(f32)
    return color, np.full(F, ALL, np.uint8), np.zeros((F, h, w, 2), f32), np.full((F, h, w), 255, np.uint8)


# ---- hand-built cases, one rule each; tests/test_gpu_tracks.py runs the same cases on the device ----
def case_remapped_row():
    """384x224: candidates only where the dynamic mask is set (min distance 0).  Row 31 is checked at row 30, so (x, 30) and (x, 31)
    share one checked pixel; (200, 31) is alone."""
    F, h, w = 2, 224, 384
    color, flags, flow, fmask = clip(F, h, w, seed=3)
    dyn = np.zeros((F, h, w), np.uint8)
    dyn[0, 30:32, 100] = 255; dyn[0, 31, 200] = 255
    return dict(color=color, flags=flags, flow=flow, flow_mask=fmask, dyn_masks=dyn, spawn_distance=0, prune_distance=0,
                min_dynamic_distance=0, inv_aspect=f32(h) / f32(w))


def case_continue_ge_spawn_gt():
    """min distance 1: frame 1's mask has column 4 dynamic, so column 5 is at distance exactly 1: tracks continue onto it (>=) but no
    track spawns on it (>)."""
    F, h, w = 3, 16, 16
    color, flags, flow, fmask = clip(F, h, w, seed=4)
    dyn = np.full((F, h, w), 255, np.uint8)
    dyn[0] = 0; dyn[0, 3:10, 3:10] = 255          # frame 0: candidates in the block's interior (distance > 1)
    dyn[1, :, 4] = 0
    return dict(color=color, flags=flags, flow=flow, flow_mask=fmask, dyn_masks=dyn, spawn_distance=0, prune_distance=0,
                min_dynamic_distance=1, inv_aspect=1.0)


def case_negative_x(dx):
    """Every pixel flows to x = dx; prune 0 keeps one track per landing row."""
    F, h, w = 2, 12, 16
    color, flags, flow, fmask = clip(F, h, w, seed=5)
    flow[1, :, :, 0] = f32(dx) - np.arange(w, dtype=f32)[None, :]
    return dict(color=color, flags=flags, flow=flow, flow_mask=fmask, spawn_distance=0, prune_distance=0, min_dynamic_distance=3, inv_aspect=0.75)


def case_spawn_mask():
    """The spawn candidates of frame f are restricted by the mask of (f-1 -> f): none at local frame 0 (no MASK flag there), the left
    half of frame 1 masked out."""
    F, h, w = 3, 12, 16
    color, flags, flow, fmask = clip(F, h, w, seed=6)
    flags[0] = IN_RANGE | HAS_COLOR
    fmask[0] = 0                                   # would forbid every spawn in frame 0 if it were read
    fmask[1, :, :8] = 0
    return dict(color=color, flags=flags, flow=flow, flow_mask=fmask, spawn_distance=0, prune_distance=0, min_dynamic_distance=3, inv_aspect=0.75)


def case_equal_scores():
    """Flat colour: every corner score is 0, so candidates are taken in scan order."""
    F, h, w = 2, 12, 16
    color, flags, flow, fmask = clip(F, h, w)
    color[:] = 0.5
    return dict(color=color, flags=flags, flow=flow, flow_mask=fmask, spawn_distance=2, prune_distance=0, min_dynamic_distance=3, inv_aspect=0.75)


CASES = {"remapped_row": case_remapped_row, "continue_ge_spawn_gt": case_continue_ge_spawn_gt, "negative_x_kept": lambda: case_negative_x(-1.2),
         "negative_x_dropped": lambda: case_negative_x(-1.6), "spawn_mask": case_spawn_mask, "equal_scores": case_equal_scores}


def test_restatement_against_committed_golden():
    """tests/golden/tracks_golden.npz (written by `python tests/tracks_ref.py`) pins the restatement."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "tracks_golden.npz"))
    for name, kw in tracks_ref.golden_configs():
        (off, ids, locs), n = tracks_ref.run_golden(name, kw)
        np.testing.assert_array_equal(off, g[f"{name}_offsets"], err_msg=name)
        np.testing.assert_array_equal(ids, g[f"{name}_ids"], err_msg=name)
        assert locs.tobytes() == g[f"{name}_locs"].tobytes(), name
        assert n == int(g[f"{name}_count"]), name


def test_spawn_on_a_remapped_row_and_a_shared_checked_pixel():
    c = case_remapped_row()
    h, w, ia = 224, 384, c["inv_aspect"]
    assert mapped_row(31, h, ia) == 30 and mapped_row(30, h, ia) == 30
    tracks, frames = tracks_ref.compute_tracks(**c)
    rows = sorted(int(round(float(t[0][2] / ia * h))) for t in tracks)
    cols = sorted(int(round(float(t[0][1] * w))) for t in tracks)
    assert len(frames[0]) == 2 and cols == [100, 200]      # one of (100, 30) / (100, 31): they share the checked pixel (100, 30)
    assert 31 in rows
    assert frames[1] == frames[0]                           # last frame: no spawn, both tracks continue (distance 0 >= 0)


def test_continuation_uses_ge_and_spawn_uses_gt():
    tracks, frames = tracks_ref.compute_tracks(**case_continue_ge_spawn_gt())
    born0 = set(frames[0])
    on_col5 = [tid for tid in frames[1] if int(round(float(tracks[tid][-1][1] * 16))) == 5]
    assert on_col5 and set(on_col5) <= born0               # continued onto distance 1, none spawned there
    spawned1 = [tid for tid in frames[1] if tid not in born0]
    assert spawned1 and all(int(round(float(tracks[t][0][1] * 16))) not in (4, 5) for t in spawned1)


def test_continuation_accepted_just_left_of_the_image():
    tracks, frames = tracks_ref.compute_tracks(**case_negative_x(-1.2))
    xs = [tracks[t][-1][1] for t in frames[1]]
    assert len(xs) == 12 and all(-1.5 / 16 < x < -1.0 / 16 for x in xs)   # fx1 ~ -1.2, int(fx1 + 0.5) = 0: inside
    _, frames = tracks_ref.compute_tracks(**case_negative_x(-1.6))
    assert frames[1] == []


def test_spawn_mask_comes_from_the_pair_into_the_frame():
    tracks, frames = tracks_ref.compute_tracks(**case_spawn_mask())
    assert len(frames[0]) == 12 * 16                        # spawn 0 and no mask: every pixel of frame 0
    new1 = [t for t in frames[1] if t >= 12 * 16]
    assert new1 == []                                       # the continued tracks cover every right-half pixel
    assert len(frames[1]) == 12 * 8 and all(tracks[t][-1][1] >= f32(0.5) for t in frames[1])
    assert len(frames[2]) == 12 * 8


def test_equal_scores_are_taken_in_scan_order():
    tracks, frames = tracks_ref.compute_tracks(**case_equal_scores())
    first = [(int(round(float(tracks[t][0][1] * 16))), int(round(float(tracks[t][0][2] / f32(0.75) * 12)))) for t in frames[0][:3]]
    assert first == [(0, 0), (3, 0), (6, 0)]


def test_short_tracks_leave_invalid_ids():
    tracks, _ = tracks_ref.compute_tracks(**case_spawn_mask())
    table = tracks_ref.delete_short(tracks, 3)
    dead = [i for i, t in enumerate(table) if t is None]   # left-half tracks end in frame 0, right-half ones live 3 frames
    assert len(dead) == 12 * 8 and all(tracks[i][0][1] < f32(0.5) for i in dead) and len(table) == 12 * 16
    data = tracks_ref.serialize(table, 3)
    assert len(data) == 8 + 12 * 16 + 12 * 8 * (16 + 3 * 8) + 16      # one byte per deleted id


# ---- file format through lib_python ----
def test_track_table_file_round_trip(tmp_path):
    lp = pytest.importorskip("lib_python")
    tracks, _ = tracks_ref.compute_tracks(**case_spawn_mask())
    table = tracks_ref.delete_short(tracks, 2)
    data = tracks_ref.serialize(table, 7, first_frame=2)
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    src.write_bytes(data)
    t = lp.DepthVideoTrackTable()
    t.load(str(src))
    t.save(str(dst))
    assert dst.read_bytes() == data
    got = t._tracks()
    assert len(got) == len(table)
    for a, b in zip(got, table):
        assert (a is None) == (b is None)
        if b is not None:
            assert a[0] == b[0][0] + 2
            assert a[1].tobytes() == np.asarray([(x, y) for _, x, y in b], f32).tobytes()
    with pytest.raises(RuntimeError, match="Could not open file"):
        t.load(str(tmp_path / "missing.bin"))
    empty = tmp_path / "empty.bin"
    lp.DepthVideoTrackTable().save(str(empty))
    assert empty.read_bytes() == tracks_ref.serialize([], 0)


# ---- the C ABI and lib_python without a device ----
def _no_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is present")
    except ImportError:
        pass


def test_solver_compute_tracks_needs_a_device():
    import ctypes as C
    from robust_cvd_b200 import abi, solver
    _no_gpu()
    c = case_equal_scores()
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        solver.compute_tracks(c["color"], c["flags"], c["flow"], c["flow_mask"])
    prm = abi.TrackParams(num_frames=2, width=16, height=12, spawn_distance=2, prune_distance=0, min_dynamic_distance=3, inv_aspect=0.75)
    off = np.zeros(3, np.int64); n = C.c_int64(0)
    color, flags = np.ascontiguousarray(c["color"]), np.full(2, IN_RANGE | HAS_COLOR, np.uint8)
    rc = solver.lib().rcvd_compute_tracks(C.byref(prm), 0, color.ctypes.data_as(C.c_void_p), None, None, None, flags.ctypes.data_as(C.c_void_p),
                                          off.ctypes.data_as(C.c_void_p), None, None, C.c_int64(0), C.byref(n))
    assert rc == abi.ERR_NO_DEVICE


@pytest.fixture(scope="module")
def scene_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("tracks_scene"))
    synthetic_files.write_scene(synthetic.Scene(5, 24, 16, seed=2), root, dynamic_masks=np.full((5, 16, 24), 255, np.uint8))
    return root


def _open(root, down_type=CV_32FC3, dynamic=False):
    lp = pytest.importorskip("lib_python")
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", down_type)
    if dynamic:
        v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
    return lp, v


def test_lib_python_compute_tracks_needs_a_device(scene_root):
    _no_gpu()
    lp, v = _open(scene_root, dynamic=True)
    p = lp.DepthVideoProcessor.Params(); p.frameRange.fromString("1-4")
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        lp.DepthVideoProcessor(v).computeTracks(p)


def test_process_does_not_dispatch_compute_tracks(scene_root):
    lp, v = _open(scene_root)
    p = lp.DepthVideoProcessor.Params(); p.op = lp.DepthVideoProcessor.Op.ComputeTracks
    with pytest.raises(RuntimeError, match="Unsupported operation selected."):
        lp.DepthVideoProcessor(v).process(p)


def test_lib_python_compute_tracks_argument_errors(scene_root, tmp_path):
    lp, v = _open(scene_root)
    proc = lp.DepthVideoProcessor(v)
    p = lp.DepthVideoProcessor.Params(); p.frameRange.fromString("0-4")
    p.trackSpawnDistance = -1
    with pytest.raises(RuntimeError, match="must not be negative"):
        proc.computeTracks(p)
    p.trackSpawnDistance = 20; p.trackPruneDistance = -2
    with pytest.raises(RuntimeError, match="must not be negative"):
        proc.computeTracks(p)
    p.trackPruneDistance = 5
    lp, v8 = _open(scene_root, down_type=CV_8UC3)
    with pytest.raises(RuntimeError, match="CV_32FC3"):
        lp.DepthVideoProcessor(v8).computeTracks(p)
    import shutil
    root = str(tmp_path / "scene")
    shutil.copytree(scene_root, root)
    os.remove(os.path.join(root, "dynamic_mask", "frame_000003.png"))
    lp, vd = _open(root, dynamic=True)
    with pytest.raises(RuntimeError, match="Dynamic mask stream is missing frame 3"):
        lp.DepthVideoProcessor(vd).computeTracks(p)
    p.frameRange.fromString("0-2,4")                           # frame 3 outside the range: its mask is not needed
    _no_gpu()
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        lp.DepthVideoProcessor(vd).computeTracks(p)
