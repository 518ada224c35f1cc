"""Long point tracks on the GPU (csrc/rcvd_tracks.cuh) against the sequential float32 restatement of the reference loop
(tests/tracks_ref.py, lib/Processor.cpp:646-886): the same track ids in every frame and bit-equal locations, through the C ABI and
through lib_python (the saved file byte for byte)."""
import os
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

from tests import tracks_ref  # noqa: E402
from tests.test_tracks import CASES, mapped_row  # noqa: E402
from robust_cvd_b200 import solver, synthetic, synthetic_files  # noqa: E402

pytestmark = pytest.mark.gpu
f32 = np.float32
CV_8UC1, CV_32FC3 = 0, 21


def assert_same(kw):
    """GPU lists == restatement lists (before the deletion of short tracks); returns the restatement's (tracks, frames)."""
    tracks, frames = tracks_ref.compute_tracks(**kw)
    off, ids, locs, n = solver.compute_tracks(kw["color"], kw["flags"], kw.get("flow"), kw.get("flow_mask"), kw.get("dyn_masks"),
                                              kw["spawn_distance"], kw["prune_distance"], kw["min_dynamic_distance"], kw["inv_aspect"])
    roff, rids, rlocs = tracks_ref.frame_lists(tracks, len(kw["flags"]))
    assert n == len(tracks)
    np.testing.assert_array_equal(off, roff)
    np.testing.assert_array_equal(ids, rids)
    assert locs.tobytes() == rlocs.tobytes()
    return tracks, frames


@pytest.mark.parametrize("name", sorted(CASES))
def test_rule_cases(name):
    assert_same(CASES[name]())


def _scene(root, N, w, h, seed, dyn=None):
    sc = synthetic.Scene(N, w, h, seed=seed, hole_fraction=0.0)
    synthetic_files.write_scene(sc, root, pairs=[(i, i + 1) for i in range(N - 1)], dynamic_masks=dyn)
    return sc


def _blobs(N, h, w, seed):
    rng = np.random.default_rng(seed)
    m = np.full((N, h, w), 255, np.uint8)
    for f in range(N):
        for _ in range(3):
            cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(2, max(3, min(h, w) // 5))
            yy, xx = np.mgrid[0:h, 0:w]
            m[f][(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = rng.integers(0, 127)
    return m


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("gpu_tracks"))
    sc = _scene(root, 8, 64, 40, seed=5)
    return root, sc


def _inputs(root, sc, frames, dynamic=False, **kw):
    color, flags, flow, fmask, dyn = tracks_ref.load_inputs(root, frames, sc.w, sc.h, dynamic=dynamic)
    return dict(color=color, flags=flags, flow=flow, flow_mask=fmask, dyn_masks=dyn, inv_aspect=sc.inv_aspect32, **kw)


@pytest.mark.parametrize("spawn", [20, 7, 1, 0])
@pytest.mark.parametrize("prune", [5, 0])
def test_scene_spawn_prune_grid(scene, spawn, prune):
    root, sc = scene
    tracks, frames = assert_same(_inputs(root, sc, list(range(8)), spawn_distance=spawn, prune_distance=prune, min_dynamic_distance=3))
    assert sum(len(t) > 1 for t in tracks) > 0


@pytest.mark.parametrize("variant", ["min_dyn_-1", "dyn_colour_size", "dyn_other_size", "range_from_2", "range_gap", "missing_flow_bad_mask"])
def test_scene_variants(tmp_path, variant):
    N, w, h = 8, 64, 40
    root = str(tmp_path / "s")
    frames, dyn, mdd = list(range(N)), None, 3
    if variant == "dyn_colour_size":
        dyn = _blobs(N, h, w, 1)
    elif variant == "dyn_other_size":
        dyn = _blobs(N, 27, 45, 2)
    elif variant == "min_dyn_-1":
        mdd = -1
    elif variant == "range_from_2":
        frames = list(range(2, N))
    elif variant == "range_gap":
        frames = [0, 1, 2, 4, 5, 7]
    sc = _scene(root, N, w, h, seed=7, dyn=dyn)
    if variant == "missing_flow_bad_mask":
        os.remove(os.path.join(root, "flow", "flow_000002_000003.raw"))
        synthetic_files.write_png_gray(os.path.join(root, "flow_mask", "mask_000005_000006.png"), np.full((h - 1, w), 255, np.uint8))
    kw = _inputs(root, sc, frames, dynamic=dyn is not None, spawn_distance=7, prune_distance=2, min_dynamic_distance=mdd)
    assert_same(kw)


def test_remapped_rows_at_384x224(tmp_path):
    """At 384x224 some rows are checked one row up; the default Params spawn on at least one of them."""
    root = str(tmp_path / "s")
    sc = _scene(root, 3, 384, 224, seed=9)
    tracks, _ = assert_same(_inputs(root, sc, [0, 1, 2], spawn_distance=20, prune_distance=5, min_dynamic_distance=3))
    ia = sc.inv_aspect32
    rows = {int(f32(f32(t[0][2] / ia) * f32(224))) for t in tracks}
    assert any(mapped_row(y, 224, ia) != y for y in rows)


def test_dense_tracks_at_scale(tmp_path):
    """Spawn 0 / prune 0: thousands of live tracks per frame, several landing on one pixel: the prune selection at scale."""
    root = str(tmp_path / "s")
    sc = _scene(root, 4, 96, 64, seed=3)
    tracks, frames = assert_same(_inputs(root, sc, [0, 1, 2, 3], spawn_distance=0, prune_distance=0, min_dynamic_distance=3))
    assert min(len(frames[f]) for f in range(3)) > 3000
    assert_same(_inputs(root, sc, [0, 1, 2, 3], spawn_distance=0, prune_distance=5, min_dynamic_distance=3))


def test_lib_python_save_matches_restatement(tmp_path):
    lp = pytest.importorskip("lib_python")
    N, w, h = 8, 64, 40
    root = str(tmp_path / "s")
    sc = _scene(root, N, w, h, seed=11, dyn=_blobs(N, h, w, 4))
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    v.createColorStream("down", "color_down", ".raw", CV_32FC3)
    v.createColorStream("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)
    p = lp.DepthVideoProcessor.Params(); p.frameRange.fromString("1-6")
    p.trackSpawnDistance = 7; p.trackPruneDistance = 2
    l0 = solver.lib().rcvd_tracks_launch_count()
    table = lp.DepthVideoProcessor(v).computeTracks(p)
    assert solver.lib().rcvd_tracks_launch_count() > l0          # the CUDA path ran
    out = tmp_path / "tracks.bin"
    table.save(str(out))
    kw = _inputs(root, sc, list(range(1, 7)), dynamic=True, spawn_distance=7, prune_distance=2, min_dynamic_distance=3)
    kw["inv_aspect"] = f32(v.invAspect())
    tracks, _ = tracks_ref.compute_tracks(**kw)
    ref = tracks_ref.serialize(tracks_ref.delete_short(tracks, p.minTrackLength), N, first_frame=1)
    assert out.read_bytes() == ref
    assert sum(t is None for t in table._tracks()) > 0 and sum(t is not None for t in table._tracks()) > 0
