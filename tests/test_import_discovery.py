"""DepthVideoImporter on CPU: stream discovery (importVideo(video, path, True)) and track import (importTracks), each against a small
restatement of the reference's rules in this file; and the remaining lib_python names (computeDepthRange, Extrinsics.worldToCamera /
fromWorldToCamera, DepthVideo's frame times, reset and colorFrame) against numpy restatements."""
import ctypes
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

lp = pytest.importorskip("lib_python")
from robust_cvd_b200 import synthetic, synthetic_files  # noqa: E402

f32 = np.float32
CV_8UC1, CV_32FC3 = synthetic_files.CV_8UC1, synthetic_files.CV_32FC3
N, W, H = 4, 32, 24
# directory, stream name, extension, type (lib/Importer.cpp:43-48)
FIXED = [("color_full", "full", ".png", CV_32FC3), ("color_down", "down", ".raw", CV_32FC3),
         ("color_down_png", "down_png", ".png", CV_32FC3), ("dynamic_mask", "dynamic_mask", ".png", CV_8UC1)]

libc = ctypes.CDLL(None)
libc.atoi.argtypes, libc.atoi.restype = [ctypes.c_char_p], ctypes.c_int
libc.atof.argtypes, libc.atof.restype = [ctypes.c_char_p], ctypes.c_double


def _write(path, text):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write(text)


def _depth_stream(root, rel, frames=range(N)):
    d = os.path.join(root, rel, "depth"); os.makedirs(d, exist_ok=True)
    for i in frames:
        synthetic_files.write_raw(os.path.join(d, f"frame_{i:06d}.raw"), np.full((H, W), 0.5, f32))


def _scene(root):
    """A synthetic video directory (frames.txt, color_down, an empty color_full, depth_midas2, flow) plus the layouts discovery looks
    for: colour streams named by stream_info.txt, nested depth streams, a ground-truth stream with poses.txt and COLMAP depth."""
    synthetic_files.write_scene(synthetic.Scene(N, W, H, seed=5), root)
    _write(os.path.join(root, "extra_rgb", "stream_info.txt"), "color .png 32FC3\n")
    _write(os.path.join(root, "extra_mask", "stream_info.txt"), "color\n.png\n8UC1")
    _write(os.path.join(root, "flow", "stream_info.txt"), "flow .raw 32FC2\n")          # not a colour stream
    _write(os.path.join(root, "full", "stream_info.txt"), "color .png 32FC3\n")         # has a fixed stream's name: skipped
    _write(os.path.join(root, "color_down", "stream_info.txt"), "color .raw 32FC3\n")   # a fixed stream's directory: found again
    _depth_stream(root, "a/b")
    _depth_stream(root, "a/c/d")
    _depth_stream(root, "depth_midas2/x")      # inside a depth stream: not looked at
    _depth_stream(root, "depth_gt")
    _write(os.path.join(root, "depth_gt", "poses.txt"), "2\n1 2 3 0 0 0 1 0.5 0.4\n4 5 6 0 0 0 1 0.6 0.3\n")
    d = os.path.join(root, "depth_colmap_dense", "depth"); os.makedirs(d)
    for i in range(N):
        synthetic_files.write_raw(os.path.join(d, f"frame_{i:06d}.raw"), np.full((H, W), 2.0, f32))
    _write(os.path.join(root, "colmap_dense", "scales.csv"), "frame_000000.png,0.5\nframe_000001.png,1.5\n")
    return root


def expected_streams(root):
    """lib/Importer.cpp:39-164 restated: colour streams (name, dir, extension, type) and depth streams (name, dir), in order."""
    color = [(name, d, ext, t) for d, name, ext, t in FIXED if os.path.isdir(os.path.join(root, d))]
    for e in sorted(os.scandir(root), key=lambda e: e.path):
        info = os.path.join(e.path, "stream_info.txt")
        if not e.is_dir() or e.name in [name for _, name, _, _ in FIXED] or not os.path.exists(info):
            continue
        tok = open(info).read().split()
        if tok[0] == "color":
            color.append((e.name, e.name, tok[1], {"32FC3": CV_32FC3, "8UC1": CV_8UC1}[tok[2]]))
    found = []

    def walk(d):
        for e in os.scandir(d):
            if e.is_dir():
                if os.path.isdir(os.path.join(e.path, "depth")):
                    found.append(os.path.relpath(e.path, root))
                else:
                    walk(e.path)
    walk(root)
    depth = [(s, "depth_colmap_dense_imported" if s == "depth_colmap_dense" else s) for s in sorted(found) if s != "depth_colmap_dense_imported"]
    return color, depth


def _color_streams_of_saved_video(root):
    """(name, dir, extension, type) of each colour stream, read back from the video.dat that DepthVideo.save() writes."""
    b = open(os.path.join(root, "video.dat"), "rb").read()
    o = 12
    n, = struct.unpack_from("<i", b, o); o += 4 + 4 * n
    ncs, = struct.unpack_from("<i", b, o); o += 4
    out = []
    for _ in range(ncs):
        s = []
        for _ in range(3):
            k, = struct.unpack_from("<Q", b, o); s.append(b[o + 8:o + 8 + k].decode()); o += 8 + k
        t, = struct.unpack_from("<i", b, o); o += 13
        out.append((*s, t))
    return out


def _discover(root):
    v = lp.DepthVideo()
    lp.DepthVideoImporter.importVideo(v, root, True)
    return v


def _check_streams(v, root):
    color, depth = expected_streams(root)
    v.save()
    assert _color_streams_of_saved_video(root) == color
    assert [(v.colorStream(i).name(), v.colorStream(i).path(), v.colorStream(i).extension()) for i in range(v.numColorStreams())] == \
        [(name, root + "/" + d, ext) for name, d, ext, _ in color]
    assert [(v.depthStream(i).name(), v.depthStream(i).path()) for i in range(v.numDepthStreams())] == [(n, root + "/" + d) for n, d in depth]
    return color, depth


def test_discovery_finds_the_streams_in_the_reference_order(tmp_path):
    root = _scene(str(tmp_path / "v"))
    v = _discover(root)
    color, depth = _check_streams(v, root)
    # the quirks the restatement shares with the reference, spelled out
    assert [c[0] for c in color] == ["full", "down", "color_down", "extra_mask", "extra_rgb"]
    assert [d[0] for d in depth] == ["a/b", "a/c/d", "depth_colmap_dense", "depth_gt", "depth_midas2"]
    # COLMAP depth scaled into depth_colmap_dense_imported by (1 + 0.5 + 1.5) / 2
    got = synthetic_files.read_raw(os.path.join(root, "depth_colmap_dense_imported", "depth", "frame_000002.raw"))
    assert (got == f32(2.0) * f32(1.5)).all()
    # poses.txt of depth_gt: two frames set, the others disabled; no other stream touched
    gt = v.depthStream(v.depthStreamIndex("depth_gt"))
    assert list(np.asarray(gt.frame(1).extrinsics.position)) == [4, 5, 6] and f32(gt.frame(1).intrinsics.hFov) == f32(0.6)
    assert [gt.frame(i)._enabled for i in range(N)] == [True, True, False, False]
    assert all(v.depthStream(0).frame(i)._enabled for i in range(N))
    assert not os.path.exists(os.path.join(root, "long_tracks.tracktable"))
    # a second import reads the imported COLMAP depth as it is and skips its directory as a stream
    fn = os.path.join(root, "depth_colmap_dense_imported", "depth", "frame_000001.raw")
    before = os.stat(fn).st_mtime_ns
    _check_streams(_discover(root), root)
    assert os.stat(fn).st_mtime_ns == before


def test_discovery_rejects_a_bad_format_string(tmp_path):
    root = _scene(str(tmp_path / "v"))
    _write(os.path.join(root, "extra_bad", "stream_info.txt"), "color .png 16UC1\n")
    with pytest.raises(RuntimeError, match="Invalid format string."):
        _discover(root)


def _colmap_npz(path, shift):
    from scipy.spatial.transform import Rotation
    extr = np.zeros((N, 3, 4))
    for i in range(N):
        extr[i, :, :3] = Rotation.from_rotvec([0.1 * i, -0.05, 0.02 * i]).as_matrix()
        extr[i, :, 3] = [shift + i, 2.0 * i, -1.0]
    intr = np.tile([30.0, 30.0, W / 2, H / 2], (N, 1))
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez(path, extrinsics=extr, intrinsics=intr)
    return extr


def test_discovery_imports_the_first_colmap_reconstruction_into_every_depth_stream(tmp_path):
    root = _scene(str(tmp_path / "v"))
    first = _colmap_npz(os.path.join(root, "metadata.npz"), 10.0)
    _colmap_npz(os.path.join(root, "colmap_dense", "metadata.npz"), -7.0)
    v = _discover(root)
    _, depth = _check_streams(v, root)
    scale = f32(f32(f32(1) + f32(0.5)) + f32(1.5)) / f32(2)
    for s in range(len(depth)):
        for i in range(N):
            fr = v.depthStream(s).frame(i)
            assert fr._enabled     # also depth_gt's frames 2 and 3, which poses.txt disabled
            np.testing.assert_array_equal(np.asarray(fr.extrinsics.position), first[i, :, 3].astype(f32) / scale)
    os.remove(os.path.join(root, "metadata.npz"))
    v = _discover(root)
    assert f32(v.depthStream(0).frame(1).extrinsics.position[0]) == f32(-6.0) / scale


# --- importTracks ---

def _lines(text, sep):
    """std::getline over text with the separator: a trailing empty piece is dropped, an inner one is kept."""
    parts = text.split(sep)
    if parts[-1] == "":
        parts.pop()
    return parts


def tracks_restated(text, w):
    """lib/Importer.cpp:481-534 restated: the .tracktable bytes (TrackTable::serialize) and the tracks as (first frame, [n, 2])."""
    tracks, ids, last = [], {}, -1
    for line in _lines(text, "\n"):
        p = [s.strip() for s in _lines(line, ",")]
        if len(p) != 4:
            continue
        frame, tid = libc.atoi(p[0].encode()), libc.atoi(p[1].encode())
        x, y = f32(libc.atof(p[2].encode())), f32(libc.atof(p[3].encode()))
        assert frame >= last and frame >= 0
        last = frame
        if tid in ids:
            first, obs = tracks[ids[tid]]
            assert first + len(obs) == frame
            obs.append((x / f32(w), y / f32(w)))
        else:
            ids[tid] = len(tracks)
            tracks.append((frame, [(x / f32(w), y / f32(w))]))
    tracks = [(first, np.array(obs, f32).reshape(-1, 2)) for first, obs in tracks]
    data = struct.pack("<Q", len(tracks)) + b"".join(b"\x01" + struct.pack("<QQ", first, len(o)) + o.tobytes() for first, o in tracks)
    return data + struct.pack("<QQ", 0, last + 1), tracks


def _full_frame(root, w=W):
    os.makedirs(os.path.join(root, "color_full"), exist_ok=True)
    synthetic_files.write_png_gray(os.path.join(root, "color_full", "frame_000000.png"), np.zeros((H, w), np.uint8))


TRACKS = ("frame,track,x,y\n"                  # a header: track 0 at frame 0 at (0, 0)
          "0, 7, 12.5, 3.25\n"
          "0,9,1e1,  -2\r\n"
          " 1 ,7 , 13.75 ,\t4.0\n"
          "1,9,11,-1.5,\n"                     # a trailing empty field is dropped: four fields
          "1,3\n"                              # short: skipped
          "1,4,5,6,7\n"                        # long: skipped
          "1,,2,2\n"                           # an inner empty field is kept: track 0, which is at frame 0
          "\n"
          "2,7,0x10,1.5e-3\n"
          "2,3,31.999,23\n"
          "3,3,1,1\n")


def test_import_tracks_writes_the_reference_table(tmp_path, capfd):
    root = str(tmp_path / "v")
    synthetic_files.write_scene(synthetic.Scene(N, W, H, seed=5), root)
    _full_frame(root, w=40)
    v = _discover(root)
    text = TRACKS
    csv = os.path.join(root, "track2d.csv"); _write(csv, text)
    lp.DepthVideoImporter.importTracks(v, csv)
    out = os.path.join(root, "long_tracks.tracktable")
    want, tracks = tracks_restated(text, 40)
    assert open(out, "rb").read() == want
    assert [t[0] for t in tracks] == [0, 0, 0, 2] and len(tracks[1][1]) == 3
    cap = capfd.readouterr()
    assert "ERROR: invalid line '1,3'." in cap.out + cap.err and "ERROR: invalid line '1,4,5,6,7'." in cap.out + cap.err
    t = lp.DepthVideoTrackTable(); t.load(out)
    got = t._tracks()
    assert len(got) == len(tracks)
    for (gf, go), (wf, wo) in zip(got, tracks):
        assert gf == wf and go.dtype == f32
        np.testing.assert_array_equal(go, wo)
    t.save(str(tmp_path / "again.tracktable"))
    assert open(str(tmp_path / "again.tracktable"), "rb").read() == want
    # discovery imports track2d.csv the same way
    os.remove(out)
    _discover(root)
    assert open(out, "rb").read() == want


@pytest.mark.parametrize("text, msg", [
    ("0,1,1,1\n2,1,1,1\n", "after its last one at frame 0"),                 # a gap within a track
    ("0,1,1,1\n1,2,1,1\n1,1,1,1\n1,1,2,2\n", "after its last one at frame 1"),   # a repeated frame within a track
    ("0,,1,1\n1,1,1,1\n2,,2,2\n", "after its last one at frame 0"),         # track 0 (an empty field) continued late
    ("1,1,1,1\n0,2,1,1\n", "Frames not in consecutive order"),
    ("-1,1,1,1\n", "at frame -1"),
    ("-4,1,1,1\n", "Frames not in consecutive order"),
], ids=["gap", "repeat", "empty-id", "order", "minus-one", "negative"])
def test_import_tracks_rejects_what_the_reference_cannot_file(tmp_path, text, msg):
    root = str(tmp_path / "v")
    synthetic_files.write_scene(synthetic.Scene(N, W, H, seed=5), root)
    _full_frame(root)
    v = _discover(root)
    csv = os.path.join(root, "track2d.csv"); _write(csv, text)
    with pytest.raises(RuntimeError, match=msg):
        lp.DepthVideoImporter.importTracks(v, csv)
    assert not os.path.exists(os.path.join(root, "long_tracks.tracktable"))
    with pytest.raises(RuntimeError, match=msg):
        _discover(root)
    assert not os.path.exists(os.path.join(root, "long_tracks.tracktable"))


def test_import_tracks_needs_the_file_and_the_full_stream(tmp_path):
    root = str(tmp_path / "v")
    synthetic_files.write_scene(synthetic.Scene(N, W, H, seed=5), root)
    v = _discover(root)                                              # color_full exists but has no frame 0
    with pytest.raises(RuntimeError, match="Cannot open track file."):
        lp.DepthVideoImporter.importTracks(v, os.path.join(root, "missing.csv"))
    csv = os.path.join(root, "track2d.csv"); _write(csv, "0,1,1,1\n")
    with pytest.raises(RuntimeError, match="'full' has no image for frame 0"):
        lp.DepthVideoImporter.importTracks(v, csv)
    v = lp.DepthVideo(); lp.DepthVideoImporter.importVideo(v, root, False)
    with pytest.raises(RuntimeError, match="Color stream 'full' not found."):
        lp.DepthVideoImporter.importTracks(v, csv)
    assert not os.path.exists(os.path.join(root, "long_tracks.tracktable"))


# --- the remaining bindings ---

def test_the_reference_names_are_bound():
    for owner, names in [(lp, ["computeDepthRange", "MetaFrame"]), (lp.DepthFrame, ["warp"]),
                         (lp.Extrinsics, ["worldToCamera", "fromWorldToCamera"]), (lp.MetaFrame, ["pts"]),
                         (lp.DepthVideo, ["reset", "frame", "duration", "timeToFrame", "time", "colorFrame"]),
                         (lp.DepthVideoImporter, ["importTracks"])]:
        assert [n for n in names if not hasattr(owner, n)] == []


def depth_range_restated(d):
    v = d[np.isfinite(d) & (d > 0)]
    fmax, fmin = np.finfo(f32).max, np.finfo(f32).tiny
    return (min(v.min(), fmax), max(v.max(), fmin)) if v.size else (fmax, fmin)


def test_compute_depth_range():
    rng = np.random.default_rng(4)
    d = rng.uniform(-2, 9, (7, 11)).astype(f32)
    d.flat[:6] = [np.nan, np.inf, -np.inf, 0.0, -0.0, 3e-39]
    cases = [d, np.array([[np.nan, np.inf], [-np.inf, -1.0]], f32), np.zeros((3, 2), f32), np.array([[3e-39, 1e-40]], f32),
             np.array([[np.inf, 2.5, 0.0]], f32), np.zeros((0, 4), f32), d.astype(np.float64)[:, ::2]]
    for a in cases:
        got = lp.computeDepthRange(a)
        assert tuple(f32(g) for g in got) == depth_range_restated(np.asarray(a, f32)), a
    assert lp.computeDepthRange(np.zeros((3, 2), f32)) == (float(np.finfo(f32).max), float(np.finfo(f32).tiny))
    with pytest.raises(RuntimeError):
        lp.computeDepthRange(np.ones(4, f32))


def _extrinsics(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    e = lp.Extrinsics()
    e.position = rng.normal(size=3) * 3
    e.orientation = lp._makeQuat(*q.astype(f32))
    return e


def world_to_camera_restated(e):
    """rotate * translate in float32; the rows of rotate are the orientation's rotation matrix's columns (q * unit axes)."""
    x, y, z, w = (f32(c) for c in (e.orientation.x(), e.orientation.y(), e.orientation.z(), e.orientation.w()))
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], f32)
    rotate, translate = np.eye(4, dtype=f32), np.eye(4, dtype=f32)
    rotate[:3, :3] = R.T
    translate[:3, 3] = -np.asarray(e.position, f32)
    return rotate @ translate


def test_world_to_camera_and_back():
    rng = np.random.default_rng(8)
    for _ in range(50):
        e = _extrinsics(rng)
        M = e.worldToCamera()
        assert M.dtype == f32 and M.shape == (4, 4)
        np.testing.assert_allclose(M, world_to_camera_restated(e), rtol=1e-6, atol=1e-6)
        np.testing.assert_array_equal(M[:3, :3], np.stack([e.right(), e.up(), e.backward()]))
        b = lp.Extrinsics.fromWorldToCamera(M)
        np.testing.assert_allclose(np.asarray(b.position), np.asarray(e.position), rtol=0, atol=1e-5)
        qa = np.array([e.orientation.x(), e.orientation.y(), e.orientation.z(), e.orientation.w()])
        qb = np.array([b.orientation.x(), b.orientation.y(), b.orientation.z(), b.orientation.w()])
        assert min(np.abs(qa - qb).max(), np.abs(qa + qb).max()) <= 1e-5
    with pytest.raises(RuntimeError):
        lp.Extrinsics.fromWorldToCamera(np.eye(3, dtype=f32))


def test_frame_times_and_time_to_frame(tmp_path):
    root = str(tmp_path / "v")
    stamps = ["10.0", "10.5", "11.25", "13.0", "13.1"]
    _write(os.path.join(root, "frames.txt"), f"{len(stamps)}\n{W}\n{H}\n" + "\n".join(stamps) + "\n")
    os.makedirs(os.path.join(root, "color_down"))
    v = _discover(root)
    pts = [f32(s) - f32(stamps[0]) for s in stamps]
    assert [v.time(i) for i in range(5)] == pts and [v.frame(i).pts() for i in range(5)] == pts
    duration = f32(f32(pts[-1] * f32(5)) / f32(4))
    assert f32(v.duration()) == duration
    for t, want in [(0.0, 0), (0.49, 0), (0.5, 1), (1.3, 2), (pts[3], 3), (3.05, 3), (pts[4], 4), (float(duration), 4)]:
        assert v.timeToFrame(t) == want, t
    with pytest.raises(RuntimeError, match="Query time before first frame's time."):
        v.timeToFrame(-0.01)
    with pytest.raises(RuntimeError, match="Query time after video duration."):
        v.timeToFrame(float(duration) + 0.01)
    for bad in (5, -1):
        with pytest.raises(IndexError):
            v.frame(bad)
        with pytest.raises(IndexError):
            v.time(bad)
    assert v.colorFrame(0, 4).image() is None           # color_down has no files
    for s, f in ((1, 0), (0, 5), (-1, 0)):
        with pytest.raises(IndexError):
            v.colorFrame(s, f)
    v.reset()
    assert (v.numFrames(), v.numColorStreams(), v.numDepthStreams(), v.path(), v.duration(), v.aspect(), v.invAspect()) == (0, 0, 0, "", 0, 0, 0)
    assert (v.width(), v.height()) == (W, H)             # kept, as in the reference
    with pytest.raises(RuntimeError, match="Video has no frames."):
        v.timeToFrame(0.0)
