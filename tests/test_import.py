"""DepthVideoImporter on CPU: ground-truth poses (importPoses), scales.csv (loadScale), COLMAP depth maps (importColmapDepth) and
COLMAP cameras from metadata.npz (importColmapRecon), each against a numpy float32 restatement of the reference's arithmetic."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robust_cvd_b200", "host"))

lp = pytest.importorskip("lib_python")
from robust_cvd_b200 import synthetic_files  # noqa: E402

f32 = np.float32
N, W, H = 6, 40, 24


def _video_dir(root, n=N):
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "frames.txt"), "w") as f:
        f.write(f"{n}\n{W}\n{H}\n" + "".join(f"{i / 30.0:.6f}\n" for i in range(n)))
    return root


def _open(root):
    v = lp.DepthVideo()
    lp.DepthVideoImporter.importVideo(v, root, False)
    return v


def _scale_f32(values):
    """loadScale's arithmetic: a float sum that starts at 1, divided by the count."""
    s = f32(1)
    for x in values:
        s = f32(s + f32(x))
    return f32(s / f32(len(values)))


def _write_scales(path, values, extra_lines=()):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write("".join(f"frame_{i:06d}.png,{x!r}\n" for i, x in enumerate(values)) + "".join(extra_lines))


def eigen_quat_f32(R):
    """Eigen::Quaternionf(Matrix3f) restated in numpy float32, returns (x, y, z, w) and the branch taken. The trace is summed as Eigen's
    unrolled reduction does, R00 + (R11 + R22). Eigen is not available here, so this restatement is not itself checked against Eigen."""
    R = np.asarray(R, f32)
    q = np.zeros(4, f32)
    t = R[0, 0] + (R[1, 1] + R[2, 2])
    if t > 0:
        t = np.sqrt(t + f32(1)); q[3] = f32(0.5) * t; t = f32(0.5) / t
        q[0] = (R[2, 1] - R[1, 2]) * t; q[1] = (R[0, 2] - R[2, 0]) * t; q[2] = (R[1, 0] - R[0, 1]) * t
        return q, "trace"
    i = 0
    if R[1, 1] > R[0, 0]:
        i = 1
    if R[2, 2] > R[i, i]:
        i = 2
    j = (i + 1) % 3; k = (j + 1) % 3
    t = np.sqrt(R[i, i] - R[j, j] - R[k, k] + f32(1)); q[i] = f32(0.5) * t; t = f32(0.5) / t
    q[3] = (R[k, j] - R[j, k]) * t; q[j] = (R[j, i] + R[i, j]) * t; q[k] = (R[k, i] + R[i, k]) * t
    return q, i


def _quat(e):
    return np.array([e.orientation.x(), e.orientation.y(), e.orientation.z(), e.orientation.w()], f32)


# --- importPoses ---

def test_import_poses_reads_float32_and_disables_trailing_frames(tmp_path):
    root = _video_dir(str(tmp_path / "v"))
    rng = np.random.default_rng(1)
    vals = rng.normal(size=(4, 9))
    # 17 significant digits for some values, 9 for others: both must parse as std::istream >> float does
    text = "4\n" + "".join(" ".join(f"{x:.17g}" if (r + c) % 2 else f"{x:.9g}" for c, x in enumerate(row)) + "\n" for r, row in enumerate(vals))
    with open(os.path.join(root, "poses.txt"), "w") as f:
        f.write(text)
    want = np.array(text.split()[1:], dtype=f32).reshape(4, 9)
    v = _open(root)
    v.createDepthStream("depth_gt", "depth_gt", [-1, -1])
    lp.DepthVideoImporter.importPoses(v, os.path.join(root, "poses.txt"), 0)
    ds = v.depthStream(0)
    for i in range(4):
        fr = ds.frame(i)
        np.testing.assert_array_equal(np.asarray(fr.extrinsics.position), want[i, 0:3])
        np.testing.assert_array_equal(_quat(fr.extrinsics), want[i, 3:7])
        assert (f32(fr.intrinsics.hFov), f32(fr.intrinsics.vFov)) == (want[i, 7], want[i, 8])
    flags = [ds.frame(i)._enabled for i in range(N)]
    assert flags == [True] * 4 + [False] * (N - 4)
    v.save()
    v2 = lp.DepthVideo(); v2.load(root)
    assert [v2.depthStream(0).frame(i)._enabled for i in range(N)] == flags
    np.testing.assert_array_equal(np.asarray(v2.depthStream(0).frame(2).extrinsics.position), want[2, 0:3])


def test_import_poses_rejects_longer_files_and_missing_files(tmp_path):
    root = _video_dir(str(tmp_path / "v"))
    with open(os.path.join(root, "poses.txt"), "w") as f:
        f.write(f"{N + 1}\n" + "0 0 0 0 0 0 1 0.5 0.4\n" * (N + 1))
    v = _open(root)
    v.createDepthStream("depth_gt", "depth_gt", [-1, -1])
    with pytest.raises(RuntimeError, match="more frames than the video"):
        lp.DepthVideoImporter.importPoses(v, os.path.join(root, "poses.txt"), 0)
    with pytest.raises(RuntimeError, match="Could not open poses file"):
        lp.DepthVideoImporter.importPoses(v, os.path.join(root, "missing.txt"), 0)


# --- loadScale ---

def test_load_scale(tmp_path):
    root = str(tmp_path / "v"); os.makedirs(root)
    assert lp.DepthVideoImporter.loadScale(root) == 1.0
    vals = [0.37, 1.61803398875, 2.5]
    _write_scales(os.path.join(root, "a", "b", "scales.csv"), vals, extra_lines=["frame_000009.png;3.0\n"])
    got = lp.DepthVideoImporter.loadScale(root)
    assert f32(got) == _scale_f32(vals) and got != f32(np.mean(np.float32(vals)))
    # several files: the last one visited in sorted name order wins ("scales.csv" < "z")
    _write_scales(os.path.join(root, "scales.csv"), [5.0])
    _write_scales(os.path.join(root, "z", "scales.csv"), [7.0, 9.0])
    assert f32(lp.DepthVideoImporter.loadScale(root)) == _scale_f32([7.0, 9.0])


# --- importColmapDepth ---

def test_import_colmap_depth(tmp_path):
    root = _video_dir(str(tmp_path / "v"))
    vals = [0.8, 1.3]
    _write_scales(os.path.join(root, "colmap_dense", "scales.csv"), vals)
    scale = _scale_f32(vals)
    src = os.path.join(root, "depth_colmap_dense", "depth"); os.makedirs(src)
    rng = np.random.default_rng(2)
    inputs = {}
    for i in (0, 3):
        d = rng.uniform(0.01, 5.0, (H, W)).astype(f32)
        d.flat[:6] = [np.nan, np.inf, -np.inf, -1.0, -1e-30, 0.0]
        inputs[i] = d
        synthetic_files.write_raw(os.path.join(src, f"frame_{i:06d}.raw"), d)
    v = _open(root)
    lp.DepthVideoImporter.importColmapDepth(v)
    dst = os.path.join(root, "depth_colmap_dense_imported", "depth")
    assert sorted(os.listdir(dst)) == ["frame_000000.raw", "frame_000003.raw"]
    for i, d in inputs.items():
        got = synthetic_files.read_raw(os.path.join(dst, f"frame_{i:06d}.raw"))
        assert got.dtype == f32 and got.shape == (H, W)
        assert (got.flat[:5] == 0).all() and got.flat[5] == 0
        want = np.where(~np.isfinite(d) | (d < 0), f32(0), d * scale).astype(f32)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    # an existing destination is left as it is, even when the scale has changed since
    fn = os.path.join(dst, "frame_000003.raw")
    before = (os.stat(fn).st_mtime_ns, open(fn, "rb").read())
    _write_scales(os.path.join(root, "colmap_dense", "scales.csv"), [9.0])
    lp.DepthVideoImporter.importColmapDepth(v)
    assert (os.stat(fn).st_mtime_ns, open(fn, "rb").read()) == before


# --- importColmapRecon ---

def _rotations():
    """Camera-to-world rotations that drive each branch of the matrix-to-quaternion algorithm: positive trace, then the largest
    diagonal element at 0, 1 and 2 (rotations by ~170 degrees about x, y and z)."""
    from scipy.spatial.transform import Rotation
    return [Rotation.from_rotvec(v).as_matrix() for v in
            ([0.1, -0.2, 0.05], [2.9, 0.2, -0.1], [0.15, 2.95, 0.2], [-0.1, 0.2, 2.97], [0.4, 0.3, -1.2], [1.0, -2.0, 0.5])]


def _recon_scene(root, frames, scale_vals=(1.7, 2.2)):
    """A video of N frames whose COLMAP stream has depth files for `frames`; returns the metadata arrays and the expected scale."""
    _video_dir(root)
    _write_scales(os.path.join(root, "scales.csv"), list(scale_vals))
    dd = os.path.join(root, "depth_colmap_dense_imported", "depth"); os.makedirs(dd, exist_ok=True)
    for i in frames:
        synthetic_files.write_raw(os.path.join(dd, f"frame_{i:06d}.raw"), np.full((H, W), 0.5, f32))
    rng = np.random.default_rng(3)
    Rs = _rotations()[:len(frames)]
    extr = np.zeros((len(frames), 3, 4))
    for n, R in enumerate(Rs):
        extr[n, :, :3] = R; extr[n, :, 3] = rng.normal(size=3) * 3
    intr = np.stack([rng.uniform(20, 60, len(frames)), rng.uniform(20, 60, len(frames)), np.full(len(frames), W / 2), np.full(len(frames), H / 2)], 1)
    return extr, intr, _scale_f32(scale_vals)


def _recon(root, npz, silent=True):
    v = _open(root)
    v.createDepthStream("colmap_dense", "depth_colmap_dense_imported", [-1, -1])
    lp.DepthVideoImporter.importColmapRecon(v, npz, v.depthStreamIndex("colmap_dense"), silent)
    return v


@pytest.mark.parametrize("save", [np.savez, np.savez_compressed], ids=["stored", "deflated"])
def test_import_colmap_recon(tmp_path, save):
    root = str(tmp_path / "v")
    frames = [0, 2, 3, 5]
    extr, intr, scale = _recon_scene(root, frames)
    npz = os.path.join(root, "metadata.npz")
    save(npz, extrinsics=extr, intrinsics=intr, extra=np.arange(3, dtype=np.int32))
    v = _recon(root, npz, silent=False)
    ds = v.depthStream(0)
    branches = set()
    for n, f in enumerate(frames):
        fr = ds.frame(f)
        assert fr._enabled
        np.testing.assert_array_equal(np.asarray(fr.extrinsics.position), extr[n, :, 3].astype(f32) / scale)
        q, branch = eigen_quat_f32(extr[n, :, :3].astype(f32)); branches.add(branch)
        np.testing.assert_array_equal(_quat(fr.extrinsics), q)
        assert f32(fr.intrinsics.hFov) == f32(2 * np.arctan2(W / 2.0, intr[n, 0]))
        assert f32(fr.intrinsics.vFov) == f32(2 * np.arctan2(H / 2.0, intr[n, 1]))
    assert branches == {"trace", 0, 1, 2}
    for f in (1, 4):    # no depth file: disabled, camera untouched
        fr = ds.frame(f)
        assert not fr._enabled and not np.asarray(fr.extrinsics.position).any() and fr.extrinsics.orientation.w() == 1.0


def _write_zip64_npz(path, **arrays):
    """An .npz whose central directory and end record use zip64 for every field (what np.savez writes for members past 4 GiB):
    sizes, local header offsets, entry count and directory offset are all saturated and given in zip64 records."""
    import io
    import struct
    import zlib
    local, central = b"", b""
    for key, a in arrays.items():
        buf = io.BytesIO(); np.lib.format.write_array(buf, np.asanyarray(a)); data = buf.getvalue()
        name = (key + ".npy").encode(); crc = zlib.crc32(data); off = len(local); n = len(data)
        local += struct.pack("<IHHHHHIIIHH", 0x04034b50, 45, 0, 0, 0, 0, crc, 0xFFFFFFFF, 0xFFFFFFFF, len(name), 20) + name
        local += struct.pack("<HHQQ", 1, 16, n, n) + data
        central += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014b50, 45, 45, 0, 0, 0, 0, crc, 0xFFFFFFFF, 0xFFFFFFFF, len(name), 28, 0, 0, 0, 0, 0xFFFFFFFF)
        central += name + struct.pack("<HHQQQ", 1, 24, n, n, off)
    eocd64 = struct.pack("<IQHHIIQQQQ", 0x06064b50, 44, 45, 45, 0, 0, len(arrays), len(arrays), len(central), len(local))
    locator = struct.pack("<IIQI", 0x07064b50, 0, len(local) + len(central), 1)
    eocd = struct.pack("<IHHHHIIH", 0x06054b50, 0, 0, 0xFFFF, 0xFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0)
    with open(path, "wb") as f:
        f.write(local + central + eocd64 + locator + eocd)


def test_import_colmap_recon_reads_zip64_central_directory(tmp_path):
    root = str(tmp_path / "v")
    frames = [1, 2, 4]
    extr, intr, scale = _recon_scene(root, frames)
    npz = os.path.join(root, "metadata.npz")
    _write_zip64_npz(npz, intrinsics=intr, extrinsics=extr)
    with np.load(npz) as z:     # the hand-built archive is one numpy itself reads
        np.testing.assert_array_equal(z["extrinsics"], extr)
    v = _recon(root, npz)
    ds = v.depthStream(0)
    for n, f in enumerate(frames):
        np.testing.assert_array_equal(np.asarray(ds.frame(f).extrinsics.position), extr[n, :, 3].astype(f32) / scale)
        np.testing.assert_array_equal(_quat(ds.frame(f).extrinsics), eigen_quat_f32(extr[n, :, :3])[0])
        assert f32(ds.frame(f).intrinsics.vFov) == f32(2 * np.arctan2(H / 2.0, intr[n, 1]))


def test_import_colmap_recon_rejects_malformed_metadata(tmp_path):
    root = str(tmp_path / "v")
    frames = [0, 1, 4]
    extr, intr, _ = _recon_scene(root, frames)
    npz = os.path.join(root, "metadata.npz")
    cases = [
        (dict(extrinsics=np.zeros((3, 4, 4)), intrinsics=intr), r"has shape \(3, 4, 4\); expected \(N, 3, 4\)"),
        (dict(extrinsics=extr, intrinsics=intr[:, :3]), r"has shape \(3, 3\); expected \(N, 4\)"),
        (dict(extrinsics=extr.astype(f32), intrinsics=intr), r"dtype '<f4'"),
        (dict(extrinsics=extr.astype(">f8"), intrinsics=intr), r"dtype '>f8'"),
        (dict(extrinsics=np.asfortranarray(extr), intrinsics=intr), "Fortran-order"),
        (dict(extrinsics=extr), "has no array 'intrinsics'"),
        (dict(extrinsics=extr[:2], intrinsics=intr[:2]), "has 2 cameras but .* has 3 depth files"),
        (dict(extrinsics=extr, intrinsics=intr[:2]), "has 3 extrinsics but 2 intrinsics"),
    ]
    for arrays, msg in cases:
        np.savez(npz, **arrays)
        v = _open(root)
        v.createDepthStream("colmap_dense", "depth_colmap_dense_imported", [-1, -1])
        with pytest.raises(RuntimeError, match=msg):
            lp.DepthVideoImporter.importColmapRecon(v, npz, 0, True)
        assert all(v.depthStream(0).frame(i)._enabled for i in range(N))   # nothing changed before the check
    with open(npz, "wb") as f:
        f.write(b"not a zip file at all, just some bytes")
    with pytest.raises(RuntimeError, match="not a readable .npz archive"):
        _recon(root, npz)
    with pytest.raises(RuntimeError, match="Could not open"):
        _recon(root, os.path.join(root, "missing.npz"))


def test_import_colmap_recon_rejects_badly_named_depth_files(tmp_path):
    root = str(tmp_path / "v")
    extr, intr, _ = _recon_scene(root, [0, 1])
    npz = os.path.join(root, "metadata.npz")
    np.savez(npz, extrinsics=extr, intrinsics=intr)
    _recon(root, npz)
    dd = os.path.join(root, "depth_colmap_dense_imported", "depth")
    for bad in ("frame_1.raw", "image_000002.raw", "frame_00000x.raw"):
        synthetic_files.write_raw(os.path.join(dd, bad), np.full((H, W), 0.5, f32))
        with pytest.raises(RuntimeError, match="does not have the expected format"):
            _recon(root, npz)
        os.remove(os.path.join(dd, bad))
