"""Named edge cases of the residual and Jacobian evaluation, shared by tests/test_eval_edges_ref.py (the CPU oracle against its own
Jet autodiff and finite differences) and tests/test_gpu_eval_edges.py (the CUDA kernels against the oracle's Jet autodiff).

helpers.make_case builds an interior problem: ground-truth poses plus 0.01 noise, records inside smooth cells.  Every case here starts
from it and then overwrites records and state so that the evaluation takes a branch the interior never reaches:
  rotations  angle-axis exactly 0, |w| = 1e-9, theta^2 within ulps of DBL_EPSILON (ceres::AngleAxisRotatePoint's small-angle branch
             switch, theta^2 > DBL_EPSILON), |w| = 3 near pi -- on every frame, so at both ends of every pair and all three frames of
             every triplet
  locations  ndc coordinates exactly -1 and +1 (the clamp of the cell coordinate to nextafter(g - 1, 0)), exactly on the interior grid
             lines and one float32 ulp either side, on 2 x 2, 3 x 3 and 4 x 3 depth grids (bilinear and bicubic: grids of 2 and 3
             nodes make the bicubic tap folding at ix == 0 and ix == g - 2 coincide or touch) and on the spatial transforms
  depths     the transformed target depth B below the 1e-6 clamp, and source depths negated so that the point lies behind the
             receiving camera (A < 0): for the disparity, depth-ratio and log-depth losses.  log(min / max) of a negative ratio is
             NaN: those cases carry non-finite residuals
  robust     Huber with records on both sides of its threshold, Cauchy far out in its tail
  groups     pairs of 0, 1, 31, 32, 33, 127, 128, 129, 255, 256 and 257 records (warp, tile and empty boundaries of the tensor-core
             pair kernels), pairs whose records all share one cell pair (one run through warps and tiles), and pairs whose records
             alternate between two cells (the run path's device sort reorders them)
build(name) returns (cfg, pairs, offs, rec, med, x, triplets), triplets = (centres, offsets, records)."""
import numpy as np

from robust_cvd_b200 import abi
from tests import helpers

F32 = np.float32
NUM_FRAMES, W, H, SEP = 4, 64, 48, 4
LOSSES = {"disparity": abi.LOSS_REPRO_DISPARITY, "ratio": abi.LOSS_REPRO_DEPTH_RATIO, "log": abi.LOSS_REPRO_LOG_DEPTH}
SMOOTH_OF_LOSS = {abi.LOSS_REPRO_DISPARITY: 1, abi.LOSS_REPRO_DEPTH_RATIO: 2, abi.LOSS_REPRO_LOG_DEPTH: 3}
GRID = dict(depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=3)          # the tensor-core kernels' configuration
GROUP_COUNTS = [0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 64]

_LOCATIONS = {f"loc_depth_{'bicubic' if cubic else 'bilinear'}_{gx}x{gy}": dict(depth_type=abi.DEPTH_GRID, depth_cubic=cubic, depth_grid_x=gx, depth_grid_y=gy)
              for cubic in (0, 1) for gx, gy in ((2, 2), (3, 3), (4, 3))}
_LOCATIONS.update({
    f"loc_spatial_{kind}_{gx}x{gy}": dict(spatial_type=t, spatial_grid_x=gx, spatial_grid_y=gy)
    for kind, t in (("bilinear", abi.SPATIAL_BILINEAR_GRID), ("bicubic", abi.SPATIAL_BICUBIC_GRID)) for gx, gy in ((2, 2), (3, 2))})
_LOCATIONS.update({"loc_spatial_corners": dict(spatial_type=abi.SPATIAL_CORNERS_BILINEAR),
                   "loc_spatial_vertical": dict(spatial_type=abi.SPATIAL_VERTICAL_LINEAR)})

ROTATIONS = ["rot_zero", "rot_tiny", "rot_threshold", "rot_large"]
LOCATIONS = list(_LOCATIONS)
DEPTHS = [f"{loss}_{what}" for loss in LOSSES for what in ("clamp", "behind")]
ROBUST = ["huber_both_sides", "cauchy_tail"]
GROUPS = ["groups_sizes", "groups_one_run", "groups_alternating"]
CASES = ROTATIONS + LOCATIONS + DEPTHS + ROBUST + GROUPS
NONFINITE = ["log_behind"]          # the cases whose residuals are not all finite


def overrides(name):
    """Config overrides of case `name` (on top of abi.default_config)."""
    if name in _LOCATIONS:
        return dict(_LOCATIONS[name], smooth_loss_type=1)
    if name in DEPTHS:
        loss = LOSSES[name.split("_")[0]]
        return dict(GRID, static_loss_type=loss, smooth_loss_type=SMOOTH_OF_LOSS[loss])
    if name == "huber_both_sides":
        return dict(GRID, robust_type=abi.ROBUST_HUBER, smooth_loss_type=1)
    if name == "cauchy_tail":
        return dict(GRID, robustness=0.01, smooth_loss_type=1)
    assert name in CASES, name
    return dict(GRID, smooth_loss_type=1)


def axis_values(cfg):
    """ndc values that put a record on an edge of cfg's gathers: the borders -1 and +1 and one float32 ulp inside them, the interior
    grid lines of the depth and spatial grids and one float32 ulp either side of each, and 0 (the middle of the corner and vertical
    transforms).  (x values, y values)."""
    def lines(g):
        out = []
        for i in range(1, g - 1):
            v = F32(-1.0 + 2.0 * i / (g - 1))
            out += [np.nextafter(v, F32(-2)), v, np.nextafter(v, F32(2))]
        return out
    xs = [F32(-1), np.nextafter(F32(-1), F32(0)), F32(0), np.nextafter(F32(1), F32(0)), F32(1)]
    ys = list(xs)
    if cfg.depth_type == abi.DEPTH_GRID:
        xs += lines(cfg.depth_grid_x); ys += lines(cfg.depth_grid_y)
    if cfg.spatial_type in (abi.SPATIAL_BILINEAR_GRID, abi.SPATIAL_BICUBIC_GRID):
        xs += lines(cfg.spatial_grid_x); ys += lines(cfg.spatial_grid_y)
    return np.unique(np.asarray(xs, F32)), np.unique(np.asarray(ys, F32))


def edge_locations(n, xs, ys, salt):
    """(x, y) of n records from the edge values: along the records every x value meets every y value."""
    k = np.arange(n) * 7 + salt
    return xs[k % len(xs)], ys[(k // len(xs)) % len(ys)]


def rotation_state(name, x):
    """Angle-axis of every frame for the rotation cases (in place)."""
    n = x.shape[0]
    axes = np.eye(3)[np.arange(n) % 3]
    if name == "rot_zero":
        x[:, 3:6] = 0.0
    elif name == "rot_tiny":
        d = np.random.default_rng(4).normal(size=(n, 3))
        x[:, 3:6] = 1e-9 * d / np.linalg.norm(d, axis=1, keepdims=True)
    elif name == "rot_threshold":
        # one axis component a per frame, a = 2^-26 moved by k ulps: theta^2 = a * a is DBL_EPSILON (k = 0, the small-angle branch:
        # the test is theta^2 > DBL_EPSILON) or k * 2 ulps of it above or below
        for f in range(n):
            k = (-1, 0, 1, 2, -2, 3)[f % 6]
            a = 2.0 ** -26
            for _ in range(abs(k)):
                a = np.nextafter(a, np.inf if k > 0 else 0.0)
            x[f, 3:6] = axes[f] * a
            t2 = x[f, 3] * x[f, 3] + x[f, 4] * x[f, 4] + x[f, 5] * x[f, 5]
            assert (t2 > np.finfo(np.float64).eps) == (k > 0) and (t2 == np.finfo(np.float64).eps) == (k == 0)
    elif name == "rot_large":
        # every camera turned by about 3 rad about nearly the same axis: relative rotations stay small, so the scene stays in front
        base = np.array([0.3, 0.9, 0.3]) / np.linalg.norm([0.3, 0.9, 0.3])
        x[:, 3:6] = 3.0 * base[None, :] + x[:, 3:6]
    return x


def build(name, num_frames=NUM_FRAMES):
    """(cfg, pairs, offs, rec, med, x, triplets) of case `name`."""
    ov = overrides(name)
    if name in GROUPS:
        # every ordered pair of frames, dense records (sep 2: about 500 per pair) cut to the group sizes
        all_pairs = [(a, b) for a in range(num_frames) for b in range(num_frames) if a != b]
        from robust_cvd_b200 import synthetic
        sc = synthetic.Scene(num_frames, W, H, seed=1)
        cfg = abi.default_config(num_frames, sc.aspect, **ov)
        pairs, offs, rec = sc.constraints(pairs=all_pairs, sep=2)
        med = sc.median_depths()
        parts = []
        for p in range(len(pairs)):
            n = GROUP_COUNTS[p % len(GROUP_COUNTS)]
            assert offs[p + 1] - offs[p] >= n
            parts.append(rec[offs[p]:offs[p] + n])
        offs = np.concatenate([[0], np.cumsum([len(q) for q in parts])]).astype(np.int64)
        rec = np.concatenate(parts).copy()
    else:
        sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=num_frames, w=W, h=H, sep=SEP, **ov)
        rec = rec.copy()
    centres, toffs, trec = sc.triplets(sep=SEP)
    trec = trec.copy()
    off_d, nd = helpers.layout_numbers(cfg)
    stride = frame_stride(cfg)
    x = helpers.initial_state(sc, cfg, stride, off_d, nd)
    n = rec.shape[0]
    if name in ROTATIONS:
        rotation_state(name, x)
    elif name in LOCATIONS:
        xs, ys = axis_values(cfg)
        rec[:, 0], rec[:, 1] = edge_locations(n, xs, ys, 0)
        rec[:, 3], rec[:, 4] = edge_locations(n, xs, ys, 3)
        for o in range(3):
            trec[:, 3 * o], trec[:, 3 * o + 1] = edge_locations(trec.shape[0], xs, ys, 5 * o + 1)
    elif name.endswith("_clamp"):
        rec[::11, 5] = F32(1e-8)                 # target depth times its scale: B far below the 1e-6 clamp
    elif name.endswith("_behind"):
        rec[::7, 2] = -rec[::7, 2]               # the point lies behind its own camera, so (nearly) behind the receiving one: A < 0
    elif name == "huber_both_sides":
        cfg.robustness = huber_threshold(cfg, pairs, offs, rec, med, x)
    elif name == "cauchy_tail":
        x = helpers.initial_state(sc, cfg, stride, off_d, nd, perturb=0.05)
    elif name == "groups_one_run":
        for c in (0, 3):                         # every record in cell 0 of the 4 x 3 grid, at both ends
            rec[:, c] = F32(-1.0) + (rec[:, c] + F32(1.0)) * F32(0.3)
            rec[:, c + 1] = F32(-1.0) + (rec[:, c + 1] + F32(1.0)) * F32(0.45)
    elif name == "groups_alternating":
        for c in (0, 3):                         # even records in cell 0, odd records in the last cell
            rec[:, c] = F32(-1.0) + (rec[:, c] + F32(1.0)) * F32(0.3)
            rec[:, c + 1] = F32(-1.0) + (rec[:, c + 1] + F32(1.0)) * F32(0.45)
            rec[1::2, c] = -rec[1::2, c]; rec[1::2, c + 1] = -rec[1::2, c + 1]
    return cfg, pairs, offs, rec, med, x, (centres, toffs, trec)


def huber_threshold(cfg, pairs, offs, rec, med, x):
    """The median squared static residual norm of the problem, as Huber's a = sqrt(b): half of the records lie beyond it."""
    from oracle import oracle
    O = oracle.OracleProblem(cfg)
    helpers.setup_problem(O, cfg, pairs, offs, rec, med, x)
    r, _ = O.static_jacobian(jac=False)
    return float(np.sqrt(np.median((r.reshape(-1, 3) ** 2).sum(1))))


def log_step_behind():
    """A finite log-depth problem whose first Levenberg-Marquardt steps drive points behind the receiving camera: every 211th record's
    source depth is scaled by 0.01, so its point sits just in front of the receiving camera (A small and positive) with a large log
    residual.  From this state (seed 0) the full step at the default initial radius 1e4, and the next ones down to radius 1e2, give
    non-finite candidate costs (found by restating the first step on the CPU oracle, tests/test_eval_edges_ref.py).
    (cfg, pairs, offs, rec, med, x)."""
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=NUM_FRAMES, w=W, h=H, sep=SEP, **overrides("log_clamp"))
    rec = rec.copy()
    rec[::211, 2] *= F32(0.01)
    x = helpers.initial_state(sc, cfg, frame_stride(cfg), *helpers.layout_numbers(cfg), seed=0)
    return cfg, pairs, offs, rec, med, x


def frame_stride(cfg):
    off_d, nd = helpers.layout_numbers(cfg)
    return off_d + nd + 2 * {abi.SPATIAL_IDENTITY: 0, abi.SPATIAL_VERTICAL_LINEAR: 2, abi.SPATIAL_CORNERS_BILINEAR: 4}.get(
        cfg.spatial_type, cfg.spatial_grid_x * cfg.spatial_grid_y)
