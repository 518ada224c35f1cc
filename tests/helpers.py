"""Shared builders for the parity tests: the same seeded problem is handed to the CPU oracle
(oracle/) and to the CUDA path (robust_cvd_b200.solver) through identical array-level calls."""
import numpy as np

from robust_cvd_b200 import abi, synthetic

# (name, config overrides) -- transform / intrinsics / loss variants of the reference
VARIANTS = [
    ("bilinear_perframe_disp", dict(depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=4)),
    ("global_perframe_disp", dict(depth_type=abi.DEPTH_GLOBAL)),
    ("bicubic_shared_ratio_bicubicwarp", dict(depth_type=abi.DEPTH_GRID, depth_cubic=1, depth_grid_x=5, depth_grid_y=4,
                                              spatial_type=abi.SPATIAL_BICUBIC_GRID, spatial_grid_x=4, spatial_grid_y=3,
                                              intr_opt=abi.INTR_SHARED, static_loss_type=abi.LOSS_REPRO_DEPTH_RATIO)),
    ("global_fixed_log_bilinearwarp", dict(depth_type=abi.DEPTH_GLOBAL, spatial_type=abi.SPATIAL_BILINEAR_GRID, spatial_grid_x=3,
                                           spatial_grid_y=2, intr_opt=abi.INTR_FIXED, static_loss_type=abi.LOSS_REPRO_LOG_DEPTH)),
    ("bicubic_scaleshift_euclid_corners", dict(depth_type=abi.DEPTH_GRID, depth_cubic=1, value_xform=abi.VALUE_SCALESHIFT,
                                               depth_grid_x=4, depth_grid_y=3, spatial_type=abi.SPATIAL_CORNERS_BILINEAR,
                                               static_loss_type=abi.LOSS_EUCLIDEAN, position_reg=0.3)),
    ("bilinear_vertical_huber", dict(depth_type=abi.DEPTH_GRID, depth_grid_x=6, depth_grid_y=4, spatial_type=abi.SPATIAL_VERTICAL_LINEAR,
                                     robust_type=abi.ROBUST_HUBER, robustness=0.05)),
    ("identitydepth_fixposes", dict(depth_type=abi.DEPTH_IDENTITY, fix_poses=1)),
    ("bilinear_fixedintr_ratio", dict(depth_type=abi.DEPTH_GRID, depth_grid_x=5, depth_grid_y=3, intr_opt=abi.INTR_FIXED,
                                      static_loss_type=abi.LOSS_REPRO_DEPTH_RATIO)),
    ("global_euclid", dict(depth_type=abi.DEPTH_GLOBAL, static_loss_type=abi.LOSS_EUCLIDEAN)),
    ("identitydepth_perframe", dict(depth_type=abi.DEPTH_IDENTITY)),
]


def make_case(num_frames=8, w=128, h=96, seed=1, sep=10, perturb=0.01, start="gt", **overrides):
    sc = synthetic.Scene(num_frames, w, h, seed=seed)
    cfg = abi.default_config(num_frames, sc.aspect, **overrides)
    pairs, offs, rec = sc.constraints(sep=sep)
    med = sc.median_depths()
    return sc, cfg, pairs, offs, rec, med


def initial_state(sc, cfg, stride, off_depth, nd, seed=0, perturb=0.01, start="gt"):
    k = 2 if cfg.value_xform == abi.VALUE_SCALESHIFT else 1
    if start == "gt":
        x = sc.gt_state(stride, off_depth, nd)
        if k == 2:
            x[:, off_depth + 1:off_depth + nd:2] = 0.0
    else:
        x = sc.identity_state(stride, off_depth, nd, k)
    rng = np.random.default_rng(seed)
    x = x + rng.normal(0, perturb, x.shape)
    return x


def layout_numbers(cfg):
    k = 2 if cfg.value_xform == abi.VALUE_SCALESHIFT else 1
    G = {abi.DEPTH_IDENTITY: 0, abi.DEPTH_GLOBAL: 1}.get(cfg.depth_type, cfg.depth_grid_x * cfg.depth_grid_y)
    return 7, G * k


def setup_problem(P, cfg, pairs, offs, rec, med, x, adaptive=None):
    P.set_frames(np.ones(cfg.num_frames, np.uint8), med, adaptive)
    P.set_constraints(pairs, offs, rec)
    P.set_state(x)
    return P


def write_masked_scene(root):
    """8-frame 128x96 synthetic scene directory with one dynamic blob per frame (0 = dynamic, 255 = static) so that the static flag
    matters; the scene of tests/test_host.py and of the recorded pose_optimization.py trace (tests/golden/make_golden.py)."""
    from robust_cvd_b200 import synthetic, synthetic_files
    sc = synthetic.Scene(8, 128, 96, seed=3)
    rng = np.random.default_rng(5)
    masks = []
    for i in range(sc.N):
        m = np.full((96, 128), 255, np.uint8); cx, cy = rng.integers(30, 100), rng.integers(30, 70); m[cy - 8:cy + 8, cx - 10:cx + 10] = 0; masks.append(m)
    pairs = synthetic_files.write_scene(sc, root, dynamic_masks=masks)
    return sc, pairs, masks
