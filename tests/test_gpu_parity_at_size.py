"""Parity at the sizes bench.py times (VERDICT r1 item 1): the CUDA path against the CPU oracle on BASELINE config 2
(300 frames, 384x224, 16x12 bilinear grid, hierarchical2 pairs, matchSeparation 10: 43 elimination levels, ~2.1 k factor
blocks, two-stream factorisation graph) and on a 40-frame 32x24-grid problem that takes the large-block path (npad > 224:
panel/trailing potrf, inverse-times-block TRSM).  Reference semantics: lib/PoseOptimizer.cpp:954-987 (ceres::Solve + write-back).

Checks per case
  * cost and gradient vs the oracle, <= 1e-9 relative (observed ~1e-13);
  * device-side residual of the damped normal equations |(S H S + D2) y - S g| / |S g| < 1e-8, computed with the SpMV over the
    assembled H (independent of the factorisation kernels);
  * the linear solve against the oracle's block Cholesky on the same S, D2, b;
  * four (three at the large grid) LM iterations from radius 1 against the oracle: same accept/reject sequence, final cost <= 1e-9 relative, state <= 1e-7 relative.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _case(name, frames=None):
    import bench
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case(name, frames=frames)
    return spec, sc, cfg, pairs, offs, rec, med


def _both(cfg, pairs, offs, rec, med, x0):
    from robust_cvd_b200 import solver
    from oracle import oracle
    G = solver.Problem(cfg); O = oracle.OracleProblem(cfg)
    for P in (G, O):
        P.set_frames(np.ones(cfg.num_frames, np.uint8), med)
        P.set_constraints(pairs, offs, rec)
        P.set_state(x0)
    return G, O


def _check_case(name, frames, lm_iters=4):
    import bench
    from robust_cvd_b200 import abi
    spec, sc, cfg, pairs, offs, rec, med = _case(name, frames)
    G, O = None, None
    from robust_cvd_b200 import solver
    x0 = bench.initial_state(sc, cfg, solver.frame_stride(cfg))
    G, O = _both(cfg, pairs, offs, rec, med, x0)
    info = G.structure_info()
    # cost / gradient
    cg, gg = G.evaluate(True)
    co, go = O.evaluate(True)
    assert abs(cg - co) <= 1e-9 * abs(co), (cg, co)
    assert np.abs(gg - go).max() <= 1e-9 * np.abs(go).max(), np.abs(gg - go).max() / np.abs(go).max()
    # device-side residual of the damped system at two radii (the LM loop's first radius and a large one = weak damping)
    for radius in (1e4, 1e9):
        r = G.linear_residual(radius)
        assert r["pivot_fail"] == 0
        assert r["rel_residual"] < 1e-8, (radius, r)
        assert abs(r["cost"] - co) <= 1e-9 * abs(co)
        assert abs(r["grad_norm"] - np.linalg.norm(go)) <= 1e-9 * np.linalg.norm(go)
    # linear solve vs the oracle's block Cholesky on identical S, D2, b
    rng = np.random.default_rng(3)
    U = cfg.num_frames * G.stride
    S = 1.0 / (1.0 + rng.uniform(0.5, 50.0, U)); D2 = rng.uniform(1e-4, 1e-2, U); b = rng.normal(0, 1, U)
    O.time_iteration()                # assembles the oracle's H at the current state (block_solve factors the last assembled H)
    yg = G.debug_linear_solve(S, D2, b); yo = O.block_solve(S, D2, b)
    assert np.linalg.norm(yg - yo) <= 1e-9 * np.linalg.norm(yo), np.linalg.norm(yg - yo) / np.linalg.norm(yo)
    # a few LM iterations
    opt = abi.default_solve_options(max_iterations=lm_iters)
    opt.initial_radius = 1.0          # Ceres' default 1e4 spends the first five iterations shrinking the region at this start
    sg, so = G.solve(opt), O.solve(opt)
    assert sg.iterations == so.iterations and sg.num_successful_steps == so.num_successful_steps and so.num_successful_steps >= 3
    assert so.final_cost < 0.8 * so.initial_cost
    assert abs(sg.final_cost - so.final_cost) <= 1e-9 * abs(so.final_cost), (sg.final_cost, so.final_cost)
    xg, xo = G.get_state(), O.get_state()
    assert np.linalg.norm(xg - xo) <= 1e-7 * np.linalg.norm(xo), np.linalg.norm(xg - xo) / np.linalg.norm(xo)
    return info


def test_config2_300_frames_matches_oracle():
    info = _check_case("config2_300f_384x224_grid16x12_sep10", None)
    assert info["frames"] == 300 and info["npad"] == 208 and info["levels"] >= 30


def test_large_block_path_40_frames_grid32x24_matches_oracle():
    info = _check_case("config4_600f_640x384_grid32x24_sep10", 40, lm_iters=3)
    assert info["npad"] > 224
