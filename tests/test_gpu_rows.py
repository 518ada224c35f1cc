"""Per-block residual rows on the H100 (rcvd_row_layout / rcvd_evaluate_rows, the counterpart of ceres::Problem::Evaluate).

Every family is pinned row by row against a CPU restatement of the same rows: the static pairs against the oracle's
orc_static_jacobian, the smoothness triplets against orc_triplet_jacobian, the regulariser rows against orc_regulariser_jacobian and the
depth-normalisation pairs against tests/depth_pairs_ref.py.  The GPU's (cols, J) are scattered into a dense matrix and compared with the
restatement's, whose columns of constant parameters are zeroed (the GPU leaves them out, as the gradient does).  Then the rows must add up
to what rcvd_evaluate returns: 1/2 sum rho is the cost and sum rho'(s) J^T r the gradient, on the small cases and at config-2 size."""
import numpy as np
import pytest

from robust_cvd_b200 import abi
from tests import depth_pairs_ref as R
from tests import helpers

pytestmark = pytest.mark.gpu


def _take(offs, rec, sel):
    """The groups `sel` of a record family: (offsets, records)."""
    offs = np.asarray(offs, np.int64)
    parts = [rec[offs[g]:offs[g + 1]] for g in sel]
    counts = [len(p) for p in parts]
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64), np.concatenate(parts) if parts else rec[:0]


def _constant(cfg, stride):
    """Per global column: the parameter is held constant."""
    from robust_cvd_b200 import solver
    offS = solver.spatial_param_offset(cfg)
    c = np.zeros(stride, bool)
    c[:6] = bool(cfg.fix_poses); c[6] = cfg.intr_opt == abi.INTR_FIXED
    c[7:offS] = bool(cfg.fix_depth_xforms); c[offS:] = bool(cfg.fix_spatial_xforms)
    return np.tile(c, cfg.num_frames)


def _dense(cols, J, U):
    """(cols, J) [n, m, k] -> J [n * m, U]; checks the padding (-1 and 0, after the used slots) and that no column repeats in a row."""
    n, m, k = J.shape
    c = cols.reshape(n * m, k); v = J.reshape(n * m, k)
    used = c >= 0
    assert (v[~used] == 0).all()
    assert (used[:, 1:] <= used[:, :-1]).all()                 # the unused slots come last
    s = np.sort(np.where(used, c, -1 - np.arange(k)[None, :]), axis=1)
    assert (s[:, 1:] != s[:, :-1]).all()
    assert c.max(initial=-1) < U
    D = np.zeros((n * m, U))
    rr = np.repeat(np.arange(n * m), k).reshape(n * m, k)
    D[rr[used], c[used]] = v[used]
    return D


def _match(r, J, r_ref, J_ref, rho, rho_ref):
    r, r_ref = r.reshape(-1), r_ref.reshape(-1)
    assert r.shape == r_ref.shape and J.shape == J_ref.shape
    assert np.abs(r - r_ref).max(initial=0) <= 1e-10 * np.abs(r_ref).max(initial=0)
    assert np.abs(rho - rho_ref).max(initial=0) <= 1e-10 * np.abs(rho_ref).max(initial=0)
    if J.size:
        assert (np.abs(J - J_ref).max(axis=1) <= 1e-9 * np.abs(J_ref).max(axis=1)).all()


def _gradient(rows, rho_prime, U):
    """sum over blocks of rho'(s) J^T r."""
    g = np.zeros(U)
    for fam, (r, rho, cols, J) in rows.items():
        if r.size == 0:
            continue
        contrib = (rho_prime[fam][:, None, None] * J * r[:, :, None]).reshape(-1)
        c = cols.reshape(-1); ok = c >= 0
        g += np.bincount(c[ok], weights=contrib[ok], minlength=U)
    return g


def _consistent(G, rows, rho_prime):
    cg, gg = G.evaluate(True)
    cost = 0.5 * sum(rho.sum() for (_, rho, _, _) in rows.values())
    assert abs(cost - cg) <= 1e-11 * abs(cg), (cost, cg)
    g = _gradient(rows, rho_prime, G.U)
    assert np.abs(g - gg).max() <= 1e-9 * np.abs(gg).max()


def _check(overrides, num_frames=8, in_range=None, shuffle=False):
    from oracle import oracle
    from robust_cvd_b200 import solver
    sc, cfg, pairs, offs, rec, med = helpers.make_case(num_frames=num_frames, smooth_loss_type=1, **overrides)
    ce, to, tr = sc.triplets(sep=14)
    inr = np.ones(num_frames, np.uint8) if in_range is None else np.asarray(in_range, np.uint8)
    # the host passes only constraints whose frames are all in range
    keep = [i for i, (a, b) in enumerate(pairs) if inr[a] and inr[b]]
    offs, rec = _take(offs, rec, keep); pairs = np.asarray(pairs)[keep]
    keep_t = [i for i, c in enumerate(ce) if inr[c - 1] and inr[c] and inr[c + 1]]
    to, tr = _take(to, tr, keep_t); ce = np.asarray(ce)[keep_t]
    if shuffle:          # records of each pair in an order the run path's device sort changes
        rng = np.random.default_rng(11)
        rec = np.concatenate([rec[offs[i]:offs[i + 1]][rng.permutation(offs[i + 1] - offs[i])] for i in range(len(pairs))])
    dp_offs, dp_rec = _take(offs, rec, range(min(6, len(pairs)))); dp_pairs = pairs[:min(6, len(pairs))]
    off_d, nd = helpers.layout_numbers(cfg)
    O = oracle.OracleProblem(cfg); G = solver.Problem(cfg)
    x = helpers.initial_state(sc, cfg, G.stride, off_d, nd)
    for P in (O, G):
        P.set_frames(inr, med); P.set_constraints(pairs, offs, rec); P.set_triplets(ce, to, tr); P.set_state(x)
    G.set_depth_pairs(dp_pairs, dp_offs, dp_rec)
    U, const = G.U, _constant(cfg, G.stride)
    lay = G.row_layout()
    assert lay["pairs"]["blocks"] == rec.shape[0] and lay["triplets"]["blocks"] == tr.shape[0] and lay["depth_pairs"]["blocks"] == dp_rec.shape[0]
    assert (lay["pairs"]["residuals"], lay["triplets"]["residuals"], lay["depth_pairs"]["residuals"], lay["regularisers"]["residuals"]) == (3, 3, 1, 1)
    rows = {f: G.rows(f, jacobian=True) for f in abi.ROW_FAMILIES}
    for f, (r, rho, cols, J) in rows.items():
        assert r.shape == (lay[f]["blocks"], lay[f]["residuals"]) and cols.shape == J.shape == r.shape + (lay[f]["max_cols"],)
        r2, rho2 = G.rows(f)                                         # without the Jacobian: the same residuals
        assert np.abs(r2 - r).max(initial=0) <= 1e-13 * np.abs(r).max(initial=0) and np.abs(rho2 - rho).max(initial=0) <= 1e-13 * np.abs(rho).max(initial=0)

    ref = {}
    ro, Jo = O.static_jacobian()
    so = (ro.reshape(-1, 3) ** 2).sum(1)
    ref["pairs"] = (ro, Jo, R.robust(cfg, so)[0])
    rt, Jt = O.triplet_jacobian()
    w = tr[:, 9].astype(np.float64)
    ref["triplets"] = (rt, Jt, w * (rt.reshape(-1, 3) ** 2).sum(1))
    rd, Jd = R.DepthPairs(cfg, dp_pairs, dp_offs, dp_rec).rows(x)
    ref["depth_pairs"] = (rd, Jd, R.robust(cfg, rd * rd)[0])
    rg, Jg = O.regulariser_jacobian()
    ref["regularisers"] = (rg, Jg, rg * rg)
    for f in abi.ROW_FAMILIES:
        r, rho, cols, J = rows[f]
        r_ref, J_ref, rho_ref = ref[f]
        J_ref = np.where(const[None, :], 0.0, J_ref)
        _match(r, _dense(cols, J, U), r_ref, J_ref, rho, rho_ref)

    rho_prime = {"pairs": R.robust(cfg, (rows["pairs"][0] ** 2).sum(1))[1], "triplets": w,
                 "depth_pairs": R.robust(cfg, rows["depth_pairs"][0][:, 0] ** 2)[1], "regularisers": np.ones(lay["regularisers"]["blocks"])}
    _consistent(G, rows, rho_prime)
    return G, lay


@pytest.mark.parametrize("name,overrides", helpers.VARIANTS, ids=[v[0] for v in helpers.VARIANTS])
def test_rows_match_the_cpu_restatements(name, overrides):
    _check(overrides)


def test_run_path_returns_rows_in_the_callers_record_order():
    """bilinear grid, PerFrame focal, nothing fixed: the accumulate kernel's run path, which sorts each pair's records on the device."""
    _check(dict(helpers.VARIANTS)["bilinear_perframe_disp"], shuffle=True)


def test_fixed_poses_and_spatial_transforms():
    G, lay = _check(dict(depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=4, spatial_type=abi.SPATIAL_BILINEAR_GRID, spatial_grid_x=3,
                         spatial_grid_y=2, fix_poses=1, fix_spatial_xforms=1, position_reg=0.2))
    assert lay["pairs"]["max_cols"] == 2 * (1 + 4)          # PerFrame focal and the four depth nodes of each end


def test_frame_range_with_gaps():
    """Out-of-range frames have no regulariser rows; the position rows skip every triplet that reaches one."""
    inr = [0, 1, 1, 1, 0, 1, 1, 1, 1, 0]
    G, lay = _check(dict(depth_type=abi.DEPTH_GRID, depth_grid_x=4, depth_grid_y=3, position_reg=0.3), num_frames=10, in_range=inr)
    cfg = G.cfg
    per_frame = cfg.scale_grid_x * cfg.scale_grid_y + (3 * 3 + 4 * 2) + 1      # scale lattice, grid edges, focal (identity spatial)
    assert lay["regularisers"]["blocks"] == 7 * per_frame + 3 * 3             # triplets starting at frames 1, 5 and 6


def test_config2_rows_add_up_to_the_cost_and_gradient():
    """BASELINE config 2 (300 frames, 384x224, 16x12 bilinear grid, about 10^6 pair constraints): 1/2 sum rho is rcvd_evaluate's cost and
    sum rho'(s) J^T r its gradient; two calls return bit-identical arrays."""
    import bench
    from robust_cvd_b200 import solver
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case("config2_300f_384x224_grid16x12_sep10")
    G = solver.Problem(cfg)
    G.set_frames(np.ones(cfg.num_frames, np.uint8), med); G.set_constraints(pairs, offs, rec)
    G.set_state(bench.initial_state(sc, cfg, G.stride))
    assert rec.shape[0] > 500_000
    rows = {f: G.rows(f, jacobian=True) for f in abi.ROW_FAMILIES}
    rho_prime = {"pairs": R.robust(cfg, (rows["pairs"][0] ** 2).sum(1))[1], "triplets": np.zeros(0), "depth_pairs": np.zeros(0),
                 "regularisers": np.ones(rows["regularisers"][0].shape[0])}
    _consistent(G, rows, rho_prime)
    for f in ("pairs", "regularisers"):
        again = G.rows(f, jacobian=True)
        for a, b in zip(rows[f], again):
            assert np.array_equal(a, b), f
