"""CPU restatement of the pairwise depth-normalisation rows (normalizeDepth with normalizeDepthFromFirstFrame = false, reference
lib/PoseOptimizer.cpp:1005-1095): one DisparityDissimilarityCost residual (:425-462) per constraint record,

    r = 1 / max(xform_a(d_a), 1e-6) - 1 / max(xform_b(d_b), 1e-6),   robustified by the config's loss (the reference: CauchyLoss),

evaluated two independent ways: literally on a forward-mode Jet with 4 derivative lanes in ceil(P / 4) passes (what
ceres::DynamicAutoDiffCostFunction<., 4> does), and with the closed-form Jacobian.  The depth gathers are the oracle's
(oracle.gather_depth), so both frames' transforms are the reference's Identity / Global / bilinear / Catmull-Rom grids with Scale or
ScaleShift.  `solve` minimises this family plus the oracle's regulariser rows under the normalisation's lower bound: the reference
minimum the device solve is compared against.  Test infrastructure only; dense matrices, small problems."""
import ctypes as C

import numpy as np

from oracle import oracle
from robust_cvd_b200 import abi

EPS = 1e-6


class Jet:
    """ceres::Jet<double, 4>: value a, derivative lanes v."""
    __slots__ = ("a", "v")

    def __init__(self, a, v=None):
        self.a = float(a)
        self.v = np.zeros(4) if v is None else v

    def __add__(self, o):
        return Jet(self.a + o.a, self.v + o.v) if isinstance(o, Jet) else Jet(self.a + o, self.v.copy())

    __radd__ = __add__

    def __sub__(self, o):
        return Jet(self.a - o.a, self.v - o.v)

    def __mul__(self, o):
        return Jet(self.a * o.a, self.a * o.v + o.a * self.v) if isinstance(o, Jet) else Jet(self.a * o, self.v * o)

    __rmul__ = __mul__

    def __rtruediv__(self, s):          # s / Jet
        return Jet(s / self.a, -s * self.v / (self.a * self.a))

    def __lt__(self, o):
        return self.a < (o.a if isinstance(o, Jet) else o)


def jet_max(f, g):
    """ceres max(Jet, Jet): (f < g) ? g : f."""
    return g if f < g else f


def robust(cfg, s):
    """rho(s), rho'(s) of the config's loss (ceres/loss_function.cc)."""
    if cfg.robust_type == abi.ROBUST_CAUCHY:
        b = cfg.robustness ** 2
        return b * np.log1p(s / b), np.maximum(np.finfo(np.float64).tiny, 1.0 / (1.0 + s / b))
    if cfg.robust_type == abi.ROBUST_HUBER:
        a = cfg.robustness; b = a * a
        big = s > b; rr = np.sqrt(np.where(big, s, 1.0))
        return np.where(big, 2 * a * rr - b, s), np.where(big, np.maximum(np.finfo(np.float64).tiny, a / rr), 1.0)
    return s, np.ones_like(s)


def frame_stride(cfg):
    return oracle.lib().orc_frame_stride(C.byref(cfg))


class DepthPairs:
    def __init__(self, cfg, pair_frames, offsets, records):
        self.cfg = cfg
        self.N, self.stride = cfg.num_frames, frame_stride(cfg)
        self.U = self.N * self.stride
        self.k = 2 if cfg.value_xform == abi.VALUE_SCALESHIFT else 1
        pf = np.asarray(pair_frames, np.int64).reshape(-1, 2); off = np.asarray(offsets, np.int64)
        self.rec = np.asarray(records, np.float32).reshape(-1, 6)
        self.frames = np.repeat(pf, np.diff(off), axis=0)            # [C, 2]
        # per constraint and end: (parameter index, d D / d parameter without the value transform's src factor, src factor flag)
        self.cols = []
        for c in range(self.rec.shape[0]):
            ends = []
            for s in range(2):
                idx, w = ([], []) if cfg.depth_type == abi.DEPTH_IDENTITY else oracle.gather_depth(cfg, float(self.rec[c, 3 * s]), float(self.rec[c, 3 * s + 1]))
                ends.append((np.asarray(idx, np.int64), np.asarray(w, np.float64)))
            self.cols.append(ends)

    def _depth_params(self, x, c, s):
        """The end's parameter indices in node order: scale (and shift) of every gathered node."""
        idx, w = self.cols[c][s]
        base = int(self.frames[c, s]) * self.stride + 7
        return [(base + i * self.k + j, wi, j) for i, wi in zip(idx, w) for j in range(self.k)]

    def rows(self, x, jet=False):
        """Unrobustified residuals r [C] and Jacobian J [C, U]."""
        x = np.asarray(x, np.float64).reshape(-1)
        n = self.rec.shape[0]
        r = np.zeros(n); J = np.zeros((n, self.U))
        for c in range(n):
            params = [self._depth_params(x, c, 0), self._depth_params(x, c, 1)]
            src = [float(self.rec[c, 2]), float(self.rec[c, 5])]
            if jet:
                flat = [(s, p) for s in range(2) for p in params[s]]
                for p0 in range(0, max(len(flat), 1), 4):     # ceil(P / 4) passes, the last also when P = 0
                    lanes = {flat[i][1][0]: i - p0 for i in range(p0, min(p0 + 4, len(flat)))}

                    def functor(s):   # GridDepthFunctor / GlobalDepthFunctor: sum_i (src * s_i (+ o_i)) * w_i in node order
                        if self.cfg.depth_type == abi.DEPTH_IDENTITY:
                            return Jet(src[s])
                        D = Jet(0.0); ps = params[s]
                        for q in range(0, len(ps), self.k):
                            def var(t):
                                v = np.zeros(4)
                                if ps[q + t][0] in lanes:
                                    v[lanes[ps[q + t][0]]] = 1.0
                                return Jet(x[ps[q + t][0]], v)
                            val = var(0) * src[s]
                            if self.k == 2:
                                val = val + var(1)
                            D = D + val * ps[q][1]
                        return D
                    res = 1.0 / jet_max(functor(0), Jet(EPS)) - 1.0 / jet_max(functor(1), Jet(EPS))
                    r[c] = res.a
                    for pi, lane in lanes.items():
                        J[c, pi] += res.v[lane]
            else:
                D = []
                for s in range(2):
                    ps = params[s]
                    if self.cfg.depth_type == abi.DEPTH_IDENTITY:
                        D.append(src[s]); continue
                    D.append(sum((src[s] * x[ps[q][0]] + (x[ps[q + 1][0]] if self.k == 2 else 0.0)) * ps[q][1] for q in range(0, len(ps), self.k)))
                r[c] = 1.0 / max(D[0], EPS) - 1.0 / max(D[1], EPS)
                for s, sign in ((0, -1.0), (1, 1.0)):
                    if D[s] < EPS:
                        continue                               # the max's constant branch
                    dD = sign / (D[s] * D[s])
                    for pi, w, j in params[s]:
                        J[c, pi] += dD * w * (src[s] if j == 0 else 1.0)
        return r, J

    def evaluate(self, x, jet=False):
        """Robustified cost 1/2 sum rho(r^2), gradient J^T r and Gauss-Newton J^T J with the sqrt(rho') corrector."""
        r, J = self.rows(x, jet)
        rho0, rho1 = robust(self.cfg, r * r)
        sc = np.sqrt(rho1)
        Js = J * sc[:, None]
        return 0.5 * rho0.sum(), Js.T @ (r * sc), Js.T @ Js


def regulariser_problem(cfg, in_range, median):
    """The oracle holding the regulariser rows of cfg (no static constraints)."""
    O = oracle.OracleProblem(cfg)
    O.set_frames(in_range, median)
    O.set_constraints(np.zeros((0, 2), np.int32), np.zeros(1, np.int64), np.zeros((0, 6), np.float32))
    return O


def total(O, ref, x):
    O.set_state(x)
    co, go = O.evaluate(True)
    H = O.normal_matrix_dense()
    cp, gp, Hp = ref.evaluate(x)
    return co + cp, go + gp, H + Hp


def lower_bounded(cfg, in_range):
    """Parameters under the normalisation's lower bound 0: parameter 0 of every depth node block of the in-range frames (:1108-1115)."""
    stride = frame_stride(cfg); k = 2 if cfg.value_xform == abi.VALUE_SCALESHIFT else 1
    m = np.zeros((cfg.num_frames, stride), bool)
    if cfg.depth_lower_bound:   # the depth block is [7, 7 + nd), spatial parameters follow
        nd = {abi.DEPTH_IDENTITY: 0, abi.DEPTH_GLOBAL: 1}.get(cfg.depth_type, cfg.depth_grid_x * cfg.depth_grid_y) * k
        m[np.asarray(in_range, bool), 7:7 + nd:k] = True
    return m.reshape(-1)


def solve(O, ref, x0, bounded, iters=1000, tol=1e-14):
    """Projected Levenberg-Marquardt on the Gauss-Newton model to a tight stationary point of the bounded problem: the reference
    minimum (not a restatement of the device's iteration)."""
    x = np.where(bounded, np.maximum(x0.reshape(-1), 0.0), x0.reshape(-1)).astype(np.float64)
    lam = 1e-6
    c, g, H = total(O, ref, x)
    for _ in range(iters):
        proj = x - np.where(bounded, np.maximum(x - g, 0.0), x - g)
        if np.abs(proj).max() <= tol * max(1.0, np.abs(g).max()):
            break
        free = (np.diag(H) > 0) & ~(bounded & (x <= 0.0) & (g > 0.0))
        Hf = H[np.ix_(free, free)]
        while True:
            d = np.zeros_like(x)
            d[free] = np.linalg.solve(Hf + lam * np.diag(np.diag(Hf)), -g[free])
            xt = x + d
            xt = np.where(bounded, np.maximum(xt, 0.0), xt)
            ct, gt, Ht = total(O, ref, xt)
            if ct <= c:
                step = np.abs(xt - x).max()
                x, c, g, H = xt, ct, gt, Ht
                lam = max(lam / 10.0, 1e-12)
                break
            lam *= 10.0
            if lam > 1e12:
                return x
        if step <= 1e-15 * max(1.0, np.abs(x).max()):
            break
    return x
