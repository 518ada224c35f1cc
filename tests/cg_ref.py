"""numpy restatement of the block-Jacobi preconditioned conjugate gradients of robust_cvd_b200/csrc/rcvd_cg.cuh (TEST INFRASTRUCTURE,
no GPU): Ceres' ConjugateGradientsSolver as LevenbergMarquardtStrategy drives it -- x0 = 0, q_tolerance eta, r_tolerance disabled,
min_num_iterations 0, max_num_iterations 500, residual_reset_period 10 -- with the frames' diagonal blocks of A as the preconditioner.
Where Ceres reports FAILURE or an indefinite matrix, and on a NaN in those scalars, the restatement reports a breakdown (the solver's
*fail flag)."""
import numpy as np

ETA = 0.1
MAX_ITERATIONS = 500
RESET_PERIOD = 10


def block_jacobi(A, nf):
    """z = M^-1 r with M the nf x nf diagonal blocks of A, by their Cholesky factors (as the solver applies L^-T L^-1)."""
    n = A.shape[0] // nf
    Ls = [np.linalg.cholesky(A[f * nf:(f + 1) * nf, f * nf:(f + 1) * nf]) for f in range(n)]

    def apply(r):
        z = np.empty_like(r)
        for f, L in enumerate(Ls):
            s = slice(f * nf, (f + 1) * nf)
            z[s] = np.linalg.solve(L.T, np.linalg.solve(L, r[s]))
        return z
    return apply


def pcg(A, b, nf, eta=ETA, max_iterations=MAX_ITERATIONS):
    """Solves A x = b.  Returns dict(x, iterations, capped, broke, zeta): zeta is the quadratic-model ratio i (Q_i - Q_i-1) / Q_i of
    every iteration run; the solve stops at the first below eta, or at max_iterations (capped: its iterate is the step)."""
    x = np.zeros_like(b)
    out = dict(x=x, iterations=0, capped=False, broke=False, zeta=[])
    if np.linalg.norm(b) == 0.0:
        return out
    precond = block_jacobi(A, nf)
    r = b.copy()
    rho, q0 = 1.0, 0.0                                  # Q(x0) = 0
    p = None
    for i in range(1, max_iterations + 1):
        out["iterations"] = i
        z = precond(r)
        last, rho = rho, float(r @ z)
        if rho == 0.0 or not np.isfinite(rho):
            out["broke"] = True
            return out
        if i == 1:
            p = z.copy()
        else:
            beta = rho / last
            if beta == 0.0 or not np.isfinite(beta):
                out["broke"] = True
                return out
            p = z + beta * p
        q = A @ p
        pq = float(p @ q)
        if not pq > 0.0 or np.isinf(pq):
            out["broke"] = True
            return out
        alpha = rho / pq
        if not np.isfinite(alpha):
            out["broke"] = True
            return out
        x = x + alpha * p
        r = b - A @ x if i % RESET_PERIOD == 0 else r - alpha * q
        q1 = -float(x @ (b + r))                         # Q(x) = x'Ax - 2 b'x = -x'(b + r)
        zeta = i * (q1 - q0) / q1
        out["zeta"].append(zeta)
        out["x"] = x
        if zeta < eta:
            return out
        q0 = q1
    out["capped"] = True
    return out


def spd_system(n, nf, pairs, cond_spread, seed=0):
    """(A, b): an SPD matrix on the frame graph (every block row of J touches one frame or one coupled pair) with column scales
    10^[-cond_spread/2, cond_spread/2], and a random right-hand side."""
    from tests import linalg_ref as R
    rng = np.random.default_rng(seed)
    H = R.normal_matrix(n, nf, pairs, rng)
    c = 10.0 ** rng.uniform(-cond_spread / 2, cond_spread / 2, size=n * nf)
    A = H * c[:, None] * c[None, :]
    return 0.5 * (A + A.T), rng.normal(size=n * nf)
