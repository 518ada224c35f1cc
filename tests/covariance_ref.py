"""Numpy restatement of rcvd_covariance (TEST INFRASTRUCTURE; robust_cvd_b200/csrc/rcvd_selinv.cuh): the Jacobi scaling with held
parameters, the pivots of the rank test and the block Takahashi recurrence of the selected inversion, on top of
tests/linalg_ref.block_cholesky and the solver's elimination order and levels (linalg_ref.elimination_order / levels restate
rcvd_plan.h; tests/test_covariance.py checks them against rcvd_debug_factor_plan).  Plain numpy, no GPU."""
import numpy as np
import scipy.linalg

from tests import linalg_ref as R


def scaled(H, hold):
    """(S, A): S = diag(H)^-1/2 on the free parameters, 0 on the held ones and where the diagonal is not positive; A = S H S + D2 with
    D2 = 1 on the held parameters (a decoupled unit pivot), 0 elsewhere."""
    hold = np.asarray(hold, bool)
    d = np.diag(H)
    S = np.where(~hold & (d > 0), 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 0.0)
    A = H * S[:, None] * S[None, :] + np.diag(hold.astype(np.float64))
    return S, A


def pivots(A, order, nf):
    """The pivots of the unblocked elimination of P A P^T (frames in `order`), i.e. the squared diagonal of its Cholesky factor where
    that exists, also past a non-positive pivot.  Returns [U] in elimination order."""
    M, _ = R.permute(A, order, nf)
    M = M.copy()
    d = np.zeros(M.shape[0])
    for j in range(M.shape[0]):
        d[j] = M[j, j]
        if d[j] != 0.0:
            M[j + 1:, j + 1:] -= np.outer(M[j + 1:, j], M[j, j + 1:]) / d[j]
    return d


def first_failing_pivot(A, hold, order, nf, min_pivot=1e-10):
    """(frame, parameter, pivot) of the first free parameter in elimination order whose pivot is <= min_pivot, or None."""
    d = pivots(A, order, nf)
    held = np.asarray(hold, bool)
    for q, f in enumerate(order):
        for i in range(nf):
            if not held[f * nf + i] and not d[q * nf + i] > min_pivot:
                return f, i, d[q * nf + i]
    return None


def selected_inverse(A, n, nf, pairs, slack=4):
    """The blocks of A^-1 on the filled pattern of the block Cholesky, by the recurrence of rcvd_selinv.cuh over the levels in reverse:
      Y_rk = sum_{j in S_k} Z_rj X_jk,  Z_rk = -Y_rk inv(L_kk),  Z_kk = inv(L_kk)^T (inv(L_kk) - sum_{j in S_k} X_jk^T Z_jk).
    Returns (Z, products): Z[(r, c)] with r eliminated after c (or r == c) the block of rows of frame r and columns of frame c;
    products = the block products of the first and third steps."""
    order, L = R.block_cholesky(A, n, nf, pairs, slack)
    _, cs = R.elimination_order(n, pairs, slack)
    lvl = R.levels(order, cs)
    pos = {k: q for q, k in enumerate(order)}
    blk = lambda f: slice(pos[f] * nf, (pos[f] + 1) * nf)
    Z = {}
    z = lambda r, j: Z[(r, j)] if r == j or pos[r] > pos[j] else Z[(j, r)].T
    products = 0
    for l in reversed(range(max(lvl.values()) + 1)):
        for k in [k for k in order if lvl[k] == l]:
            Li = scipy.linalg.solve_triangular(L[blk(k), blk(k)], np.eye(nf), lower=True)
            sk = cs[k]
            X = {j: L[blk(j), blk(k)] for j in sk}
            Y = {r: sum((z(r, j) @ X[j] for j in sk), np.zeros((nf, nf))) for r in sk}
            for r in sk:
                Z[(r, k)] = -Y[r] @ Li
            Z[(k, k)] = Li.T @ (Li - sum((X[j].T @ Z[(j, k)] for j in sk), np.zeros((nf, nf))))
            products += len(sk) * len(sk) + len(sk)
    return Z, products


def covariance(H, n, nf, pairs, hold, slack=4):
    """Cov = S (S H S + D2)^-1 S on the filled pattern: {(r, c): block} as selected_inverse, and its block products."""
    S, A = scaled(H, hold)
    Z, products = selected_inverse(A, n, nf, pairs, slack)
    return {(r, c): S[r * nf:(r + 1) * nf, None] * B * S[None, c * nf:(c + 1) * nf] for (r, c), B in Z.items()}, products


def reduced_inverse(H, hold):
    """The dense reference: the inverse of H restricted to the free parameters, zeros on the held rows and columns."""
    free = ~np.asarray(hold, bool)
    C = np.zeros_like(H)
    C[np.ix_(free, free)] = np.linalg.inv(H[np.ix_(free, free)])
    return C
