"""Dense float64 / long-double reference of the block-sparse Cholesky (TEST INFRASTRUCTURE; checks the factorisation and solve
kernels of robust_cvd_b200/csrc/rcvd_linalg.cuh and rcvd_update.cuh through tests/test_gpu_linalg.py).  Plain numpy, no GPU.

- frame-graph builders (undirected frame pairs a < b);
- SPD matrices restricted to a frame graph (H = J^T J, every block row of J touches one frame or one coupled pair): well-conditioned
  with a manufactured solution, LM-like (gauge null direction, graded column scales, Jacobi scaling and trust-region damping), and a
  pivot-negating variant;
- backward-error metrics in units of u = 2^-53;
- a right-looking block Cholesky over the solver's elimination order and level schedule, with optional injected defects that each
  model a plausible kernel bug (tests/test_linalg_ref.py shows that the metrics catch every one of them)."""
import numpy as np
import scipy.linalg

U_ROUND = 2.0 ** -53

# thresholds of the kernel tests (units of u, except the forward error)
FACTOR_TOL = 64.0            # componentwise factor backward error
SOLVE_TOL = 32.0             # normwise solve backward error
LINV_TOL_PER_NF = 64.0       # Linv residual: 64 * nf
FORWARD_TOL = 1e-12          # forward error of the well-conditioned mode


# ---------------------------------------------------------------------------------------------------------
# frame graphs
# ---------------------------------------------------------------------------------------------------------
def chain(n):
    return [(i, i + 1) for i in range(n - 1)]


def star(n):
    return [(0, i) for i in range(1, n)]


def complete(n):
    return [(i, j) for i in range(n) for j in range(i + 1, n)]


def disconnected(n):
    """Two chains and a complete part over frames 0 .. n-2; frame n-1 is coupled to nothing."""
    a = max(2, (n - 1) // 3)
    b = max(a + 2, 2 * (n - 1) // 3)
    return [(i, i + 1) for i in range(a - 1)] + [(i, i + 1) for i in range(a, b - 1)] + complete_range(b, n - 1)


def complete_range(lo, hi):
    return [(i, j) for i in range(lo, hi) for j in range(i + 1, hi)]


def hierarchical2(n):
    from robust_cvd_b200 import synthetic
    return sorted({(min(a, b), max(a, b)) for a, b in synthetic.hierarchical2_pairs(n)})


GRAPHS = {"chain": chain, "star": star, "complete": complete, "disconnected": disconnected, "hierarchical2": hierarchical2}


def adjacency(n, pairs):
    adj = [set() for _ in range(n)]
    for a, b in pairs:
        if a != b:
            adj[a].add(b); adj[b].add(a)
    return adj


def elimination_order(n, pairs, slack=4):
    """The solver's multiple-minimum-degree order (robust_cvd_b200/csrc/rcvd_plan.h, make_factor_plan): each round eliminates a maximal
    independent set of frames whose degree is within `slack` of the minimum (slack < 0: one frame per round).  Returns (order, cs) with cs[k] the
    later-eliminated frames coupled to k after fill, sorted by elimination position."""
    adj = adjacency(n, pairs)
    done = [False] * n; order = []; pos = [-1] * n; cs = [[] for _ in range(n)]
    while len(order) < n:
        md = min(len(adj[f]) for f in range(n) if not done[f])
        lim = md + (slack if slack > 0 else 0)
        cand = sorted((f for f in range(n) if not done[f] and len(adj[f]) <= lim), key=lambda f: len(adj[f]))
        blocked = [False] * n; chosen = []
        for f in cand:
            if blocked[f]:
                continue
            chosen.append(f); blocked[f] = True
            for a in adj[f]:
                blocked[a] = True
            if slack < 0:
                break
        for k in chosen:
            done[k] = True; pos[k] = len(order); order.append(k)
            nb = sorted(adj[k]); cs[k] = nb
            for a in nb:
                adj[a].discard(k)
            for i in range(len(nb)):
                for j in range(i + 1, len(nb)):
                    adj[nb[i]].add(nb[j]); adj[nb[j]].add(nb[i])
    for f in range(n):
        cs[f].sort(key=lambda a: pos[a])
    return order, cs


def levels(order, cs):
    lvl = {k: 0 for k in order}
    for k in order:
        for a in cs[k]:
            lvl[a] = max(lvl[a], lvl[k] + 1)
    return lvl


def owners(order, cs, lvl, nranks):
    """The distributed factorisation's frame owners (rcvd_plan.h): (LB, owner).  Levels >= LB are the replicated tail of levels with
    fewer than 3 frames; LB = 0 means no distribution.  Owners are greedy LPT, level by level, over each column's incoming phase-A update
    work (symmetric targets count half) plus 0.6 per off-diagonal block + 0.3 for its own TRSM / POTRF in phase A."""
    nl = max(lvl.values()) + 1
    lf = [[k for k in order if lvl[k] == l] for l in range(nl)]
    LB = nl
    while LB > 0 and len(lf[LB - 1]) < 3:
        LB -= 1
    owner = [0] * len(order)
    if nranks < 2 or LB == 0:
        return 0, owner
    tot_in = [0.0] * len(order)
    for l in range(LB):
        for k in lf[l]:
            for a in range(len(cs[k])):
                for b in range(a + 1):
                    tot_in[cs[k][b]] += 0.5 if a == b else 1.0
    load = [0.0] * nranks
    for l in range(nl):
        w = {k: tot_in[k] + (0.6 * len(cs[k]) + 0.3 if l < LB else 0.0) for k in lf[l]}
        for k in sorted(lf[l], key=lambda k: -w[k]):
            q = min(range(nranks), key=lambda t: load[t])
            owner[k] = q
            load[q] += w[k]
    return LB, owner


# ---------------------------------------------------------------------------------------------------------
# SPD generators restricted to the frame graph
# ---------------------------------------------------------------------------------------------------------
def normal_matrix(n, nf, pairs, rng, gauge=False):
    """H = J^T J, accumulated block by block, for a J with one nf-row block row per frame and one per coupled pair (each touches only
    its frame / its two frames).  gauge: column 0 of every frame gets opposite coefficients in a pair row and zero in a frame row, so
    J v = 0 for v = sum_f e_(f, 0)."""
    H = np.zeros((n * nf, n * nf))
    s = lambda f: slice(f * nf, (f + 1) * nf)
    for f in range(n):
        B = rng.normal(size=(nf, nf)) + 2.0 * np.eye(nf)
        if gauge:
            B[:, 0] = 0.0
        H[s(f), s(f)] += B.T @ B
    for a, b in pairs:
        Ba, Bb = rng.normal(size=(nf, nf)), rng.normal(size=(nf, nf))
        if gauge:
            Bb[:, 0] = -Ba[:, 0]
        H[s(a), s(a)] += Ba.T @ Ba; H[s(b), s(b)] += Bb.T @ Bb
        H[s(a), s(b)] += Ba.T @ Bb; H[s(b), s(a)] += Bb.T @ Ba
    return 0.5 * (H + H.T)


def well_conditioned(n, nf, pairs, seed=0):
    """(A, D2, b, x*): A = J^T J + mu I with cond(A) <= ~1e2, D2 = 0, b = A x* computed in long double."""
    rng = np.random.default_rng(seed)
    H = normal_matrix(n, nf, pairs, rng)
    mu = np.abs(H).sum(1).max() / 100.0         # Gershgorin: lambda_max(H) <= max row sum, so cond(H + mu I) <= 101
    A = H + mu * np.eye(n * nf)
    A = 0.5 * (A + A.T)
    x = rng.normal(size=n * nf)
    xl = x.astype(np.longdouble)
    b = np.concatenate([(A[i:i + 512].astype(np.longdouble) @ xl).astype(np.float64) for i in range(0, n * nf, 512)])
    return A, np.zeros(n * nf), b, x


def lm_like(n, nf, pairs, radius, seed=0):
    """(Hs, D2, b): the damped system of one LM step.  J has a gauge null direction and column scales 10^[-4, 4]; Jacobi scaling
    S = 1 / (1 + sqrt(diag H)), Hs = S H S, D2 = clamp(S^2 diag H, 1e-6, 1e32) / radius (the solver's k_lm_prepare)."""
    rng = np.random.default_rng(seed)
    H = normal_matrix(n, nf, pairs, rng, gauge=True)
    c = 10.0 ** rng.uniform(-4, 4, size=n * nf)          # J <- J diag(c)
    H = H * c[:, None] * c[None, :]
    S =1.0 / (1.0 + np.sqrt(np.diag(H)))
    Hs = H * S[:, None] * S[None, :]
    D2 = np.clip(S * S * np.diag(H), 1e-6, 1e32) / radius
    return Hs, D2, rng.normal(size=n * nf)


def permute(A, order, nf):
    """P A P^T with the frames in elimination order."""
    idx = np.concatenate([np.arange(f * nf, (f + 1) * nf) for f in order])
    return A[np.ix_(idx, idx)], idx


def negate_pivot(A, order, nf, j, margin=0.5):
    """A copy of A whose pivot j of the factorisation of P A P^T (elimination order `order`) is -margin * d_j, d_j = L_jj^2: A_jj is
    lowered by (1 + margin) d_j, which leaves the pivots before j unchanged."""
    M, idx = permute(A, order, nf)
    d = np.linalg.cholesky(M)[j, j] ** 2
    out = A.copy()
    out[idx[j], idx[j]] -= (1.0 + margin) * d
    return out


# ---------------------------------------------------------------------------------------------------------
# metrics
# ---------------------------------------------------------------------------------------------------------
def factor_error(L, M, nf, order=None, lvl=None, inverse_tile=None):
    """Componentwise backward error max |L L^T - M| / (|L| |L|^T) over the lower triangle, in units of u, with the location of the
    worst entry: (row frame, column frame, 8x8 unit (i, j) inside the block, level of the column frame).  An entry whose denominator
    is 0 counts as infinite unless its residual is 0 too, and so does a NaN.  Evaluated block by block over the blocks of L L^T and M
    that can be non-zero, so that U = 8000 stays cheap.
    inverse_tile = None: the plain metric.  Otherwise the off-diagonal blocks' denominator also gets tile_inverse_bound(.., inverse_tile):
    the looser metric of a TRSM that multiplies by explicit inverses of inverse_tile x inverse_tile diagonal tiles."""
    n = L.shape[0] // nf
    nzL = np.abs(L).reshape(n, nf, n, nf).sum(axis=(1, 3)) != 0
    nzM = np.abs(M).reshape(n, nf, n, nf).sum(axis=(1, 3)) != 0
    cols = [set(np.nonzero(nzL[i, :i + 1])[0]) for i in range(n)]
    best, where = -1.0, None
    for i in range(n):
        for j in range(i + 1):
            ks = sorted(cols[i] & cols[j])
            if not ks and not nzM[i, j]:
                continue
            idx = np.concatenate([np.arange(k * nf, (k + 1) * nf) for k in ks]) if ks else np.zeros(0, int)
            Li, Lj = L[i * nf:(i + 1) * nf][:, idx], L[j * nf:(j + 1) * nf][:, idx]
            R = Li @ Lj.T - M[i * nf:(i + 1) * nf, j * nf:(j + 1) * nf]
            D = np.abs(Li) @ np.abs(Lj).T
            if i == j:
                R, D = np.tril(R), np.tril(D)
            elif inverse_tile is not None:
                D = D + tile_inverse_bound(L[i * nf:(i + 1) * nf, j * nf:(j + 1) * nf], L[j * nf:(j + 1) * nf, j * nf:(j + 1) * nf], inverse_tile)
            with np.errstate(divide="ignore", invalid="ignore"):
                E = np.where(D > 0, np.abs(R) / D, np.where(R != 0, np.inf, 0.0))
            E[np.isnan(E)] = np.inf
            a, b = np.unravel_index(int(np.argmax(E)), E.shape)
            if E[a, b] > best:
                best = float(E[a, b])
                where = (order[i] if order is not None else i, order[j] if order is not None else j, (a // 8, b // 8),
                         None if lvl is None or order is None else lvl[order[j]])
    return best / U_ROUND, where


def trsm_inverse_tile(npad, nf):
    """Size of the explicit inverses the off-diagonal TRSM of this block size multiplies by: k_trsm_ll (npad <= 416) uses the 16x16
    diagonal-tile inverses of k_potrf_*, the k_gemm_nt TRSM (npad >= 432) the whole inverse of L_kk from k_trinv."""
    return 16 if npad <= 416 else nf


def tile_inverse_bound(X, Ljj, tile):
    """The TRSM kernels form X[:, t] = T[:, t] Di_t^T with the explicit inverse Di_t of a diagonal tile D_t of L_jj (16x16 in k_trsm_ll,
    the whole block in the k_gemm_nt TRSM), not by substitution.  Each X entry is a tile-long dot product with Di_t, and Di_t's columns
    come from tile-long forward substitutions, so |X D_t^T - T| <= 2 gamma_tile |T| |Di_t|^T |D_t|^T (T = X D_t^T): relative to
    |X| |D_t|^T this grows with the componentwise condition number of the tile, which the LM damping makes large.  Returns
    |T| |Di_t|^T |D_t|^T per column tile, the extra denominator of the off-diagonal entries of factor_error.  (The panel solve of
    k_potrf_panel also multiplies by 16x16 tile inverses, but inside diagonal blocks, which this term does not loosen.)"""
    out = np.zeros_like(X)
    for t in range(0, Ljj.shape[0], tile):
        s = slice(t, min(t + tile, Ljj.shape[0]))
        Dt = Ljj[s, s]
        if not np.all(np.diag(Dt) > 0):
            continue
        Di = scipy.linalg.solve_triangular(Dt, np.eye(Dt.shape[0]), lower=True)
        out[:, s] = np.abs(X[:, s] @ Dt.T) @ np.abs(Di).T @ np.abs(Dt).T
    return out


def solve_error(A, y, b):
    """Normwise backward error |b - A y|_inf / (|A|_inf |y|_inf + |b|_inf) in units of u; the residual in long double."""
    yl = y.astype(np.longdouble)
    r = max(float(np.abs(b[i:i + 512].astype(np.longdouble) - A[i:i + 512].astype(np.longdouble) @ yl).max()) for i in range(0, len(b), 512))
    den = np.abs(A).sum(1).max() * np.abs(y).max() + np.abs(b).max()
    return r / den / U_ROUND


def linv_error(X, Lkk):
    """max |X L_kk - I| / (|X| |L_kk|) in units of u."""
    R = X @ Lkk - np.eye(Lkk.shape[0])
    D = np.abs(X) @ np.abs(Lkk)
    with np.errstate(divide="ignore", invalid="ignore"):
        E = np.where(D > 0, np.abs(R) / D, np.where(R != 0, np.inf, 0.0))
    return float(E.max() / U_ROUND)


def forward_error(y, x):
    return float(np.abs(y - x).max() / np.abs(x).max())


# ---------------------------------------------------------------------------------------------------------
# block Cholesky with injected defects
# ---------------------------------------------------------------------------------------------------------
DEFECTS = ("drop_pair", "drop_k_tail", "skip_warp_tile", "skip_diag_split", "perturb_pivot", "stale_u2")


def block_cholesky(A, n, nf, pairs, slack=4, defect=None):
    """Right-looking block Cholesky of P A P^T over the solver's elimination order, level by level as enqueue_factor_solve runs it:
    potrf + TRSM of every frame of a level, then every target A_rc -= sum_k X_rk X_ck^T over the level's frames k.  Returns
    (order, L) with L the dense factor in elimination order.  `defect` injects one modelled kernel bug (DEFECTS):
      drop_pair        one source pair of one update is skipped;
      drop_k_tail      one update skips its last 8 K columns (the half last K stage, neff = 8 mod 16);
      skip_warp_tile   one 8x8 unit of one target is not updated (a warp tile that was never issued);
      skip_diag_split  a symmetric diagonal target skips its lower-left warp tile instead of the upper-right one;
      perturb_pivot    one pivot is off by 1e-12 relative;
      stale_u2         a target misses one overlapped (side-stream) update because the next level read it before it landed."""
    order, cs = elimination_order(n, pairs, slack)
    lvl = levels(order, cs)
    pos = {k: q for q, k in enumerate(order)}
    M, _ = permute(A, order, nf)
    W = M.copy()
    L = np.zeros_like(M)
    blk = lambda f: slice(pos[f] * nf, (pos[f] + 1) * nf)
    neff = min((nf + 7) // 8 * 8, (nf + 15) // 16 * 16)
    nl = max(lvl.values()) + 1
    frames_of = [[k for k in order if lvl[k] == l] for l in range(nl)]
    # update lists per level: target (r, c) -> source frames k
    upd = [dict() for _ in range(nl)]
    for k in order:
        for a in range(len(cs[k])):
            for b in range(a + 1):
                r, c = cs[k][a], cs[k][b]
                upd[lvl[k]].setdefault((r, c), []).append(k)
    # where each defect strikes: the first update (in level order) that has what the defect needs
    hit = None
    for l in range(nl):
        for (r, c), ks in upd[l].items():
            later = any((r, c) in upd[m] for m in range(l + 1, nl))
            if defect in ("drop_pair", "drop_k_tail", "skip_warp_tile") and r != c and hit is None:
                hit = (l, r, c)
            if defect == "skip_diag_split" and r == c and nf > 8 and hit is None:
                hit = (l, r, c)
            if defect == "stale_u2" and lvl[c] != l + 1 and later and hit is None:
                hit = (l, r, c)
    if defect in ("drop_pair", "drop_k_tail", "skip_warp_tile", "skip_diag_split", "stale_u2") and hit is None:
        raise ValueError(f"graph has no update for defect {defect}")
    for l in range(nl):
        for k in frames_of[l]:
            try:
                Lkk = np.linalg.cholesky(W[blk(k), blk(k)])
            except np.linalg.LinAlgError:           # a defect made the block indefinite: the kernels would flag the pivot
                Lkk = np.full((nf, nf), np.nan)
            if defect == "perturb_pivot" and l == 0 and k == frames_of[0][0]:
                Lkk[nf // 2, nf // 2] *= 1.0 + 1e-12
            L[blk(k), blk(k)] = Lkk
            for r in cs[k]:
                L[blk(r), blk(k)] = scipy.linalg.solve_triangular(Lkk, W[blk(r), blk(k)].T, lower=True, check_finite=False).T
        for (r, c), ks in upd[l].items():
            if defect == "stale_u2" and hit == (l, r, c):
                continue
            acc = np.zeros((nf, nf))
            for q, k in enumerate(ks):
                if defect == "drop_pair" and hit == (l, r, c) and q == 0:
                    continue
                Xr, Xc = L[blk(r), blk(k)], L[blk(c), blk(k)]
                if defect == "drop_k_tail" and hit == (l, r, c) and q == 0:
                    Xr, Xc = Xr[:, :neff - 8], Xc[:, :neff - 8]
                acc += Xr @ Xc.T
            if hit == (l, r, c):
                if defect == "skip_warp_tile":
                    acc[:8, :8] = 0.0
                elif defect == "skip_diag_split":
                    tile = min(80, neff); h = ((tile // 8) + 1) // 2 * 8      # k_update_tma: rows / columns of warp-row / -column 0
                    acc[h:min(2 * h, nf), :h] = 0.0
            W[blk(r), blk(c)] -= acc
            if r == c:
                W[blk(r), blk(c)] = np.tril(W[blk(r), blk(c)]) + np.tril(W[blk(r), blk(c)], -1).T
    return order, L
