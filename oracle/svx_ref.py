"""oracle/svx_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_equilibrate / cflx_lu_svx and
cflx_chol_equilibrate / cflx_chol_svx (conflux_b200/csrc/equil.cu, lu.cu, chol.cu).

  * geequ / laqge, poequ / laqsy: LAPACK's dgeequ + dlaqge and dpoequ + dlaqsy (UPLO = 'L'), elementwise in LAPACK's
    operation order, so that their results are bit-identical to LAPACK's;
  * rpvgrw: dgesvx's reciprocal pivot growth factor of the scaled matrix and its L\\U;
  * gecon_inf: dgecon with NORM = 'I' on cond_ref.dlacn2 (the two kinds of solve swapped);
  * gesvx / posvx: dgesvx / dposvx after the factorisation, composed from the above and refine_ref.gerfs / porfs;
  * row_max_share / col_max_share / diag_share / apply_share / sym_apply_share / growth_share / zero_pivot_share: the
    per-share passes (zeros where a share holds nothing), and geequ_grid / diag_grid: their combination over the grid."""
import numpy as np

from . import chol_ref, cond_ref, layout
from . import refine_ref as rr

SAFMIN = 2.0 ** -1022                 # dlamch('S')
SMALL = SAFMIN / 2.0 ** -52           # dlamch('S') / dlamch('P')
LARGE = 1.0 / SMALL
THRESH = 0.1
EPS = 2.0 ** -53


def geequ(A):
    """dgeequ: dict(r, c, rowcnd, colcnd, amax, info).  info = i (first zero row, r holds the row maxima, c zeros) or
    M + j (first zero column, c holds the column maxima of |a| r), 1-based."""
    A = np.asarray(A, dtype=np.float64)
    m, n = A.shape
    big = 1.0 / SAFMIN
    r = np.abs(A).max(axis=1)
    out = dict(r=r, c=np.zeros(n), rowcnd=0.0, colcnd=0.0, amax=float(r.max()), info=0)
    rcmin = min(big, float(r.min()))
    if rcmin == 0.0:
        out["info"] = int(np.argmax(r == 0.0)) + 1
        return out
    r = 1.0 / np.minimum(np.maximum(r, SAFMIN), big)
    out["r"] = r
    out["rowcnd"] = max(rcmin, SAFMIN) / min(out["amax"], big)
    c = (np.abs(A) * r[:, None]).max(axis=0)
    cmin, cmax = min(big, float(c.min())), float(c.max())
    if cmin == 0.0:
        out["c"] = c
        out["info"] = m + int(np.argmax(c == 0.0)) + 1
        return out
    out["c"] = 1.0 / np.minimum(np.maximum(c, SAFMIN), big)
    out["colcnd"] = max(cmin, SAFMIN) / min(cmax, big)
    return out


def laqge(A, r, c, rowcnd, colcnd, amax):
    """dlaqge: (As, equed)"""
    A = np.asarray(A, dtype=np.float64)
    if rowcnd >= THRESH and SMALL <= amax <= LARGE:
        if colcnd >= THRESH:
            return A.copy(), "N"
        return c[None, :] * A, "C"
    if colcnd >= THRESH:
        return r[:, None] * A, "R"
    return (c[None, :] * r[:, None]) * A, "B"


def poequ(A):
    """dpoequ: dict(s, scond, amax, info); info = i for the first a_ii <= 0 (s then holds the diagonal)"""
    d = np.diag(np.asarray(A, dtype=np.float64)).copy()
    out = dict(s=d, scond=0.0, amax=float(d.max()), info=0)
    smin = float(d.min())
    if smin <= 0.0:
        out["info"] = int(np.argmax(d <= 0.0)) + 1
        return out
    out["s"] = 1.0 / np.sqrt(d)
    out["scond"] = float(np.sqrt(smin) / np.sqrt(out["amax"]))
    return out


def laqsy(A, s, scond, amax):
    """dlaqsy (UPLO = 'L'): (As, equed); only the lower triangle is scaled, the strict upper part is A's own"""
    A = np.asarray(A, dtype=np.float64)
    if scond >= THRESH and SMALL <= amax <= LARGE:
        return A.copy(), "N"
    As = A.copy()
    low = np.tril(np.ones(A.shape, dtype=bool))
    As[low] = ((s[None, :] * s[:, None]) * A)[low]
    return As, "Y"


def rpvgrw(As, LU, ncols=None):
    """dgesvx's RPVGRW over the leading ncols columns: max |As[:, :ncols]| / max |triu(LU)[:ncols, :ncols]|, 1 when the
    latter is 0"""
    n = As.shape[1] if ncols is None else ncols
    den = float(np.abs(np.triu(LU[:n, :n])).max()) if n > 0 else 0.0
    return 1.0 if den == 0.0 else float(np.abs(As[:, :n]).max()) / den


def gecon_inf(LU, anorm):
    """dgecon (NORM = 'I') on packed L\\U factors of P A: (rcond, ainvnm)"""
    from scipy.linalg import solve_triangular

    def apply(kase, x):
        if kase == 2:
            return solve_triangular(LU, solve_triangular(LU, x, lower=True, unit_diagonal=True))
        return solve_triangular(LU, solve_triangular(LU, x, trans="T"), trans="T", lower=True, unit_diagonal=True)
    ainvnm = cond_ref.dlacn2(LU.shape[0], apply)
    return cond_ref.rcond(anorm, ainvnm), ainvnm


def gesvx(As, LU, perm, B, trans=False, r=None, c=None, equed="N", rowcnd=1.0, colcnd=1.0):
    """dgesvx after the factorisation of the scaled matrix As (P As = L U): dict(X, rcond, ferr, berr, rpvgrw, info)"""
    B = np.asarray(B, dtype=np.float64).reshape(As.shape[0], -1)
    n = As.shape[0]
    rowequ, colequ = equed in "RB", equed in "CB"
    d = np.diag(LU)
    if np.any(d == 0.0):
        k = int(np.argmax(d == 0.0)) + 1
        return dict(X=None, rcond=0.0, ferr=None, berr=None, rpvgrw=rpvgrw(As, LU, k), info=k)
    if not trans:
        rc, _ = cond_ref.gecon(LU, float(np.abs(As).sum(0).max()))
        Bs = r[:, None] * B if rowequ else B.copy()
    else:
        rc, _ = gecon_inf(LU, float(np.abs(As).sum(1).max()))
        Bs = c[:, None] * B if colequ else B.copy()
    solve, solve_t = rr.lu_solvers(LU, perm, trans)
    X, ferr, berr = rr.gerfs(As, Bs, solve(Bs), solve, solve_t, trans)
    if not trans and colequ:
        X, ferr = c[:, None] * X, ferr / colcnd
    if trans and rowequ:
        X, ferr = r[:, None] * X, ferr / rowcnd
    return dict(X=X, rcond=rc, ferr=ferr, berr=berr, rpvgrw=rpvgrw(As, LU), info=n + 1 if rc < EPS else 0)


def posvx(As, L, B, s=None, equed="N", scond=1.0):
    """dposvx after the factorisation of the scaled symmetric matrix As = L L^T: dict(X, rcond, ferr, berr, info)"""
    B = np.asarray(B, dtype=np.float64).reshape(As.shape[0], -1)
    rc, _ = cond_ref.pocon(L, float(np.abs(As).sum(0).max()))
    Bs = s[:, None] * B if equed == "Y" else B.copy()
    solve = rr.chol_solver(L)
    X, ferr, berr = rr.porfs(As, Bs, solve(Bs), solve)
    if equed == "Y":
        X, ferr = s[:, None] * X, ferr / scond
    return dict(X=X, rcond=rc, ferr=ferr, berr=berr, info=As.shape[0] + 1 if rc < EPS else 0)


# ------------------------------------------------------------------------------------------------ the grid passes
def _gidx(l, P, p, v):
    return ((np.asarray(l) // v) * P + p) * v + np.asarray(l) % v


def row_max_share(A, M, v, Px, pi):
    """one share's partial row maxima: an M-vector, zeros where the share holds no row"""
    A = np.asarray(A)
    out = np.zeros(M)
    out[_gidx(np.arange(A.shape[0]), Px, pi, v)] = np.abs(A).max(axis=1)
    return out


def col_max_share(A, M, v, Px, Py, pi, pj, r):
    """one share's partial maxima of |a| r_i by column: an M-vector, zeros where the share holds no column"""
    A = np.asarray(A)
    out = np.zeros(M)
    rows = _gidx(np.arange(A.shape[0]), Px, pi, v)
    out[_gidx(np.arange(A.shape[1]), Py, pj, v)] = (np.abs(A) * r[rows][:, None]).max(axis=0)
    return out


def apply_share(A, v, Px, Py, pi, pj, r, c, equed):
    """dlaqge's scaling of one share"""
    A = np.asarray(A, dtype=np.float64)
    ri = r[_gidx(np.arange(A.shape[0]), Px, pi, v)][:, None] if r is not None else None
    cj = c[_gidx(np.arange(A.shape[1]), Py, pj, v)][None, :] if c is not None else None
    return {"N": lambda: A.copy(), "R": lambda: ri * A, "C": lambda: cj * A, "B": lambda: (cj * ri) * A}[equed]()


def diag_share(A, N, v, Kappa, Px, Py, pi, pj):
    """one share's diagonal entries of the real tiles: an N-vector, zeros elsewhere"""
    A = np.asarray(A)
    out = np.zeros(N)
    for t in range(Kappa):
        if t % Px == pi and t % Py == pj:
            blk = A[(t // Px) * v:(t // Px + 1) * v, (t // Py) * v:(t // Py + 1) * v]
            out[t * v:(t + 1) * v] = np.diag(blk)
    return out


def sym_apply_share(A, v, Kappa, Px, Py, pi, pj, s):
    """dlaqsy's scaling of one share: (s_j s_i) a over the real tiles' entries with global row >= column, the rest as
    it was"""
    A = np.array(A, dtype=np.float64)
    gr = _gidx(np.arange(A.shape[0]), Px, pi, v)[:, None]
    gc = _gidx(np.arange(A.shape[1]), Py, pj, v)[None, :]
    m = (gr // v < Kappa) & (gc // v < Kappa) & (gr >= gc)
    sr, sc = s[np.minimum(gr, len(s) - 1)], s[np.minimum(gc, len(s) - 1)]
    A[m] = ((sc * sr) * A)[m]
    return A


def growth_share(F, A, v, Px, Py, pi, pj, ncols):
    """one share's (max |F| over global row <= column, max |A|), both over the global columns < ncols"""
    F, A = np.asarray(F), np.asarray(A)
    gr = _gidx(np.arange(F.shape[0]), Px, pi, v)[:, None]
    gc = _gidx(np.arange(F.shape[1]), Py, pj, v)[None, :]
    cols = np.broadcast_to(gc < ncols, F.shape)
    up = cols & (gr <= gc)
    return (float(np.abs(F[up]).max()) if up.any() else 0.0, float(np.abs(A[cols]).max()) if cols.any() else 0.0)


def zero_pivot_share(F, M, v, Px, Py, pi, pj):
    """1 + the first global g < M on the share's diagonal tiles with F_gg == 0, or 0"""
    F = np.asarray(F)
    for g in range(M):
        t, e = divmod(g, v)
        if t % Px != pi or t % Py != pj or (t // Px) * v >= F.shape[0] or (t // Py) * v >= F.shape[1]:
            continue
        if F[(t // Px) * v + e, (t // Py) * v + e] == 0.0:
            return g + 1
    return 0


def geequ_grid(A_locals, N, v, Px=1, Py=1, Pz=1):
    """(row maxima, column maxima of |a| r) of the LU input from the layer-0 shares, combined by maxima over the grid"""
    d = layout.dims(N, v, Px, Py, Pz)
    M = d["M"]
    shares = {(pi, pj): np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(d["Ml"], d["Nl"])
              for pi in range(Px) for pj in range(Py)}
    rmax = np.max([row_max_share(a, M, v, Px, pi) for (pi, pj), a in shares.items()], axis=0)
    r = 1.0 / np.minimum(np.maximum(rmax, SAFMIN), 1.0 / SAFMIN)
    cmax = np.max([col_max_share(a, M, v, Px, Py, pi, pj, r) for (pi, pj), a in shares.items()], axis=0)
    return rmax, cmax


def diag_grid(A_locals, N, v, Px=1, Py=1, Pz=1):
    """the diagonal of the Cholesky input from the layer-0 shares (one contributor per entry)"""
    d = chol_ref.dims(N, v, Px, Py, Pz)
    out = np.zeros(d["N"])
    for pi in range(Px):
        for pj in range(Py):
            a = np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(d["Ml"], d["Nl"])
            out = out + diag_share(a, d["N"], v, d["Kappa"], Px, Py, pi, pj)
    return out
