"""oracle/svxx_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_equilibrate_b / cflx_lu_svxx and
cflx_chol_equilibrate_b / cflx_chol_svxx (conflux_b200/csrc/equil.cu, lu.cu, chol.cu).

  * geequb / poequb: LAPACK's dgeequb / dpoequb.  The exponents come from math.log (the C library's log, which LAPACK
    calls too), and RADIX**n is evaluated as an integer power is: 2^n, or 1 / 2^-n for n < 0;
  * gerpvgrw / porpvgrw: LAPACK 3.2's dla_gerpvgrw / dla_porpvgrw ('L'), the per-column reciprocal pivot growth;
  * gesvxx / posvxx: dgesvxx / dposvxx after the factorisation, composed from svx_ref.laqge / laqsy (applied by the
    caller), cond_ref and refinex_ref.gerfsx / porfsx;
  * growth_cols_share / growth_cols_grid: the per-share growth pass (zeros where a share holds nothing) and its
    combination by maxima over the grid."""
import math

import numpy as np

from . import chol_ref, cond_ref, layout
from . import refine_ref as rr
from . import refinex_ref as rx
from . import svx_ref as sr

SAFMIN = sr.SAFMIN
LOGRDX = math.log(2.0)


def _pow2i(n):
    """RADIX**n for RADIX = 2 as an integer power: 0 once 2^-n overflows"""
    with np.errstate(over="ignore"):
        return float(np.ldexp(1.0, n)) if n >= 0 else float(1.0 / np.ldexp(1.0, -n))


def _round(v):
    """2^INT(LOG(x) / LOGRDX) for every x > 0 of v, INT truncating toward zero; zeros stay"""
    return np.array([_pow2i(int(math.log(x) / LOGRDX)) if x > 0 else x for x in v])


def geequb(A):
    """dgeequb: dict(r, c, rowcnd, colcnd, amax, info) as geequ's, with the maxima rounded to powers of two before
    anything reads them.  info = i (first zero row: r holds the rounded row maxima, c zeros) or M + j (first zero column:
    c holds the rounded column maxima of |a| r), 1-based."""
    A = np.asarray(A, dtype=np.float64)
    m, n = A.shape
    big = 1.0 / SAFMIN
    r = _round(np.abs(A).max(axis=1))
    rcmin, rcmax = min(big, float(r.min())), float(r.max())
    out = dict(r=r, c=np.zeros(n), rowcnd=0.0, colcnd=0.0, amax=rcmax, info=0)
    if rcmin == 0.0:
        out["info"] = int(np.argmax(r == 0.0)) + 1
        return out
    r = 1.0 / np.minimum(np.maximum(r, SAFMIN), big)
    out["r"] = r
    out["rowcnd"] = max(rcmin, SAFMIN) / min(rcmax, big)
    c = _round((np.abs(A) * r[:, None]).max(axis=0))
    cmin, cmax = min(big, float(c.min())), float(c.max())
    if cmin == 0.0:
        out["c"] = c
        out["info"] = m + int(np.argmax(c == 0.0)) + 1
        return out
    out["c"] = 1.0 / np.minimum(np.maximum(c, SAFMIN), big)
    out["colcnd"] = max(cmin, SAFMIN) / min(cmax, big)
    return out


def poequb(A):
    """dpoequb: dict(s, scond, amax, info); info = i for the first a_ii <= 0 (s then holds the diagonal)"""
    d = np.diag(np.asarray(A, dtype=np.float64)).copy()
    smin, amax = float(d.min()), float(d.max())
    out = dict(s=d, scond=0.0, amax=amax, info=0)
    if smin <= 0.0:
        out["info"] = int(np.argmax(d <= 0.0)) + 1
        return out
    tmp = -0.5 / LOGRDX
    out["s"] = np.array([_pow2i(int(tmp * math.log(x))) for x in d])
    out["scond"] = math.sqrt(smin) / math.sqrt(amax)
    return out


def gerpvgrw(A, LU, ncols=None):
    """dla_gerpvgrw(N, ncols, A, AF): min(1, amax_j / umax_j) over the columns j < ncols with umax_j = max_{i <= j}
    |u_ij| != 0, amax_j = max_i |a_ij|"""
    A, LU = np.asarray(A), np.asarray(LU)
    ncols = A.shape[1] if ncols is None else ncols
    rpvgrw = 1.0
    for j in range(ncols):
        amax, umax = float(np.abs(A[:, j]).max()), float(np.abs(LU[:j + 1, j]).max())
        if umax != 0.0:
            rpvgrw = min(amax / umax, rpvgrw)
    return rpvgrw


def porpvgrw(A, L, ncols=None):
    """dla_porpvgrw('L', ncols, A, AF): as gerpvgrw, both maxima over the rows j <= i < ncols of the lower triangles"""
    A, L = np.asarray(A), np.asarray(L)
    ncols = A.shape[1] if ncols is None else ncols
    rpvgrw = 1.0
    for j in range(ncols):
        amax, umax = float(np.abs(A[j:ncols, j]).max()), float(np.abs(L[j:ncols, j]).max())
        if umax != 0.0:
            rpvgrw = min(amax / umax, rpvgrw)
    return rpvgrw


def gesvxx(As, LU, perm, B, trans=False, r=None, c=None, equed="N", cwise=True):
    """dgesvxx after the factorisation of the scaled matrix As (P As = L U): dict(X, rcond, rpvgrw, berr, err_norm,
    err_comp, info, Y) with Y the refined solution of the scaled system"""
    B = np.asarray(B, dtype=np.float64).reshape(As.shape[0], -1)
    n = As.shape[0]
    rowequ, colequ = equed in "RB", equed in "CB"
    dg = np.diag(LU)
    if np.any(dg == 0.0):
        k = int(np.argmax(dg == 0.0)) + 1
        return dict(X=None, rcond=0.0, rpvgrw=gerpvgrw(As, LU, k), info=k)
    if not trans:   # dgecon as dgerfsx runs it: the infinity-norm of op(A) = A, the 1-norm of op(A) = A^T
        rc, _ = sr.gecon_inf(LU, float(np.abs(As).sum(1).max()))
        Bs, d = (r[:, None] * B if rowequ else B.copy()), (c if colequ else None)
    else:
        rc, _ = cond_ref.gecon(LU, float(np.abs(As).sum(0).max()))
        Bs, d = (c[:, None] * B if colequ else B.copy()), (r if rowequ else None)
    solve, solve_t = rr.lu_solvers(LU, perm, trans)
    Y, berr, en, ec, info, _ = rx.gerfsx(As, Bs, solve(Bs), solve, solve_t, rc, trans, d, cwise)
    X = d[:, None] * Y if d is not None else Y
    return dict(X=X, Y=Y, rcond=rc, rpvgrw=gerpvgrw(As, LU), berr=berr, err_norm=en, err_comp=ec, info=info)


def posvxx(As, L, B, s=None, equed="N", cwise=True):
    """dposvxx after the factorisation of the scaled symmetric matrix As = L L^T: dict as gesvxx's"""
    B = np.asarray(B, dtype=np.float64).reshape(As.shape[0], -1)
    rc, _ = cond_ref.pocon(L, float(np.abs(As).sum(0).max()))
    d = s if equed == "Y" else None
    Bs = d[:, None] * B if d is not None else B.copy()
    solve = rr.chol_solver(L)
    Y, berr, en, ec, info, _ = rx.porfsx(As, Bs, solve(Bs), solve, rc, d, cwise)
    X = d[:, None] * Y if d is not None else Y
    return dict(X=X, Y=Y, rcond=rc, rpvgrw=porpvgrw(np.tril(As), L), berr=berr, err_norm=en, err_comp=ec, info=info)


# ------------------------------------------------------------------------------------------------ the grid pass
def growth_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj, ncols, sym):
    """(mask of A, mask of F) over one Ml x Nl share: the entries the growth pass reads"""
    gr = sr._gidx(np.arange(Ml), Px, pi, v)[:, None]
    gc = sr._gidx(np.arange(Nl), Py, pj, v)[None, :]
    cols = np.broadcast_to(gc < ncols, (Ml, Nl))
    if sym:
        m = cols & (gr // v < Kappa) & (gc // v < Kappa) & (gr >= gc) & (gr < ncols)
        return m, m
    return cols, cols & (gr <= gc)


def growth_cols_share(F, A, M, v, Kappa, Px, Py, pi, pj, ncols, sym):
    """one share's (amax, fmax): M-vectors by global column, zeros where the share holds nothing it reads"""
    F, A = np.asarray(F), np.asarray(A)
    Ml, Nl = A.shape
    ma, mf = growth_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj, ncols, sym)
    amax, fmax = np.zeros(M), np.zeros(M)
    gc = sr._gidx(np.arange(Nl), Py, pj, v)
    for c in range(Nl):
        if gc[c] < M:
            amax[gc[c]] = np.abs(A[ma[:, c], c]).max(initial=0.0)
            fmax[gc[c]] = np.abs(F[mf[:, c], c]).max(initial=0.0)
    return amax, fmax


def growth_cols_grid(F_locals, A_locals, N, v, Px=1, Py=1, Pz=1, ncols=None, sym=False):
    """(amax, fmax) of the layer-0 shares combined by maxima over the grid (the LU's layout, or the Cholesky's with
    sym)"""
    d = chol_ref.dims(N, v, Px, Py, Pz) if sym else layout.dims(N, v, Px, Py, Pz)
    M = d["N"] if sym else d["M"]
    K = d["Kappa"] if sym else 1 << 30
    ncols = M if ncols is None else ncols
    amax, fmax = np.zeros(M), np.zeros(M)
    for pi in range(Px):
        for pj in range(Py):
            r = layout.rank_of(pi, pj, 0, Px, Py, Pz)
            F = np.asarray(F_locals[r]).reshape(d["Ml"], d["Nl"])
            A = np.asarray(A_locals[r]).reshape(d["Ml"], d["Nl"])
            a, f = growth_cols_share(F, A, M, v, K, Px, Py, pi, pj, ncols, sym)
            amax, fmax = np.maximum(amax, a), np.maximum(fmax, f)
    return amax, fmax


def rpvgrw_cols(amax, fmax, ncols):
    """the reciprocal pivot growth from the combined vectors, as the host forms it"""
    rpvgrw = 1.0
    for j in range(ncols):
        if fmax[j] != 0.0:
            rpvgrw = min(amax[j] / fmax[j], rpvgrw)
    return rpvgrw
