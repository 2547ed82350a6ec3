"""oracle/refinex_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_refine_x / cflx_chol_refine_x
(conflux_b200/csrc/refine.cu refine_x_run): LAPACK's dgerfsx / dporfsx with the solves passed in as callbacks.

  * exact_residual: b - op(A) (y + t) correctly rounded (math.fsum over the Dekker-split products, every term exact);
  * Column: one column's state machine of dla_gerfsx_extended (RefineXColumn in lu_state.h), stats its statistics of a
    round, wwaddw LAPACK's dla_wwaddw;
  * rfsx / gerfsx / porfsx: the whole routine -- the lockstep loop, berr (dla_lin_berr), the normwise (dla_gercond CMODE
    -1 with d, 0 without) and componentwise (CMODE 1 with y_j, skipped where the bound is not below sqrt(eps))
    condition estimates by cond_ref.dlacn2, and the bounds;
  * partials_x_lu / partials_x_chol: the double-double partial products as the grid forms them, each rank's exact sum
    split into (hi, lo) and the pairs added in the device's order (refine_ref's _assemble order)."""
import math

import numpy as np

from . import chol_ref, cond_ref, layout
from .refine_ref import _gidx, sym_masks

EPS = 2.0 ** -53
SAFMIN = 2.0 ** -1022
ITHRESH = 10
RTHRESH = 0.5
DZ_UB = 0.25
UNSTABLE, WORKING, CONV, NOPROG = 0, 1, 2, 3
EXTRA_RESIDUAL, EXTRA_Y = 1, 2


def _split(a):
    c = a * 134217729.0                          # 2^27 + 1: Veltkamp's split, a = hi + lo with 26-bit halves
    hi = c - (c - a)
    return hi, a - hi


def _exact_terms(A, x):
    """the exact products A[i, k] x[k] as four float64 terms each: rows of 4K terms"""
    ah, al = _split(np.asarray(A, dtype=np.float64))
    xh, xl = _split(np.asarray(x, dtype=np.float64))
    return np.concatenate([ah * xh, ah * xl, al * xh, al * xl], axis=1)


def exact_sum_rows(T):
    """correctly rounded row sums of T"""
    return np.array([math.fsum(r) for r in T])


def exact_residual(Aop, b, y, t=None):
    """b - Aop (y + t) per column, correctly rounded"""
    Aop = np.asarray(Aop, dtype=np.float64)
    Y = np.asarray(y, dtype=np.float64).reshape(Aop.shape[1], -1)
    B = np.asarray(b, dtype=np.float64).reshape(Aop.shape[0], -1)
    Tt = None if t is None else np.asarray(t, dtype=np.float64).reshape(Y.shape)
    R = np.empty(B.shape)
    for j in range(B.shape[1]):
        terms = -_exact_terms(Aop, Y[None, :, j])
        if Tt is not None:
            terms = np.concatenate([terms, -_exact_terms(Aop, Tt[None, :, j])], axis=1)
        R[:, j] = exact_sum_rows(np.concatenate([B[:, j:j + 1], terms], axis=1))
    return R.reshape(np.shape(b))


def wwaddw(x, t, w):
    """LAPACK dla_wwaddw: (x, t) += w"""
    s = x + w
    s = (s + s) - s
    t = ((x - s) + w) + t
    xn = s + t
    return xn, (s - xn) + t


def stats(y, dy, d=None):
    """{normy, normx, normdx, dz_z, ymin} of one column"""
    yk, dyk = np.abs(y), np.abs(dy)
    with np.errstate(divide="ignore", invalid="ignore"):
        dz = np.where(yk != 0, dyk / np.where(yk != 0, yk, 1.0), np.where(dyk != 0, np.inf, 0.0))
    normx = yk.max() if d is None else (yk * d).max()
    normdx = dyk.max() if d is None else (dyk * d).max()
    return yk.max(), normx, normdx, dz.max(), yk.min()


class Column:
    """one column of dla_gerfsx_extended"""

    def __init__(self):
        self.x_state, self.z_state, self.y_prec, self.done = WORKING, UNSTABLE, EXTRA_RESIDUAL, False
        self.dx_x = self.dz_z = self.prev_normdx = self.prev_dz_z = math.inf
        self.dxratmax = self.dzratmax = 0.0
        self.final_dx_x = self.final_dz_z = math.inf
        self.err_norm = self.err_comp = 0.0

    def round(self, st, rcond, ignore_cwise, cnt, M):
        """0: stop without an update; 1: y += dy; 2: (y, y_tail) += dy"""
        normy, normx, normdx, dz_z, ymin = st
        self.dz_z = dz_z
        self.dx_x = normdx / normx if normx != 0 else (0.0 if normdx == 0 else math.inf)
        with np.errstate(divide="ignore", invalid="ignore"):
            dxrat = float(np.float64(normdx) / np.float64(self.prev_normdx))
            dzrat = float(np.float64(dz_z) / np.float64(self.prev_dz_z))
        incr = (not ignore_cwise) and ymin * rcond < M * EPS * normy and self.y_prec < EXTRA_Y
        if self.x_state == NOPROG and dxrat <= RTHRESH:
            self.x_state = WORKING
        if self.x_state == WORKING:
            if self.dx_x <= EPS:
                self.x_state = CONV
            elif dxrat > RTHRESH:
                if self.y_prec != EXTRA_Y:
                    incr = True
                else:
                    self.x_state = NOPROG
            elif dxrat > self.dxratmax:
                self.dxratmax = dxrat
            if self.x_state > WORKING:
                self.final_dx_x = self.dx_x
        if self.z_state == UNSTABLE and dz_z <= DZ_UB:
            self.z_state = WORKING
        if self.z_state == NOPROG and dzrat <= RTHRESH:
            self.z_state = WORKING
        if self.z_state == WORKING:
            if dz_z <= EPS:
                self.z_state = CONV
            elif dz_z > DZ_UB:
                self.z_state, self.dzratmax, self.final_dz_z = UNSTABLE, 0.0, math.inf
            elif dzrat > RTHRESH:
                if self.y_prec != EXTRA_Y:
                    incr = True
                else:
                    self.z_state = NOPROG
            elif dzrat > self.dzratmax:
                self.dzratmax = dzrat
            if self.z_state > WORKING:
                self.final_dz_z = dz_z
        if self.x_state != WORKING and (ignore_cwise or self.z_state in (NOPROG, CONV)
                                        or (self.z_state == UNSTABLE and cnt > 1)):
            self.done = True
            return 0
        if incr:
            self.y_prec = EXTRA_Y
        self.prev_normdx, self.prev_dz_z = normdx, dz_z
        return 2 if self.y_prec == EXTRA_Y else 1

    def finish(self):
        if self.x_state == WORKING:
            self.final_dx_x = self.dx_x
        if self.z_state == WORKING:
            self.final_dz_z = self.dz_z
        self.err_norm = self.final_dx_x / (1 - self.dxratmax)
        self.err_comp = self.final_dz_z / (1 - self.dzratmax)


def cond(n, solve, solve_t, g, r, r_div):
    """dla_gercond: 1 / the dlacn2 estimate on diag(g) inv(op A)^T diag(r) (kase 1) / diag(r) inv(op A) diag(g) (kase
    2), r applied by division when r_div (CMODE 1), else by multiplication"""
    R = (lambda x: x / r) if r_div else (lambda x: x * r)

    def apply(kase, x):
        return g * solve_t(R(x)) if kase == 1 else R(solve(g * x))
    est = cond_ref.dlacn2(n, apply)
    return 1.0 / est if est != 0 else 0.0


def rfsx(Aop, B, Y, solve, solve_t, rcond, d=None, cwise=True, residual=exact_residual, dys=None):
    """dgerfsx / dporfsx on op(A) = Aop: solve(x) = inv(op A) x, solve_t(x) = inv(op A)^T x; d the scales of the unscaled
    solution (None: ones).  dys (tests): a callable (j, round) -> dy replacing the solve of the correction.  Returns
    (Y, berr, err_norm, err_comp, info, columns)."""
    Aop = np.asarray(Aop, dtype=np.float64)
    n, nrhs = B.shape
    Y = np.array(Y, dtype=np.float64)
    T = np.zeros_like(Y)
    cols = [Column() for _ in range(nrhs)]
    for cnt in range(1, ITHRESH + 1):
        active = [j for j in range(nrhs) if not cols[j].done]
        if not active:
            break
        for j in active:
            if dys is not None:
                dy = dys(j, cnt)
            else:
                dy = solve(residual(Aop, B[:, j], Y[:, j], T[:, j]))
            how = cols[j].round(stats(Y[:, j], dy, d), rcond, not cwise, cnt, n)
            if how == 1:
                Y[:, j] = Y[:, j] + dy
            elif how == 2:
                Y[:, j], T[:, j] = wwaddw(Y[:, j], T[:, j], dy)
    for c in cols:
        c.finish()
    R = B - Aop @ Y
    S = np.abs(Aop) @ np.abs(Y) + np.abs(B)
    safe1 = (n + 1) * SAFMIN
    berr = np.max(np.where(S != 0, (np.abs(R) + safe1) / np.where(S != 0, S, 1.0), 0.0), axis=0)
    illthresh, err_lbnd = n * EPS, max(10.0, math.sqrt(n)) * EPS
    dd = np.ones(n) if d is None else np.asarray(d, dtype=np.float64)
    rc_norm = cond(n, solve, solve_t, np.abs(Aop) @ np.abs(1.0 / dd), dd, False)
    en, ec = np.zeros((nrhs, 3)), (np.zeros((nrhs, 3)) if cwise else None)
    first = 0

    def bound(err, rc, j, out):
        nonlocal first
        trust, err = 1.0, min(err, 1.0)
        if rc < illthresh:
            err, trust = 1.0, 0.0
            first = first or j + 1
        elif err < err_lbnd:
            err = err_lbnd
        out[j] = (trust, err, rc)
    for j in range(nrhs):
        bound(cols[j].err_norm, rc_norm, j, en)
        if cwise:
            rc = (cond(n, solve, solve_t, np.abs(Aop) @ np.abs(Y[:, j]), Y[:, j], True)
                  if cols[j].err_comp < math.sqrt(EPS) else 0.0)
            bound(cols[j].err_comp, rc, j, ec)
    return Y, berr, en, ec, (n + first if first else 0), cols


def gerfsx(A, B, Y, solve, solve_t, rcond, trans=False, d=None, cwise=True, **kw):
    A = np.asarray(A)
    return rfsx(A.T if trans else A, np.asarray(B), Y, solve, solve_t, rcond, d, cwise, **kw)


def porfsx(A, B, Y, solve, rcond, d=None, cwise=True, **kw):
    return rfsx(np.asarray(A), np.asarray(B), Y, solve, solve, rcond, d, cwise, **kw)


# ------------------------------------------------------------------------------------------------ the grid product
def _dd_add(a, b):
    s = a[0] + b[0]
    bb = s - a[0]
    e = (a[0] - (s - bb)) + (b[0] - bb)
    e = e + (a[1] + b[1])
    hi = s + e
    bb = hi - s
    return hi, (s - (hi - bb)) + (e - bb)


def _exact_pair(Aop, y, t):
    """op(A)(y + t) per row as an exact-sum pair (hi = the correctly rounded sum, lo = the rounded remainder)"""
    terms = np.concatenate([_exact_terms(Aop, y[None, :]), _exact_terms(Aop, t[None, :])], axis=1)
    hi = exact_sum_rows(terms)
    lo = np.array([math.fsum(list(r) + [-h]) for r, h in zip(terms, hi)])
    return hi, lo


def _assemble_x(nn, tn, n, v, Px, Py):
    """the sum of the (hi, lo) partials in the device's order, in double-double: (hi, lo) per row"""
    H, L = np.zeros(n), np.zeros(n)
    for g in range(n):
        T, e = divmod(g, v)
        p = (0.0, 0.0)
        if nn:
            for pj in range(Py):
                h, l = nn[(T % Px, pj)]
                p = _dd_add(p, (h[(T // Px) * v + e], l[(T // Px) * v + e]))
        if tn:
            for pi in range(Px):
                h, l = tn[(pi, T % Py)]
                p = _dd_add(p, (h[(T // Py) * v + e], l[(T // Py) * v + e]))
        H[g], L[g] = p
    return H, L


def partials_x_lu(A_locals, y, t, N, v, Px=1, Py=1, Pz=1, trans=False):
    """(hi, lo) of op(A)(y + t) of the padded LU input (one column) from the layer-0 shares, as the grid forms it"""
    d = layout.dims(N, v, Px, Py, Pz)
    M, Ml, Nl = d["M"], d["Ml"], d["Nl"]
    parts = {}
    for pi in range(Px):
        for pj in range(Py):
            A = np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(Ml, Nl)
            if trans:
                idx = [_gidx(l, Px, pi, v) for l in range(Ml)]
                parts[(pi, pj)] = _exact_pair(A.T, y[idx], t[idx])
            else:
                idx = [_gidx(l, Py, pj, v) for l in range(Nl)]
                parts[(pi, pj)] = _exact_pair(A, y[idx], t[idx])
    return _assemble_x(None if trans else parts, parts if trans else None, M, v, Px, Py)


def partials_x_chol(A_locals, y, t, N, v, Px=1, Py=1, Pz=1):
    """(hi, lo) of A (y + t) for the symmetric matrix whose lower triangle the layer-0 shares hold; reads nothing the
    device must not read"""
    d = chol_ref.dims(N, v, Px, Py, Pz)
    n, K, Ml, Nl = d["N"], d["Kappa"], d["Ml"], d["Nl"]
    nn, tn = {}, {}
    for pi in range(Px):
        for pj in range(Py):
            A = np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(Ml, Nl)
            mnn, mtn = sym_masks(Ml, Nl, v, K, Px, Py, pi, pj)
            rows = [min(_gidx(l, Px, pi, v), n - 1) for l in range(Ml)]
            cols = [min(_gidx(l, Py, pj, v), n - 1) for l in range(Nl)]
            nn[(pi, pj)] = _exact_pair(np.where(mnn, A, 0.0), y[cols], t[cols])
            tn[(pi, pj)] = _exact_pair(np.where(mtn, A, 0.0).T, y[rows], t[rows])
    return _assemble_x(nn, tn, n, v, Px, Py)
