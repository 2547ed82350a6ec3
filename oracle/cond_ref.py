"""oracle/cond_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_rcond / cflx_chol_rcond (conflux_b200/csrc/
solve.cu estimate_inv_norm1, norm.cu).

  * dlacn2(n, apply): LAPACK's Hager-Higham 1-norm estimator with its reverse communication unrolled; apply(kase, x)
    returns inv(A) x (kase 1) or inv(A)^T x (kase 2).  gecon / pocon drive it as LAPACK's dgecon (NORM = '1') and dpocon
    (UPLO = 'L') do, with the triangular solves of the assembled factors and no dlatrs scaling;
  * norm1_lu / norm1_chol: the 1-norm of the matrix whose layer-0 shares are given in the conflux layout, read the way the
    device kernel reads them: every local entry for the LU input, and for the Cholesky input only the real tiles on and
    below the diagonal (the diagonal tiles' lower triangle), the strictly lower part counted again as its transpose."""
import numpy as np

from . import chol_ref, layout

ITMAX = 5


def dlacn2(n, apply):
    """estimate of ||inv(A)||_1 (LAPACK dlacn2: x = 1/n, at most ITMAX iterations, sign-vector test, final alternating
    vector)"""
    x = apply(1, np.full(n, 1.0 / n))
    if n == 1:
        return abs(float(x[0]))
    est = float(np.sum(np.abs(x)))
    x = np.where(x >= 0, 1.0, -1.0)
    isgn = x.copy()
    x = apply(2, x)
    j = int(np.argmax(np.abs(x)))
    it = 2
    while True:
        x = np.zeros(n)
        x[j] = 1.0
        x = apply(1, x)
        estold, est = est, float(np.sum(np.abs(x)))
        sg = np.where(x >= 0, 1.0, -1.0)
        if np.array_equal(sg, isgn) or est <= estold:
            break
        x, isgn = sg, sg.copy()
        x = apply(2, x)
        jlast, j = j, int(np.argmax(np.abs(x)))
        if not (x[jlast] != abs(x[j]) and it < ITMAX):
            break
        it += 1
    x = np.array([(-1.0) ** i * (1.0 + i / (n - 1)) for i in range(n)])
    x = apply(1, x)
    temp = 2.0 * (float(np.sum(np.abs(x))) / (3 * n))
    return temp if temp > est else est


def rcond(anorm, ainvnm):
    if not anorm > 0 or not ainvnm > 0 or not np.isfinite(ainvnm):
        return 0.0
    r = (1.0 / ainvnm) / anorm
    return float(r) if np.isfinite(r) else 0.0


def gecon(LU, anorm):
    """dgecon ('1') on packed L\\U factors (of P A: no permutation), returns (rcond, ainvnm)"""
    from scipy.linalg import solve_triangular

    def apply(kase, x):
        if kase == 1:
            return solve_triangular(LU, solve_triangular(LU, x, lower=True, unit_diagonal=True))
        return solve_triangular(LU, solve_triangular(LU, x, trans="T"), trans="T", lower=True, unit_diagonal=True)
    ainvnm = dlacn2(LU.shape[0], apply)
    return rcond(anorm, ainvnm), ainvnm


def pocon(L, anorm):
    """dpocon ('L') on a lower Cholesky factor, returns (rcond, ainvnm)"""
    from scipy.linalg import solve_triangular

    def apply(kase, x):
        return solve_triangular(L, solve_triangular(L, x, lower=True), lower=True, trans="T")
    ainvnm = dlacn2(L.shape[0], apply)
    return rcond(anorm, ainvnm), ainvnm


def norm1_lu(A_locals, N, v, Px=1, Py=1, Pz=1):
    """||A||_1 of the padded M x M LU input from the layer-0 shares (per-rank column sums, summed over the grid)"""
    d = layout.dims(N, v, Px, Py, Pz)
    M, Ml, Nl = d["M"], d["Ml"], d["Nl"]
    col = np.zeros(M)
    for pi in range(Px):
        for pj in range(Py):
            loc = np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(Ml, Nl)
            s = np.abs(loc).sum(0)
            for c in range(Nl):
                col[((c // v) * Py + pj) * v + c % v] += s[c]
    return float(col.max())


def norm1_chol(A_locals, N, v, Px=1, Py=1, Pz=1):
    """||A||_1 of the symmetric N x N (padded) matrix whose lower triangle the layer-0 shares hold.  Reads nothing above
    the diagonal and no tile with a global index >= Kappa (NaN there does not reach the result)."""
    d = chol_ref.dims(N, v, Px, Py, Pz)
    Np, K, Ml, Nl = d["N"], d["Kappa"], d["Ml"], d["Nl"]
    col = np.zeros(Np)
    for pi in range(Px):
        for pj in range(Py):
            loc = np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(Ml, Nl)
            for lti in range(Ml // v):
                for ltj in range(Nl // v):
                    gi, gj = lti * Px + pi, ltj * Py + pj
                    if gi >= K or gj >= K or gi < gj:
                        continue
                    blk = np.abs(loc[lti * v:(lti + 1) * v, ltj * v:(ltj + 1) * v])
                    if gi == gj:
                        low = np.tril(blk)
                        col[gj * v:(gj + 1) * v] += low.sum(0) + np.tril(blk, -1).sum(1)
                    else:
                        col[gj * v:(gj + 1) * v] += blk.sum(0)     # lower part of the columns gj
                        col[gi * v:(gi + 1) * v] += blk.sum(1)     # the same entries as rows gi: their transposes
    return float(col.max())
