"""oracle/ldlt_ref.py -- numpy restatement of the signed Cholesky of cflx_chol_factor_ldlt and of cflx_chol_rbt's
symmetric transform: the factorisation A = R S R^T without pivoting (R lower triangular with a positive diagonal,
S = diag(s), s_i = +-1), its tiny rule and inertia, the mirror of the stored lower triangle, the divisibility rule of the
local transform, and the error bounds the GPU factor is checked against.

The bounds are hp_ref's Cholesky bounds with |R| |R^T| in place of |L| |L^T|: the signed elimination computes every
entry with the same operations as the Cholesky, each product of the sum carrying a sign that multiplies exactly, so
Higham's Thm 10.3 argument holds unchanged, |A - R^ S R^T| <= gamma_{n+1} |R^| |R^T|; for the LDL^T form (Higham
ch. 11) L = R diag(R)^-1 and D = S diag(R)^2 give the same |L| |D| |L^T| = |R| |R^T|.  The normwise bound of a factor
whose panels are solved with inverted diagonal blocks is hp_ref.chol_backward_bound of that matrix.
Test infrastructure: only tests/ and tools/ import this."""
import math

import numpy as np

from oracle import hp_ref


def factor(A, tiny=0.0):
    """The signed Cholesky of the symmetric matrix whose lower triangle is A, column by column in float64: pivot d =
    a_cc - sum_{j<c} s_j r_cj^2; |d| < tiny becomes copysign(tiny, d) (+tiny for +-0); s_c = +1 for d > 0, else -1;
    r_cc = sqrt|d|; r_ic = (a_ic - sum_j r_ij s_j r_cj) / (s_c r_cc).  Returns dict(R, s, nrepl, inertia, info) with
    inertia = (positive, negative, zero) pivots and info = 1 + the first exactly zero pivot's column (0: none)."""
    A = np.tril(np.asarray(A, dtype=np.float64))
    n = A.shape[0]
    R = np.zeros((n, n))
    s = np.ones(n)
    nrepl, pos, neg, zero, info = 0, 0, 0, 0, 0
    with np.errstate(divide="ignore", invalid="ignore"):
        for c in range(n):
            d = A[c, c] - np.dot(R[c, :c] * s[:c], R[c, :c])
            if abs(d) < tiny:
                d = tiny if d == 0.0 else math.copysign(tiny, d)
                nrepl += 1
            s[c] = 1.0 if d > 0.0 else -1.0
            pos += d > 0.0
            zero += d == 0.0
            neg += not d > 0.0 and d != 0.0
            if d == 0.0 and not info:
                info = c + 1
            R[c, c] = math.sqrt(abs(d))
            R[c + 1:, c] = (A[c + 1:, c] - (R[c + 1:, :c] * s[:c]) @ R[c, :c]) / (s[c] * R[c, c])
    return dict(R=R, s=s, nrepl=nrepl, inertia=(pos, neg, zero), info=info)


def inertia(A):
    """(positive, negative, zero) eigenvalues of the symmetric matrix whose lower triangle is A, by numpy.linalg.eigvalsh;
    zero within n eps ||A||_2"""
    w = np.linalg.eigvalsh(mirror(A))
    tol = w.size * np.finfo(float).eps * max(np.abs(w).max(), 1e-300)
    return int(np.sum(w > tol)), int(np.sum(w < -tol)), int(np.sum(np.abs(w) <= tol))


def mirror(A):
    """the symmetric completion of A's lower triangle (what cflx_chol_rbt transforms)"""
    L = np.tril(np.asarray(A, dtype=np.float64))
    return L + np.tril(L, -1).T


def represented(R, s):
    """R S R^T in longdouble (hp_ref.matmul)"""
    R = np.tril(np.asarray(R, dtype=np.float64))
    return hp_ref.matmul(R * np.asarray(s, dtype=np.float64)[None, :], R.T)


def residual(A, R, s):
    """(|A - R S R^T| in longdouble, |R| |R^T| in float64), lower triangles (A: lower triangle read)"""
    R = np.tril(np.asarray(R, dtype=np.float64))
    res = np.abs(np.tril(np.tril(np.asarray(A, dtype=np.float64)).astype(hp_ref.LD) - represented(R, s)))
    aR = np.abs(R)
    return res, np.tril(aR @ aR.T)


def componentwise_ok(A, R, s, res=None):
    """|A - R^ S R^T| <= gamma_{n+1} |R^| |R^T| in every entry of the lower triangle (module doc)"""
    E, M = res if res is not None else residual(A, R, s)
    return bool(np.all(np.isfinite(R)) and np.all(E <= hp_ref.LD(hp_ref.gamma(E.shape[0] + 1)) * M.astype(hp_ref.LD)))


def normwise_ok(A, R, s, kappa_max, res=None):
    """||A - R^ S R^T||_F <= gamma_{n+1} (1 + 4 kappa_max) || |R^| |R^T| ||_F over the symmetric matrices (module doc);
    kappa_max = hp_ref.diag_block_kappa(R, nb)"""
    E, M = res if res is not None else residual(A, R, s)
    return bool(np.all(np.isfinite(R)) and hp_ref._sym_frob(E) <= hp_ref.chol_backward_bound(M, kappa_max))


def fits(N, v, Px, Py, depth):
    """cflx_chol_rbt's transform is local to every rank's share when N is a multiple of 2^depth v lcm(Px, Py): the rows
    pair within a rank when 2^depth v Px divides N, the columns when 2^depth v Py does"""
    return N % ((v * math.lcm(Px, Py)) << depth) == 0


def smallest_order(N, v, Px, Py, depth):
    """the smallest N' >= N that fits (the order cflx_chol_rbt's refusal names): pad A with the identity to it"""
    q = (v * math.lcm(Px, Py)) << depth
    return -(-N // q) * q


def kkt(n, m, seed=0, c_zero=False):
    """a quasi-definite KKT matrix [[H, B^T], [B, -C]] (lower triangle stored): H (n x n) and C (m x m) SPD, or C = 0 with
    B (m x n) of full row rank; inertia (n, m, 0)"""
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    H = G @ G.T / n + np.eye(n)
    B = rng.standard_normal((m, n))
    K = np.zeros((n + m, n + m))
    K[:n, :n] = H
    K[n:, :n] = B
    K[:n, n:] = B.T
    if not c_zero:
        F = rng.standard_normal((m, m))
        K[n:, n:] = -(F @ F.T / m + np.eye(m))
    return K


def with_inertia(n, npos, nneg, seed=0, lo=0.5, hi=2.0):
    """Q diag(lambda) Q^T with npos positive and nneg negative eigenvalues of magnitude in [lo, hi] (the rest zero), Q
    a random orthogonal matrix"""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = np.zeros(n)
    mag = rng.uniform(lo, hi, npos + nneg)
    lam[:npos] = mag[:npos]
    lam[npos:npos + nneg] = -mag[npos:]
    lam = rng.permutation(lam)
    A = (Q * lam) @ Q.T
    return (A + A.T) / 2
