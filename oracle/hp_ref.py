"""oracle/hp_ref.py -- TEST INFRASTRUCTURE: extended-precision references for the Cholesky path and the triangular
inverses, and the error bounds the GPU results are checked against.

Everything here is computed in np.longdouble (x87 extended, 64-bit significand, unit roundoff 2^-64) or exactly, so the
reference's own error is ~2^11 times below the float64 rounding it judges.  numpy's linalg has no longdouble support,
and a longdouble matmul runs at ~10^8 multiply-adds per second, so the O(n^3) products go through `matmul`: an
error-free slicing of both operands into float64 pieces of beta significant bits (Ozaki's scheme), whose float64 BLAS
products are exact, summed in longdouble.

Bounds (u = 2^-53, gamma_n = n u / (1 - n u); Higham, "Accuracy and Stability of Numerical Algorithms", 2nd ed.):
  * triangular inverse by substitution, any summation order (Sec. 14.2):  |T X^ - I| <= gamma_n |T| |X^|
  * Cholesky by substitution, any summation order (Thm 10.3):            |A - L^ L^T| <= gamma_{n+1} |L^| |L^T|
  * a panel solved with an explicit inverse of its nb x nb diagonal blocks (the 128-block tile driver, the panel TRSM of
    the factorisation): the inverse has the componentwise error above, the product with it one more gamma_nb; moving
    them to the residual multiplies by kappa_2(L_d), so the normwise backward error is bounded by
        ||A - L^ L^T||_F <= gamma_{n+1} (1 + 4 kappa_max) || |L^| |L^T| ||_F,
    kappa_max = the largest 2-norm condition number of an inverted diagonal block.  The first-order analysis gives
    2 kappa_max (one term per rounding); the factor 2 on top is a chosen margin for the second-order terms it drops, so
    this bound is a worst-case normwise one and loose by design.  The sharp checks are the componentwise ones on the
    kernels, and the bit-for-bit pins of the default path (tests/golden/chol_factor_bits.json);
  * forward error (Sun 1991): L^ is the exact factor of A + dA with dA = L^ L^T - A, so
        ||L^ - L||_F / ||L||_2 <= kappa_2(A) eps / (1 - kappa_2(A) eps),   eps = (the bound above on ||dA||_F) / ||A||_2
    (Sun's constant is 2^-1/2; 1 is used).

The LU path (gemm_ok, lu_*_ok, trsm_*_ok):
  * the update GEMM D = fl(alpha acc + fl(beta c)), acc = AT^T B summed in any order (Sec. 3.5, Lemma 3.3):
        |D^ - (beta C + alpha A^T B)| <= gamma_{K+1} (|beta| |C| + |alpha| |A|^T |B|)      (derivation: gemm_ok)
  * a panel factored by elimination, any summation order (Thm 9.3, rectangular n x v form):
        |P A - L^ U^| <= gamma_v |L^| |U^|
  * a factorisation whose U rows (and, with more than one process row, L panels) are solved with inverted nb x nb
    diagonal blocks: the same argument as the Cholesky bound above,
        ||P A - L^ U^||_F <= gamma_{n+1} (1 + 4 kappa_max) || |L^| |U^| ||_F,
    kappa_max over the unit-lower diagonal blocks and, where the L panel is solved (trsm_right_upper_T), the upper ones;
  * the two TRSMs (X U = B, L Y = R with inverted diagonal blocks of U, unit-lower L):
        ||X^ U - B||_F <= gamma_{v+1} (1 + 4 kappa_max) || |X^| |U| ||_F,   ||L Y^ - R||_F <= the same with |L| |Y^|."""
import numpy as np

LD = np.longdouble
U64 = 2.0 ** -53


def gamma(n):
    return n * U64 / (1.0 - n * U64)


# ------------------------------------------------------------------------------------------------ exact products
def _slices(X, axis, beta, count):
    """X (float64 or longdouble) = sum of `count` float64 slices + a remainder below 2^(e - beta*count), e the exponent of
    the largest magnitude along `axis` (rows of a left operand, columns of a right one).  Every slice is an integer
    multiple of 2^(e - beta*(i+1)) below 2^(e - beta*i): beta bits, so it converts to float64 exactly.  (Scaling by a
    power of two, truncation and the subtraction of a truncated part are exact in either type.)"""
    X = np.asarray(X)
    R = X.copy() if X.dtype == LD else np.asarray(X, dtype=np.float64).copy()
    mx = np.max(np.abs(R), axis=axis, keepdims=True)
    e = np.where(mx > 0, np.frexp(mx)[1], 0).astype(np.int64)
    out = []
    for i in range(count):
        unit = np.ldexp(np.ones(e.shape, dtype=R.dtype), e - beta * (i + 1))
        S = np.trunc(R / unit) * unit
        R = R - S
        out.append(S.astype(np.float64))
    return out


def matmul(X, Y, count=4):
    """X @ Y in longdouble, accurate to ~2^-70 of |X| |Y| elementwise: the products of the float64 slices are exact, the
    leading one is added in longdouble, the rest (below 2^-beta of it) are summed in float64."""
    X, Y = np.asarray(X), np.asarray(Y)
    k = X.shape[1]
    beta = (53 - int(np.ceil(np.log2(max(k, 2))))) // 2      # 2 beta + log2(k) <= 53: every slice product is exact
    assert beta * count >= 70, "too few slices for an extended-precision product"
    Xs = _slices(X, 1, beta, count)
    Ys = _slices(Y, 0, beta, count)
    rest = np.zeros((X.shape[0], Y.shape[1]))
    for i in range(count):
        for j in range(count - i):
            if i + j:
                rest += Xs[i] @ Ys[j]
    return (Xs[0] @ Ys[0]).astype(LD) + rest.astype(LD)


# ------------------------------------------------------------------------------------------------ factorisations
def cholesky(A, block=128):
    """Lower Cholesky factor of the symmetric matrix whose lower triangle is A, in longdouble (blocked right-looking;
    the trailing updates through `matmul`).  Returns (L, info) with info = 1 + the first non-positive pivot, 0 = success,
    like LAPACK's dpotrf."""
    S = np.tril(np.asarray(A, dtype=LD))
    S = S + np.tril(S, -1).T
    n = S.shape[0]
    L = np.zeros((n, n), dtype=LD)
    for j0 in range(0, n, block):
        j1 = min(n, j0 + block)
        for j in range(j0, j1):                       # diagonal block, column by column
            d = S[j, j] - L[j, j0:j] @ L[j, j0:j]
            if not d > 0:
                return L, j + 1
            L[j, j] = np.sqrt(d)
            L[j + 1:j1, j] = (S[j + 1:j1, j] - L[j + 1:j1, j0:j] @ L[j, j0:j]) / L[j, j]
        if j1 < n:                                    # rows below: X L_d^T = P by substitution, all rows at once
            P = S[j1:, j0:j1]
            X = np.zeros_like(P)
            for c in range(j1 - j0):
                X[:, c] = (P[:, c] - X[:, :c] @ L[j0 + c, j0:j0 + c]) / L[j0 + c, j0 + c]
            L[j1:, j0:j1] = X
            S[j1:, j1:] -= matmul(X, X.T)
    return L, 0


def tri_inverse(T, lower, unit=False):
    """inv(T) of a triangular T in longdouble by substitution (row by row of the inverse)."""
    T = np.asarray(T, dtype=LD)
    n = T.shape[0]
    X = np.zeros((n, n), dtype=LD)
    I = np.eye(n, dtype=LD)
    rows = range(n) if lower else range(n - 1, -1, -1)
    for r in rows:
        lo, hi = (0, r) if lower else (r + 1, n)
        s = I[r] - T[r, lo:hi] @ X[lo:hi]
        X[r] = s if unit else s / T[r, r]
    return X


# ------------------------------------------------------------------------------------------------ residuals, checks
# |L^| |L^T| and |T| |X^| only scale the bounds; they are formed in float64 (nonnegative terms: relative error <= gamma_n).
def chol_residual(A, L):
    """(|A - L L^T| in longdouble, |L| |L^T| in float64), lower triangles (A: lower triangle read)"""
    L = np.tril(np.asarray(L, dtype=np.float64))
    R = np.abs(np.tril(np.tril(np.asarray(A, dtype=np.float64)).astype(LD) - matmul(L, L.T)))
    aL = np.abs(L)
    return R, np.tril(aL @ aL.T)


def _sym_frob(T):
    T = np.asarray(T)
    return float(np.sqrt(2 * np.sum(T * T) - np.sum(np.diag(T) ** 2)))


def chol_componentwise_ok(A, L, res=None):
    """Higham Thm 10.3: |A - L^ L^T| <= gamma_{n+1} |L^| |L^T| in every entry of the lower triangle."""
    R, M = res if res is not None else chol_residual(A, L)
    return bool(np.all(np.isfinite(L)) and np.all(R <= LD(gamma(R.shape[0] + 1)) * M.astype(LD)))


def diag_block_kappa(L, nb):
    """largest 2-norm condition number of the nb x nb diagonal blocks of L"""
    L = np.asarray(L, dtype=np.float64)
    return max(np.linalg.cond(L[i:i + nb, i:i + nb]) for i in range(0, L.shape[0], nb))


def chol_backward_bound(M, kappa_max):
    """bound on ||A - L^ L^T||_F of a factorisation whose panels are solved with inverted diagonal blocks (module doc);
    M = |L^| |L^T| (lower triangle)"""
    return gamma(M.shape[0] + 1) * (1.0 + 4.0 * kappa_max) * _sym_frob(M)


def chol_normwise_ok(A, L, kappa_max, res=None):
    R, M = res if res is not None else chol_residual(A, L)
    return bool(np.all(np.isfinite(L)) and _sym_frob(R) <= chol_backward_bound(M, kappa_max))


def chol_forward_ok(A, L, Lref, kappa_max, res=None):
    """||L^ - L||_F / ||L||_2 <= kappa_2(A) eps / (1 - kappa_2(A) eps), eps = the backward bound over ||A||_2 (Sun's
    first-order bound; module doc).  Lref: the longdouble factor."""
    _, M = res if res is not None else chol_residual(A, L)
    S = np.tril(np.asarray(A, dtype=np.float64))
    ev = np.linalg.eigvalsh(S + np.tril(S, -1).T)
    kappa = ev[-1] / ev[0]
    eps = chol_backward_bound(M, kappa_max) / ev[-1]
    assert kappa * eps < 0.5, "the forward bound needs kappa(A) * eps < 1/2"
    err = float(np.sqrt(np.sum((np.tril(np.asarray(L, dtype=np.float64)).astype(LD) - Lref) ** 2)))
    return err <= np.sqrt(ev[-1]) * kappa * eps / (1.0 - kappa * eps)


def inverse_componentwise_ok(T, X):
    """Higham Sec. 14.2: |T X^ - I| <= gamma_n |T| |X^| in every entry (T triangular, X^ its computed inverse)."""
    T = np.asarray(T, dtype=np.float64)
    X = np.asarray(X, dtype=np.float64)
    n = T.shape[0]
    R = np.abs(matmul(T, X) - np.eye(n, dtype=LD))
    M = np.abs(T) @ np.abs(X)
    return bool(np.all(np.isfinite(X)) and np.all(R <= LD(gamma(n)) * M.astype(LD)))


# ------------------------------------------------------------------------------------------------ the LU path
def gemm_ok(AT, B, C, alpha, beta, D):
    """Componentwise bound of gemm_tn_kernel's D = beta*C + alpha * AT^T B (AT: K x M, B: K x N; C is not read when
    beta == 0, so it may hold anything there):
        |D^ - (beta C + alpha A^T B)| <= gamma_{K+1} (|beta| |C| + |alpha| |A|^T |B|).
    Derivation.  The accumulator acc is the K-term dot product summed in some order with fma or separate roundings:
    |acc - A^T B| <= gamma_K |A|^T |B| (Higham Sec. 3.5).  The epilogue forms t = fl(beta c) = beta c (1 + d1) and
    D^ = fma(alpha, acc, t) = (alpha acc + t)(1 + d2), |d1|, |d2| <= u.  So
        D^ - (beta c + alpha a^T b) = alpha (acc - a^T b)(1 + d2) + alpha a^T b d2 + beta c ((1 + d1)(1 + d2) - 1),
    whose terms are bounded by (gamma_K (1 + u) + u) |alpha| |a|^T |b| <= gamma_{K+1} |alpha| |a|^T |b| (Lemma 3.3) and
    gamma_2 |beta| |c| <= gamma_{K+1} |beta| |c|.  A product alpha*acc rounded before the add would be one more rounding:
    still inside this bound, which is why the bit-for-bit tests on exact accumulators are the ones that see it."""
    AT = np.asarray(AT, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    D = np.asarray(D, dtype=np.float64)
    ref = LD(alpha) * matmul(AT.T, B)
    M = abs(alpha) * (np.abs(AT).T @ np.abs(B))
    if beta != 0:
        C = np.asarray(C, dtype=np.float64)
        ref = ref + LD(beta) * C.astype(LD)
        M = M + abs(beta) * np.abs(C)
    R = np.abs(D.astype(LD) - ref)
    return bool(np.all(np.isfinite(D)) and np.all(R <= LD(gamma(AT.shape[0] + 1)) * M.astype(LD)))


def lu_unpack(LU, v=None):
    """(L, U) of a packed L\\U: LU is n x v (a panel, rows in pivoted order) or n x n; L unit lower n x v, U v x v"""
    LU = np.asarray(LU, dtype=np.float64)
    v = LU.shape[1] if v is None else v
    L = np.tril(LU[:, :v], -1) + np.eye(LU.shape[0], v)
    return L, np.triu(LU[:v, :v])


def lu_residual(A, LU, perm):
    """(|P A - L^ U^| in longdouble, |L^| |U^| in float64) with P A = A[perm] (perm[i] = the original row at pivoted
    position i) and L\\U packed in LU, n x v: a whole factor (v = n) or a panel (L^ n x v, U^ v x v)"""
    A = np.asarray(A, dtype=np.float64)
    L, U = lu_unpack(LU)
    # six slices: the product is exact down to 2^-144 of each row's largest multiplier, so tiny multipliers left by near-
    # exact cancellations (integer inputs) are resolved to their last bit, as the componentwise check needs
    R = np.abs(A[np.asarray(perm)].astype(LD) - matmul(L, U, count=6))
    return R, np.abs(L) @ np.abs(U)


def lu_componentwise_ok(A, LU, perm, res=None):
    """Higham Thm 9.3 (the rectangular form): |P A - L^ U^| <= gamma_v |L^| |U^| in every entry, for a panel factored by
    elimination.  Entry (i, j) is a sum of min(i, j) + 1 <= v terms (one division for the L part)."""
    R, M = res if res is not None else lu_residual(A, LU, perm)
    v = np.asarray(LU).shape[1]
    return bool(np.all(np.isfinite(LU)) and np.all(R <= LD(gamma(v)) * M.astype(LD)))


def lu_backward_bound(M, kappa_max):
    """bound on ||P A - L^ U^||_F of a factorisation that solves with inverted diagonal blocks (module doc);
    M = |L^| |U^|"""
    return gamma(M.shape[0] + 1) * (1.0 + 4.0 * kappa_max) * float(np.linalg.norm(M))


def lu_normwise_ok(A, LU, perm, kappa_max, res=None):
    """||P A - L^ U^||_F <= gamma_{n+1} (1 + 4 kappa_max) || |L^| |U^| ||_F (module doc); kappa_max from lu_kappa_max"""
    R, M = res if res is not None else lu_residual(A, LU, perm)
    return bool(np.all(np.isfinite(LU)) and float(np.sqrt(np.sum(R * R))) <= lu_backward_bound(M, kappa_max))


def lu_kappa_max(LU, nb, upper=False):
    """largest condition number of the nb x nb unit-lower diagonal blocks of the packed factor, and with upper=True of
    the upper ones too (the blocks the factorisation inverts)"""
    L, U = lu_unpack(LU)
    k = diag_block_kappa(L[:U.shape[0]], nb)
    return max(k, diag_block_kappa(U, nb)) if upper else k


def trsm_upper_ok(U, B, X, kappa_max):
    """X^ = B inv(U) by trsm_right_upper_T (U v x v upper, B n x v):
        ||X^ U - B||_F <= gamma_{v+1} (1 + 4 kappa_max) || |X^| |U| ||_F,
    kappa_max over U's inverted nb x nb diagonal blocks.  The argument is the one of chol_backward_bound: each block of
    X^ is a product with an inverse that has a componentwise error gamma_nb |inv(U_jj)| |U_jj| |inv(U_jj)| (Sec. 14.2),
    the product adds gamma_nb, and the rank-nb updates gamma_v; moving the first two to the residual multiplies them by
    kappa_2(U_jj), and the factor 2 over the first-order 2 kappa_max covers the second-order terms."""
    U = np.triu(np.asarray(U, dtype=np.float64))
    X = np.asarray(X, dtype=np.float64)
    R = matmul(X, U) - np.asarray(B, dtype=np.float64).astype(LD)
    M = np.abs(X) @ np.abs(U)
    bound = gamma(U.shape[0] + 1) * (1.0 + 4.0 * kappa_max) * float(np.linalg.norm(M))
    return bool(np.all(np.isfinite(X)) and float(np.sqrt(np.sum(R * R))) <= bound)


def trsm_lower_unit_ok(L, R, Y, kappa_max):
    """Y^ = inv(L) R by trsm_left_lower_unit (L v x v unit lower, R v x n): ||L Y^ - R||_F <= gamma_{v+1}
    (1 + 4 kappa_max) || |L| |Y^| ||_F, kappa_max over L's inverted diagonal blocks (argument: trsm_upper_ok)"""
    L = np.tril(np.asarray(L, dtype=np.float64), -1) + np.eye(np.asarray(L).shape[0])
    Y = np.asarray(Y, dtype=np.float64)
    Res = matmul(L, Y) - np.asarray(R, dtype=np.float64).astype(LD)
    M = np.abs(L) @ np.abs(Y)
    bound = gamma(L.shape[0] + 1) * (1.0 + 4.0 * kappa_max) * float(np.linalg.norm(M))
    return bool(np.all(np.isfinite(Y)) and float(np.sqrt(np.sum(Res * Res))) <= bound)


def trsm_left_ok(T, R, Y, nb):
    """Y^ = inv(T) R by the solve engine's diagonal-tile sweep (T v x v triangular, as given: lower or upper, unit or not,
    a factor or its transpose; R v x n):
        ||T Y^ - R||_F <= gamma_{v+1} (1 + 4 kappa_max) || |T| |Y^| ||_F,
    kappa_max over T's nb x nb diagonal blocks.  Derivation.  The sweep takes the blocks j in the order of elimination
    (down for a lower T, up for an upper one): Y_j = fl(Xi_j R'_j) with Xi_j the cached inverse of T_jj, then
    R'_i = fl(R'_i - T_ij Y_j) for the blocks i still to solve.  Xi_j was formed by substitution, so T_jj Xi_j = I + F_j
    with |F_j| <= gamma_nb |T_jj| |Xi_j| (Sec. 14.2; a transposed or unit T_jj is the same substitution); the product adds
    Y_j = Xi_j R'_j + G_j, |G_j| <= gamma_nb |Xi_j| |R'_j| (Sec. 3.5); the updates are narrow GEMMs with
    gamma_{nb+1} (gemm_ok), and R'_j - R_j gathers at most v - nb of their terms, so the block row j of the residual is
        T_jj Y_j - R'_j + (R'_j - R_j + sum_{i<>j} T_ji Y_i) = F_j R'_j + T_jj G_j + E_j,
    with ||E_j||_F <= gamma_{v+1} || |T| |Y^| ||_F over the sweep.  Since R'_j ~ T_jj Y_j, the first two terms are at
    most gamma_nb kappa_2(T_jj) || |T_jj| |Y_j| ||_F each to first order.  So the bound is that of trsm_upper_ok, with
    the same factor 2 over the first-order 2 kappa_max for the second-order terms; reading T transposed in place
    changes which entries are summed, not how."""
    T = np.asarray(T, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    Res = matmul(T, Y) - np.asarray(R, dtype=np.float64).astype(LD)
    M = np.abs(T) @ np.abs(Y)
    bound = gamma(T.shape[0] + 1) * (1.0 + 4.0 * diag_block_kappa(T, nb)) * float(np.linalg.norm(M))
    return bool(np.all(np.isfinite(Y)) and float(np.sqrt(np.sum(Res * Res))) <= bound)


# ------------------------------------------------------------------------------------------------ test matrices
def random_spd(n, kappa, rng):
    """Q diag(logspace) Q^T with 2-norm condition number kappa (Q Haar-random orthogonal), as float64"""
    Q, R = np.linalg.qr(rng.standard_normal((n, n)))
    Q = Q * np.sign(np.diag(R))
    d = np.logspace(0, -np.log10(kappa), n)
    A = (Q * d) @ Q.T
    return (A + A.T) / 2


def exact_spd(n, rng, lmax=3, dmin=0, dmax=4):
    """A = L L^T with small-integer L (|entries| <= lmax) and diagonal 2^dmin .. 2^(dmax-1): every step of a Cholesky by
    substitution in float64 is exact, so any correct kernel of that kind returns L bit for bit.  (An explicit inverse of
    such an L is not exact, and with the defaults kappa(L) reaches 1e16 at n = 128: the 128-block tile driver wants
    lmax = 1, dmin = 3.)"""
    L = np.tril(rng.integers(-lmax, lmax + 1, (n, n)).astype(np.float64), -1)
    L[np.diag_indices(n)] = 2.0 ** rng.integers(dmin, dmax, n)
    return L @ L.T, L
