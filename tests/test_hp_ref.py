"""CPU: the extended-precision references of oracle/hp_ref.py are accurate, and each error-bound check they provide is
sharp: it accepts a correctly rounded float64 restatement of the algorithm and rejects the same computation with one
realistic defect (a term dropped from one trailing update, one wrong entry in one inverse block, a one-column shift in
one 32-column block)."""
from fractions import Fraction

import numpy as np
import pytest
import scipy.linalg

from oracle import hp_ref as hp

LD = hp.LD


def _chol64(A, drop=None):
    """right-looking Cholesky in float64, 32-column blocks like potrf_tile_kernel; drop = (i, j, k): leave the term
    L[i,k] L[j,k] out of the update of entry (i, j)"""
    S = np.tril(np.array(A, dtype=np.float64))
    n = S.shape[0]
    for k in range(n):
        S[k, k] = np.sqrt(S[k, k])
        S[k + 1:, k] /= S[k, k]
        upd = np.tril(np.outer(S[k + 1:, k], S[k + 1:, k]))
        if drop is not None and drop[2] == k:
            upd[drop[0] - k - 1, drop[1] - k - 1] = 0.0
        S[k + 1:, k + 1:] -= upd
    return np.tril(S)


def _inv_upper64(U, drop=None):
    """inv(U) by substitution, column by column, in float64; drop = (r, c, t): leave U[r,t] X[t,c] out of entry (r, c)"""
    n = U.shape[0]
    X = np.zeros((n, n))
    for c in range(n):
        X[c, c] = 1.0 / U[c, c]
        for r in range(c - 1, -1, -1):
            terms = U[r, r + 1:c + 1] * X[r + 1:c + 1, c]
            if drop is not None and drop[:2] == (r, c):
                terms[drop[2] - r - 1] = 0.0
            X[r, c] = -terms.sum() / U[r, r]
    return X


def test_matmul_is_exact_to_extended_precision():
    rng = np.random.default_rng(0)
    X = rng.standard_normal((6, 300)) * np.logspace(-3, 3, 300)
    Y = rng.standard_normal((300, 5))
    C = hp.matmul(X, Y)
    for i in range(6):
        for j in range(5):
            exact = sum(Fraction(float(a)) * Fraction(float(b)) for a, b in zip(X[i], Y[:, j]))
            scale = Fraction(float(np.abs(X[i]) @ np.abs(Y[:, j])))
            assert abs(Fraction(float(C[i, j])) + Fraction(float(C[i, j] - LD(float(C[i, j])))) - exact) <= scale * Fraction(2) ** -62


def test_longdouble_cholesky_and_inverse_are_extended_precision():
    rng = np.random.default_rng(1)
    A = hp.random_spd(300, 1e6, rng)
    L, info = hp.cholesky(A, block=64)
    assert info == 0
    R = np.abs(np.tril(A.astype(LD) - L @ L.T))          # longdouble matmul: slow, but exact enough at n = 300
    assert np.all(R <= LD(2.0 ** -64 * 4 * 300) * np.tril(np.abs(L) @ np.abs(L).T))
    X = hp.tri_inverse(L, lower=True)
    assert np.all(np.abs(L @ X - np.eye(300, dtype=LD)) <= LD(2.0 ** -64 * 4 * 300) * (np.abs(L) @ np.abs(X)))
    # and the factor is the one LAPACK approximates
    assert np.abs(np.asarray(L, dtype=np.float64) - np.linalg.cholesky(A)).max() <= 1e-9


def test_exact_input_is_factored_exactly():
    rng = np.random.default_rng(2)
    A, L0 = hp.exact_spd(96, rng)
    L, info = hp.cholesky(A, block=32)
    assert info == 0 and np.array_equal(np.asarray(L, dtype=np.float64), L0)
    assert np.array_equal(_chol64(A), L0)


@pytest.mark.parametrize("k0", [0, 37, 95])
def test_not_positive_definite_info_is_lapacks(k0):
    rng = np.random.default_rng(3)
    A, L0 = hp.exact_spd(96, rng)
    A[k0, k0] -= L0[k0, k0] ** 2 + 0.5
    assert hp.cholesky(A, block=32)[1] == k0 + 1 == scipy.linalg.lapack.dpotrf(A, lower=1)[1]


def test_cholesky_checks_accept_float64_and_reject_a_dropped_update_term():
    rng = np.random.default_rng(4)
    n = 160
    A = hp.random_spd(n, 1e4, rng)
    Lref, _ = hp.cholesky(A)
    L = _chol64(A)
    kmax = hp.diag_block_kappa(L, 32)
    assert hp.chol_componentwise_ok(A, L) and hp.chol_normwise_ok(A, L, kmax) and hp.chol_forward_ok(A, L, Lref, kmax)
    Lbad = _chol64(A, drop=(120, 70, 40))                  # one term of one trailing update missing
    assert not hp.chol_componentwise_ok(A, Lbad)
    assert not hp.chol_normwise_ok(A, Lbad, kmax)
    assert not hp.chol_forward_ok(A, Lbad, Lref, kmax)


def test_cholesky_checks_reject_a_one_column_shift_in_one_block():
    rng = np.random.default_rng(5)
    n = 128
    A = hp.random_spd(n, 1e2, rng)
    L = _chol64(A)
    Lbad = L.copy()
    Lbad[64:, 33:64] = L[64:, 32:63]                       # the block below diagonal block 1 stored one column right
    kmax = hp.diag_block_kappa(L, 32)
    assert hp.chol_componentwise_ok(A, L)
    assert not hp.chol_componentwise_ok(A, Lbad)
    assert not hp.chol_normwise_ok(A, Lbad, kmax)


def test_transposed_factor_is_rejected():
    rng = np.random.default_rng(6)
    A = hp.random_spd(64, 10.0, rng)
    L = _chol64(A)
    assert not hp.chol_componentwise_ok(A, L.T)


@pytest.mark.parametrize("kind", ["plain", "graded"])
def test_inverse_check_accepts_substitution_and_rejects_one_wrong_entry(kind):
    rng = np.random.default_rng(7)
    n = 64
    U = np.triu(rng.uniform(-1, 1, (n, n))) * 0.2 + np.diag(1.0 + rng.random(n))
    if kind == "graded":
        U = np.logspace(-6, 6, n)[:, None] * U
    X = _inv_upper64(U)
    assert hp.inverse_componentwise_ok(U, X)
    Xlong = hp.tri_inverse(U, lower=False)
    assert np.abs(X - np.asarray(Xlong, dtype=np.float64)).max() <= 1e-10 * np.abs(X).max()
    assert not hp.inverse_componentwise_ok(U, _inv_upper64(U, drop=(10, 40, 25)))
    Xbad = X.copy()
    Xbad[5, 50] *= 1 + 2.0 ** -30                          # one entry off at the 2^-30 level
    assert not hp.inverse_componentwise_ok(U, Xbad)


# ------------------------------------------------------------------------------------------------ the LU path
def _lu64(A, drop=None):
    """right-looking LU with partial pivoting in float64 (n x v: a panel), like LAPACK's dgetf2; drop = (i, j, k): leave
    the term l_ik u_kj out of the update of entry (i, j) (pivoted positions).  Returns (L\\U packed, perm)."""
    S = np.array(A, dtype=np.float64)
    n, v = S.shape
    perm = np.arange(n)
    for k in range(min(n, v)):
        p = k + int(np.argmax(np.abs(S[k:, k])))
        S[[k, p]] = S[[p, k]]
        perm[[k, p]] = perm[[p, k]]
        S[k + 1:, k] /= S[k, k]
        upd = np.outer(S[k + 1:, k], S[k, k + 1:])
        if drop is not None and drop[2] == k:
            upd[drop[0] - k - 1, drop[1] - k - 1] = 0.0
        S[k + 1:, k + 1:] -= upd
    return S, perm


def _lapack_lu(A):
    """scipy's dgetrf factor with its row interchanges turned into perm (perm[i] = original row at position i)"""
    lu, piv = scipy.linalg.lu_factor(A)
    perm = np.arange(A.shape[0])
    for i, p in enumerate(piv):
        perm[[i, p]] = perm[[p, i]]
    return lu, perm


def _lu_defects(LU, perm, v):
    """one wrong entry, a one-column shift in the second half of U, two swapped entries of perm"""
    wrong = LU.copy()
    wrong[v // 2 + 3, v // 3] *= 1 + 2.0 ** -30
    shift = LU.copy()
    shift[:v // 2, v // 2 + 1:v] = LU[:v // 2, v // 2:v - 1]
    swapped = perm.copy()
    swapped[[2, v - 2]] = swapped[[v - 2, 2]]
    return [(wrong, perm), (shift, perm), (LU, swapped)]


@pytest.mark.parametrize("n,v", [(96, 96), (300, 32), (160, 12)])
def test_lu_checks_accept_lapack_and_elimination_and_reject_defects(n, v):
    rng = np.random.default_rng(n + v)
    A = rng.standard_normal((n, v))
    for LU, perm in (_lu64(A), _lapack_lu(A)):
        assert hp.lu_componentwise_ok(A, LU, perm)
        assert hp.lu_normwise_ok(A, LU, perm, hp.lu_kappa_max(LU, 4, upper=True))
    LU, perm = _lu64(A)
    LUd, permd = _lu64(A, drop=(v - 1, v - 2, v // 2))       # one term of one update missing
    assert np.array_equal(perm, permd)
    kmax = hp.lu_kappa_max(LU, 4)                             # one process row: only L's blocks are inverted
    for i, (bad, p) in enumerate([(LUd, permd)] + _lu_defects(LU, perm, v)):
        assert not hp.lu_componentwise_ok(A, bad, p), i
        assert not hp.lu_normwise_ok(A, bad, p, kmax), i


def test_lu_residual_of_a_panel_is_rectangular():
    rng = np.random.default_rng(11)
    A = rng.standard_normal((40, 8))
    LU, perm = _lu64(A)
    R, M = hp.lu_residual(A, LU, perm)
    assert R.shape == M.shape == (40, 8)
    L, U = hp.lu_unpack(LU)
    assert L.shape == (40, 8) and U.shape == (8, 8)
    assert np.abs(np.asarray(R, dtype=np.float64)).max() <= 8 * 2.0 ** -53 * M.max()


@pytest.mark.parametrize("kind", ["normal", "graded"])
def test_gemm_check_accepts_float64_and_rejects_defects(kind):
    rng = np.random.default_rng(12)
    K, M, N = 256, 70, 64
    AT = rng.uniform(-1, 1, (K, M))
    B = rng.standard_normal((K, N))
    if kind == "graded":                                      # multipliers 1, 1e-3, 1e-7; U rows over 2^+-30
        AT *= rng.choice([1.0, 1e-3, 1e-7], size=(K, M))
        B *= np.exp2(rng.integers(-30, 31, (K, 1)).astype(np.float64))
    C = rng.standard_normal((M, N))
    for alpha, beta in [(-1.0, 1.0), (1.0, 0.0), (0.5, -2.0)]:
        D = beta * C + alpha * (AT.T @ B)
        assert hp.gemm_ok(AT, B, C, alpha, beta, D)
        if beta == 0:
            assert hp.gemm_ok(AT, B, np.full_like(C, np.nan), alpha, beta, D)      # C is not read
        drop = D.copy()                                        # the smallest term the bound can see, left out
        t = np.abs(AT[:, 5] * B[:, 7])
        seen = 2 * hp.gamma(K + 1) * (abs(beta * C[5, 7]) + np.sum(t))
        k = int(np.argmin(np.where(t > seen, t, np.inf)))
        drop[5, 7] -= alpha * AT[k, 5] * B[k, 7]
        wrong = D.copy()
        wrong[40, 33] *= 1 + 2.0 ** -30
        shift = D.copy()
        shift[:, 33:64] = D[:, 32:63]
        swapped = D.copy()
        swapped[[3, 60]] = D[[60, 3]]
        for bad in (drop, wrong, shift, swapped):
            assert not hp.gemm_ok(AT, B, C, alpha, beta, bad)


def _inv_sweep_lower_unit(L, R, nb):
    """inv(L) R in float64 the way trsm_left_lower_unit runs it: the inverse of each diagonal block, then the block
    row's product and the update of the rows below"""
    v = L.shape[0]
    R = R.copy()
    Y = np.zeros_like(R)
    for j in range(0, v, nb):
        W = scipy.linalg.solve_triangular(L[j:j + nb, j:j + nb], np.eye(nb), lower=True, unit_diagonal=True)
        Y[j:j + nb] = W @ R[j:j + nb]
        R[j + nb:] -= L[j + nb:, j:j + nb] @ Y[j:j + nb]
    return Y


@pytest.mark.parametrize("v,nb", [(128, 32), (96, 4)])
def test_trsm_checks_accept_the_blocked_solve_and_reject_defects(v, nb):
    rng = np.random.default_rng(v + nb)
    n = 80
    L = np.tril(rng.uniform(-1, 1, (v, v)), -1) * (2 / np.sqrt(v)) + np.eye(v)
    U = np.triu(rng.uniform(-1, 1, (v, v))) * (2 / np.sqrt(v)) + np.diag(1 + rng.random(v))
    R = rng.standard_normal((v, n))
    B = rng.standard_normal((n, v))
    kL = hp.diag_block_kappa(L, nb)
    kU = hp.diag_block_kappa(U, nb)
    Y = _inv_sweep_lower_unit(L, R, nb)
    d = np.diag(U)                                            # X U = B: U^T = (U^T D^-1) D, unit lower times diagonal
    X = (_inv_sweep_lower_unit(U.T / d, B.T, nb) / d[:, None]).T
    assert hp.trsm_lower_unit_ok(L, R, Y, kL)
    assert hp.trsm_lower_unit_ok(L, R, scipy.linalg.solve_triangular(L, R, lower=True, unit_diagonal=True), kL)
    assert hp.trsm_upper_ok(U, B, X, kU)
    assert hp.trsm_upper_ok(U, B, scipy.linalg.solve_triangular(U.T, B.T, lower=True).T, kU)
    for sol, ok, lhs, rhs, k in ((Y, hp.trsm_lower_unit_ok, L, R, kL), (X.T, lambda T, Bt, Xt, k: hp.trsm_upper_ok(
            T, Bt.T, Xt.T, k), U, B.T, kU)):
        wrong = sol.copy()
        wrong[v // 2, 7] += 1e-9 * np.abs(sol).max()
        shift = sol.copy()
        shift[:, 41:80] = sol[:, 40:79]
        swapped = sol.copy()
        swapped[[3, v - 5]] = sol[[v - 5, 3]]
        for bad in (wrong, shift, swapped):
            assert not ok(lhs, rhs, bad, k)
    Ld = L.copy()                                             # one term of one block update missing
    Ld[v - 1, 0] = 0.0
    assert not hp.trsm_lower_unit_ok(L, R, _inv_sweep_lower_unit(Ld, R, nb), kL)


def _inv_sweep(T, R, nb):
    """inv(T) R in float64 the way the solve engine's diagonal-tile sweep runs it: blocks in elimination order, each the
    product with the inverse of its diagonal block, then the update of the blocks still to solve"""
    v = T.shape[0]
    lower = not np.triu(T, 1).any()
    R = R.copy()
    Y = np.zeros_like(R)
    for j in (range(0, v, nb) if lower else range(v - nb, -1, -nb)):
        b = slice(j, j + nb)
        Y[b] = np.linalg.inv(T[b, b]) @ R[b]
        rest = slice(j + nb, v) if lower else slice(0, j)
        R[rest] -= T[rest, b] @ Y[b]
    return Y


@pytest.mark.parametrize("form", ["lower", "upper", "lower_t", "unit_lower_t", "upper_t"])
def test_left_trsm_check_accepts_the_block_sweep_and_rejects_defects(form):
    v, nb, n = 128, 16, 24
    rng = np.random.default_rng(len(form))
    L = np.tril(rng.uniform(-1, 1, (v, v)), -1) * (2 / np.sqrt(v)) + np.diag(1 + rng.random(v))
    U = np.triu(rng.uniform(-1, 1, (v, v)), 1) * (2 / np.sqrt(v)) + np.diag(1 + rng.random(v))
    Lu = np.tril(L, -1) + np.eye(v)
    T = {"lower": L, "upper": U, "lower_t": L.T, "unit_lower_t": Lu.T, "upper_t": U.T}[form]
    lower = not np.triu(T, 1).any()
    R = rng.standard_normal((v, n))
    Y = _inv_sweep(T, R, nb)
    assert hp.trsm_left_ok(T, R, Y, nb)
    assert hp.trsm_left_ok(T, R, scipy.linalg.solve_triangular(T, R, lower=lower), nb)
    wrong = Y.copy()
    wrong[v // 2, 7] += 1e-9 * np.abs(Y).max()
    shift = Y.copy()
    shift[:, 1:] = Y[:, :-1]
    for bad in (wrong, shift):
        assert not hp.trsm_left_ok(T, R, bad, nb)
    Td = T.copy()                                             # one term of one block update missing
    Td[(v - 1, 0) if lower else (0, v - 1)] = 0.0
    assert not hp.trsm_left_ok(T, R, _inv_sweep(Td, R, nb), nb)


def test_power_of_two_grading_commutes_with_the_factorisation():
    """the property the graded GPU test relies on: for D = diag(2^k), the float64 factor of D S D is D times the float64
    factor of S, bit for bit (in every order of summation; shown here for the right-looking restatement)"""
    rng = np.random.default_rng(8)
    n = 96
    S = hp.random_spd(n, 1e2, rng)
    d = 2.0 ** np.round(np.linspace(-10, 10, n))
    assert np.array_equal(_chol64(d[:, None] * S * d[None, :]), d[:, None] * _chol64(S))
