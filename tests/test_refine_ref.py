"""CPU: oracle/refine_ref.py, the restatement of cflx_lu_refine / cflx_chol_refine.

  * gerfs / porfs against scipy's dgesvx(fact='F', equed='N') / dposvx(fact='F', equed='N', lower=1) on the same factors,
    started from the same X (LAPACK's own getrs / potrs solution, which dgesvx / dposvx refine).  The two take the same
    decisions on the same data; what differs is the rounding of the residual products (numpy's BLAS against LAPACK's
    dgemv order).  After refinement |r| is itself at the rounding level, so berr (~u) is compared to within 1e-6 relative
    plus u.  ferr scales with w = |r| + (n + 1) u (|A| |x| + |b|): the products' rounding moves |r| by up to ~n u s_i,
    a fraction of w_i, so ferr is compared to 1e-2 relative (observed: below 1e-3).  Matrices: random, row- or
    column-scaled over 1e12, and kappa ~ 1e8 (rcond > eps, so dgesvx returns info 0);
  * the rank-by-rank grid product equals the dense op(A) X and |op(A)| |X| (to a few ulps of |op(A)| |X|) on the LU grids
    1x1x1, 2x2x1, 2x2x2, 3x3x1 and a padded case, and for the Cholesky on 1x1x1, 2x1x1, 2x2x1, 3x2x1 and 1x3x2 with NaN in
    every entry the device must not read."""
import numpy as np
import pytest
from scipy.linalg import cho_factor, lu_factor

from oracle import chol_ref, chol_solve_ref, layout
from oracle import refine_ref as rr

U = 2.0 ** -53


def _matrix(n, kind, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    s = np.logspace(0, 12, n)
    rng.shuffle(s)
    if kind == "rows":
        A = A * s[:, None]
    elif kind == "cols":
        A = A * s[None, :]
    elif kind == "kappa":
        Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
        Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
        A = (Q1 * np.logspace(0, -8, n)) @ Q2.T
    return A


def _close(a, b, what, rel=1e-6):
    assert np.all(np.abs(a - b) <= rel * np.maximum(np.abs(a), np.abs(b)) + U), (what, a, b)


@pytest.mark.parametrize("kind", ["random", "rows", "cols", "kappa"])
def test_gerfs_matches_dgesvx(kind):
    n = 128
    A = _matrix(n, kind, 1)
    B = np.random.default_rng(2).standard_normal((n, 3))
    LU, piv = lu_factor(A)
    perm = np.arange(n)
    for i, p in enumerate(piv):
        perm[[i, p]] = perm[[p, i]]
    ipiv = rr.perm_to_ipiv(perm)
    assert np.array_equal(ipiv, piv + 1)
    Xl, fe_l, be_l, info = rr.lapack_gesvx(A, LU, ipiv, B)
    assert info == 0
    solve, solve_t = rr.lu_solvers(LU, perm)
    X, fe, be = rr.gerfs(A, B, solve(B), solve, solve_t)
    _close(be, be_l, "berr")
    _close(fe, fe_l, "ferr", 1e-2)


def test_gerfs_transposed_matches_dgesvx():
    n = 128
    A = _matrix(n, "random", 3)
    B = np.random.default_rng(4).standard_normal((n, 2))
    LU, piv = lu_factor(A)
    perm = np.arange(n)
    for i, p in enumerate(piv):
        perm[[i, p]] = perm[[p, i]]
    Xl, fe_l, be_l, info = rr.lapack_gesvx(A, LU, piv + 1, B, trans=True)
    assert info == 0
    solve, solve_t = rr.lu_solvers(LU, perm, trans=True)
    X, fe, be = rr.gerfs(A, B, solve(B), solve, solve_t, trans=True)
    _close(be, be_l, "berr")
    _close(fe, fe_l, "ferr", 1e-2)


@pytest.mark.parametrize("kind", ["random", "scaled", "kappa"])
def test_porfs_matches_dposvx(kind):
    n = 128
    rng = np.random.default_rng(5)
    G = rng.standard_normal((n, n))
    A = G @ G.T + n * np.eye(n)
    if kind == "scaled":
        s = np.logspace(0, 6, n)
        A = A * s[:, None] * s[None, :]
    elif kind == "kappa":
        Q, _ = np.linalg.qr(G)
        A = (Q * np.logspace(0, -8, n)) @ Q.T
        A = (A + A.T) / 2
    B = rng.standard_normal((n, 3))
    L = np.tril(cho_factor(A, lower=True)[0])
    Xl, fe_l, be_l, info = rr.lapack_posvx(A, L, B)
    assert info == 0
    solve = rr.chol_solver(L)
    X, fe, be = rr.porfs(A, B, solve(B), solve)
    _close(be, be_l, "berr")
    _close(fe, fe_l, "ferr", 1e-2)


@pytest.mark.parametrize("N,v,Px,Py,Pz", [(64, 8, 1, 1, 1), (64, 8, 2, 2, 1), (64, 8, 2, 2, 2), (72, 8, 3, 3, 1),
                                          (100, 16, 2, 2, 1)])
@pytest.mark.parametrize("trans", [False, True])
def test_grid_product_lu(N, v, Px, Py, Pz, trans):
    d = layout.dims(N, v, Px, Py, Pz)
    rng = np.random.default_rng(N + Px)
    A = rng.standard_normal((d["M"], d["M"]))
    X = rng.standard_normal((d["M"], 3))
    P, Q = rr.partials_lu(layout.scatter(A, v, Px, Py, Pz), X, N, v, Px, Py, Pz, trans)
    Ao = A.T if trans else A
    tol = 8 * d["M"] * U * (np.abs(Ao) @ np.abs(X))
    assert np.all(np.abs(P - Ao @ X) <= tol) and np.all(np.abs(Q - np.abs(Ao) @ np.abs(X)) <= tol)


@pytest.mark.parametrize("N,v,grid", [(64, 8, (1, 1, 1)), (64, 8, (2, 1, 1)), (96, 8, (2, 2, 1)), (96, 8, (3, 2, 1)),
                                      (72, 8, (1, 3, 2))])
def test_grid_product_chol(N, v, grid):
    d = chol_ref.dims(N, v, *grid)
    n = d["N"]
    rng = np.random.default_rng(N)
    G = rng.standard_normal((n, n))
    A = G + G.T
    X = rng.standard_normal((n, 4))
    locs = chol_solve_ref.scatter(A, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)
    P, Q = rr.partials_chol(locs, X, N, v, *grid)
    tol = 8 * n * U * (np.abs(A) @ np.abs(X))
    assert np.all(np.isfinite(P)) and np.all(np.isfinite(Q))
    assert np.all(np.abs(P - A @ X) <= tol) and np.all(np.abs(Q - np.abs(A) @ np.abs(X)) <= tol)
