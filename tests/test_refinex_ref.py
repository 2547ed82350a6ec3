"""CPU: oracle/refinex_ref.py, the restatement of cflx_lu_refine_x / cflx_chol_refine_x (LAPACK dgerfsx / dporfsx).

  * exact_residual is the correctly rounded b - A (y + t) (checked against exact rational arithmetic);
  * the per-column state machine reaches every transition under scripted corrections: convergence, no progress after
    the switch to extra y, componentwise instability, and the early stop when componentwise accuracy is ignored;
  * on seeded Q1 diag(sigma) Q2 matrices with kappa from 1e2 to 1e17 (also row-, column- and solution-scaled): a trusted
    bound is never below the true normwise or componentwise error; for kappa M u <= 1e-2 every bound is trusted and the
    error is at most ERR_LBND; for kappa >= 100 / (M u) nothing is trusted and info = M + 1.  The true solution comes
    from double-double refinement with exact residuals;
  * the rank-by-rank double-double assembly equals the dense correctly rounded product within the Dot2 bound on LU
    and Cholesky grids, with NaN wherever the device must not read."""
import math
from fractions import Fraction

import numpy as np
import pytest
from scipy.linalg import cho_factor, lapack, lu_factor

from oracle import chol_ref, chol_solve_ref, layout
from oracle import refine_ref as rr
from oracle import refinex_ref as rx

U = 2.0 ** -53


def test_exact_residual_is_correctly_rounded():
    rng = np.random.default_rng(0)
    A = rng.standard_normal((7, 9)) * np.exp(rng.uniform(-20, 20, (7, 9)))
    y, t = rng.standard_normal(9), rng.standard_normal(9) * 1e-17
    b = A @ y
    r = rx.exact_residual(A, b, y, t)
    for i in range(7):
        exact = Fraction(b[i]) - sum(Fraction(A[i, k]) * (Fraction(y[k]) + Fraction(t[k])) for k in range(9))
        assert r[i] == float(exact)


def _script(seq):
    return lambda j, cnt: np.full(4, seq[min(cnt, len(seq)) - 1])


def test_state_machine_transitions():
    A, B, Y = np.eye(4), np.ones((4, 1)), np.ones((4, 1))
    one = lambda x: x
    # converge: the corrections shrink fast, x and z reach CONV in three rounds
    *_, cols = rx.rfsx(A, B, Y, one, one, 1.0, dys=_script([1e-3, 1e-9, 1e-17]))
    assert cols[0].x_state == rx.CONV and cols[0].z_state == rx.CONV and cols[0].y_prec == rx.EXTRA_RESIDUAL
    # no progress: corrections that stop shrinking switch y to extra precision, then x stops making progress
    *_, cols = rx.rfsx(A, B, Y, one, one, 1.0, dys=_script([1e-3, 1e-4, 1e-4, 1e-4]))
    assert cols[0].y_prec == rx.EXTRA_Y and cols[0].x_state == rx.NOPROG and cols[0].z_state == rx.NOPROG
    # a tiny component with rcond small asks for extra y from the first round
    Yz = np.array([[1.0], [1.0], [1.0], [1e-20]])
    *_, cols = rx.rfsx(A, B, Yz, one, one, 1e-3, dys=_script([1e-3, 1e-9, 1e-17]))
    assert cols[0].y_prec == rx.EXTRA_Y
    # componentwise unstable: a zero component with a non-zero correction (dz_z = inf); stops after the second round
    Y0 = np.array([[1.0], [1.0], [1.0], [0.0]])
    rounds = []
    *_, cols = rx.rfsx(A, B, Y0, one, one, 1.0, dys=lambda j, c: rounds.append(c) or np.full(4, 1e-17))
    assert cols[0].x_state == rx.CONV and cols[0].z_state == rx.UNSTABLE and rounds == [1, 2]
    # cwise ignored: stops as soon as x has converged
    rounds.clear()
    _, _, _, ec, _, cols = rx.rfsx(A, B, Y0, one, one, 1.0, cwise=False,
                                   dys=lambda j, c: rounds.append(c) or np.full(4, 1e-17))
    assert rounds == [1] and ec is None
    # the bounds: err = final / (1 - ratmax), capped at 1 and floored at ERR_LBND
    c = rx.Column()
    c.x_state, c.dx_x, c.dxratmax = rx.WORKING, 0.25, 0.5
    c.finish()
    assert c.err_norm == 0.5


def _matrix(n, kappa, kind, seed):
    rng = np.random.default_rng(seed)
    Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
    Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q1 * np.logspace(0, -math.log10(kappa), n)) @ Q2.T
    s = np.logspace(0, 8, n)
    rng.shuffle(s)
    if kind == "rows":
        A = A * s[:, None]
    elif kind == "cols":
        A = A * s[None, :]
    return A, s


def true_solution(Aop, B, solve):
    """double-double refinement with exact residuals: (head, tail) accurate to about u^2 kappa"""
    X = solve(B)
    T = np.zeros_like(X)
    for _ in range(6):
        for j in range(B.shape[1]):
            X[:, j], T[:, j] = rx.wwaddw(X[:, j], T[:, j], solve(rx.exact_residual(Aop, B[:, j], X[:, j], T[:, j])))
    return X, T


def errors(X, Xt, Tt, d=None):
    """the true normwise and componentwise relative errors per column of diag(d) X, from the double-double truth"""
    D = (X - Xt) - Tt
    nw = np.max(np.abs(D * d[:, None] if d is not None else D), 0) / np.max(np.abs(X * d[:, None] if d is not None else X), 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        cw = np.max(np.abs(D) / np.abs(X), 0)
    return nw, cw


def check_bounds(n, kappa, out, nw, cw, what):
    Y, berr, en, ec, info, _ = out
    lbnd = max(10.0, math.sqrt(n)) * U
    for j in range(len(nw)):
        if en[j, 0] == 1:
            assert nw[j] <= en[j, 1], (what, j, nw[j], en[j])
        if ec is not None and ec[j, 0] == 1:
            assert cw[j] <= ec[j, 1], (what, j, cw[j], ec[j])
    if kappa * n * U <= 1e-2:
        assert np.all(en[:, 0] == 1) and np.all(nw <= lbnd) and np.all(en[:, 1] == lbnd), (what, nw, en)
        assert info == 0 or ec[info - n - 1, 0] == 0, what     # only a componentwise bound may be untrusted
    if kappa >= 100 / (n * U):
        assert np.all(en[:, 0] == 0) and info == n + 1, (what, en, info)


KAPPAS = [1e2, 1e6, 1e10, 1e12, 1e15, 1e17]


@pytest.mark.parametrize("kappa", KAPPAS)
@pytest.mark.parametrize("kind", ["plain", "rows", "cols"])
@pytest.mark.parametrize("trans", [False, True])
def test_gerfsx_bounds(kappa, kind, trans):
    n = 48
    A, s = _matrix(n, kappa, kind, int(math.log10(kappa)) * 7 + len(kind))
    d = s if (kind, trans) in (("cols", False), ("rows", True)) else None     # op(A) column-scaled: its scales
    B = np.random.default_rng(3).standard_normal((n, 2))
    LU, piv = lu_factor(A)
    perm = np.arange(n)
    for i, p in enumerate(piv):
        perm[[i, p]] = perm[[p, i]]
    solve, solve_t = rr.lu_solvers(LU, perm, trans)
    Aop = A.T if trans else A
    norm = "1" if trans else "I"
    rcond = lapack.dgecon(LU, np.linalg.norm(A, 1 if trans else np.inf), norm=norm)[0]
    out = rx.gerfsx(A, B, solve(B), solve, solve_t, rcond, trans, d)
    Xt, Tt = true_solution(Aop, B, solve)
    nw, cw = errors(out[0], Xt, Tt, d)
    check_bounds(n, kappa, out, nw, cw, f"ge {kind} {kappa:g} trans={trans}")


@pytest.mark.parametrize("kappa", KAPPAS)
@pytest.mark.parametrize("scaled", [False, True])
def test_porfsx_bounds(kappa, scaled):
    n = 48
    rng = np.random.default_rng(int(math.log10(kappa)))
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q * np.logspace(0, -math.log10(kappa), n)) @ Q.T
    A = (A + A.T) / 2
    B = rng.standard_normal((n, 2))
    if scaled:                                          # a solution whose entries span many exponents
        B = A @ (rng.standard_normal((n, 2)) * np.logspace(0, 6, n)[:, None])
    try:
        c, _ = cho_factor(A, lower=True)
    except np.linalg.LinAlgError:
        pytest.skip("not numerically positive definite at this kappa")
    L = np.tril(c)
    solve = rr.chol_solver(L)
    rcond = lapack.dpocon(L, np.linalg.norm(A, 1), uplo="L")[0]
    out = rx.porfsx(A, B, solve(B), solve, rcond)
    Xt, Tt = true_solution(A, B, solve)
    nw, cw = errors(out[0], Xt, Tt)
    check_bounds(n, kappa, out, nw, cw, f"po {kappa:g} scaled={scaled}")


def test_gerfsx_beats_working_precision():
    n, kappa = 48, 1e12
    A, _ = _matrix(n, kappa, "plain", 5)
    B = np.random.default_rng(4).standard_normal((n, 2))
    LU, piv = lu_factor(A)
    perm = np.arange(n)
    for i, p in enumerate(piv):
        perm[[i, p]] = perm[[p, i]]
    solve, solve_t = rr.lu_solvers(LU, perm)
    rcond = lapack.dgecon(LU, np.linalg.norm(A, np.inf), norm="I")[0]
    Y = rx.gerfsx(A, B, solve(B), solve, solve_t, rcond)[0]
    Xw = rr.gerfs(A, B, solve(B), solve, solve_t)[0]
    Xt, Tt = true_solution(A, B, solve)
    assert np.all(errors(Y, Xt, Tt)[0] * 100 <= errors(Xw, Xt, Tt)[0])


def _dot2_ok(H, L, exact, absum, K):
    err = np.abs((H + L) - exact)
    assert np.all(err <= 2 * U * np.abs(exact) + (K * U) ** 2 * absum)


@pytest.mark.parametrize("N,v,Px,Py,Pz", [(64, 8, 1, 1, 1), (64, 8, 2, 2, 1), (96, 8, 3, 3, 1), (100, 8, 2, 2, 2)])
@pytest.mark.parametrize("trans", [False, True])
def test_grid_partials_x_lu(N, v, Px, Py, Pz, trans):
    rng = np.random.default_rng(N + Px)
    d = layout.dims(N, v, Px, Py, Pz)
    M = d["M"]
    A = rng.standard_normal((M, M))
    locs = layout.scatter(A, v, Px, Py, Pz)
    y, t = rng.standard_normal(M), rng.standard_normal(M) * 1e-17
    H, L = rx.partials_x_lu(locs, y, t, N, v, Px, Py, Pz, trans)
    Aop = A.T if trans else A
    exact = -rx.exact_residual(Aop, np.zeros(M), y, t)
    _dot2_ok(H, L, exact, np.abs(Aop) @ (np.abs(y) + np.abs(t)), M)


@pytest.mark.parametrize("N,v,grid", [(64, 8, (1, 1, 1)), (64, 8, (2, 1, 1)), (96, 8, (2, 2, 1)), (96, 8, (3, 2, 1)),
                                      (96, 8, (1, 3, 2))])
def test_grid_partials_x_chol(N, v, grid):
    rng = np.random.default_rng(N + grid[0] * 10 + grid[1])
    n = chol_ref.dims(N, v, *grid)["N"]
    A = rng.standard_normal((N, N))
    A = A + A.T
    locs = chol_solve_ref.scatter(A, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)
    y, t = rng.standard_normal(n), rng.standard_normal(n) * 1e-17
    H, L = rx.partials_x_chol(locs, y, t, N, v, *grid)
    Af = chol_ref.lower_sym(chol_ref.assemble([np.nan_to_num(l, nan=0.0) for l in locs], N, v, *grid))
    exact = -rx.exact_residual(Af, np.zeros(n), y, t)
    _dot2_ok(H, L, exact, np.abs(Af) @ (np.abs(y) + np.abs(t)), n)
