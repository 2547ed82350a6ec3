"""CPU: oracle/svxx_ref.py (the restatement of cflx_*_equilibrate_b / cflx_*_svxx) against LAPACK.

  * geequb equals scipy's dgeequb bit for bit on random, graded (2^+-300), exact-power-of-two and near-2^+-1022 inputs and
    on both info paths; poequb equals dpoequb of scipy's bundled OpenBLAS (through ctypes: scipy has no wrapper);
  * gerpvgrw / porpvgrw equal a plain double loop over scipy's LU and Cholesky factors, with ncols < M and columns whose
    umax is 0;
  * the per-share growth vectors combined over the grids of the GPU tests equal the dense ones, with NaN in every entry
    the device must not read;
  * gesvxx on power-of-two scaling returns diag(c) times refinex_ref's solution of the scaled system, exactly."""
import ctypes
import glob
import os

import numpy as np
import pytest
import scipy
from scipy.linalg import lapack

from oracle import chol_ref, chol_solve_ref, layout
from oracle import refine_ref as rr
from oracle import refinex_ref as rx
from oracle import svx_ref as sr
from oracle import svxx_ref as xr


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b))


def general(n, kind, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    s = np.exp2(rng.uniform(-300, 300, n))
    t = np.exp2(rng.uniform(-300, 300, n))
    if kind == "rows":
        return A * s[:, None]
    if kind == "cols":
        return A * t[None, :]
    if kind == "both":
        return A * s[:, None] * t[None, :]
    if kind == "pow2":                                                 # every row and column maximum a power of two
        A = np.exp2(rng.integers(-40, 40, (n, n)).astype(float)) * rng.choice([-1.0, 1.0], (n, n))
        return A
    if kind == "tiny":
        return A * 2.0 ** -1020
    if kind == "huge":
        return A * 2.0 ** 1020
    return A


KINDS = ["plain", "rows", "cols", "both", "pow2", "tiny", "huge"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_geequb_bit_identical_to_lapack(kind, seed):
    A = general(64, kind, seed)
    g = xr.geequb(A)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequb(A)
    assert info == g["info"] == 0
    assert _same(r, g["r"]) and _same(c, g["c"])
    assert (rowcnd, colcnd, amax) == (g["rowcnd"], g["colcnd"], g["amax"])
    assert np.all(np.frexp(g["r"])[0] == 0.5) and np.all(np.frexp(g["c"])[0] == 0.5)
    As, equed = sr.laqge(A, g["r"], g["c"], g["rowcnd"], g["colcnd"], g["amax"])
    if equed != "N":                                                  # power-of-two scaling is exact
        Ar = A * (g["r"][:, None] if equed in "RB" else 1.0) * (g["c"][None, :] if equed in "CB" else 1.0)
        assert _same(As, Ar)


def test_geequb_near_the_exponent_range():
    rng = np.random.default_rng(3)
    A = rng.uniform(1.0, 2.0, (16, 16)) * rng.choice([-1.0, 1.0], (16, 16))
    A[0] *= 2.0 ** -1021
    A[1] *= 2.0 ** 1022
    A[:, 2] *= 2.0 ** -1000
    A[3, :] = 2.0 ** -1022                                            # maxima exactly 2^-1022 and 2^1023
    A[4, 5] = 2.0 ** 1023
    g = xr.geequb(A)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequb(A)
    assert info == g["info"] and _same(r, g["r"]) and (rowcnd, amax) == (g["rowcnd"], g["amax"])
    if info == 0:
        assert _same(c, g["c"]) and colcnd == g["colcnd"]


def test_geequb_zero_row_and_column():
    A = general(32, "both", 4)
    A[5] = 0.0
    g = xr.geequb(A)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequb(A)
    assert g["info"] == info == 6 and _same(g["r"], r) and g["amax"] == amax
    A = general(32, "both", 5)
    A[:, 9] = 0.0
    g = xr.geequb(A)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequb(A)
    assert g["info"] == info == 32 + 10 and _same(g["r"], r) and g["rowcnd"] == rowcnd and _same(g["c"], c)


def _openblas_dpoequb():
    """scipy's bundled OpenBLAS's dpoequb (exported with the scipy_ prefix), or None"""
    d = os.path.dirname(scipy.__file__)
    for lib in sorted(glob.glob(os.path.join(os.path.dirname(d), "scipy.libs", "*openblas*")) +
                      glob.glob(os.path.join(d, ".libs", "*openblas*"))):
        L = ctypes.CDLL(lib)
        for name in ("scipy_dpoequb_", "dpoequb_"):
            if hasattr(L, name):
                return getattr(L, name)
    return None


def lapack_dpoequb(A):
    fn = _openblas_dpoequb()
    if fn is None:
        pytest.skip("scipy's OpenBLAS exports no dpoequb symbol: nothing to compare poequb with")
    n = A.shape[0]
    Af = np.asfortranarray(A, dtype=np.float64)
    s = np.zeros(n)
    N, lda, info = ctypes.c_int(n), ctypes.c_int(n), ctypes.c_int()
    scond, amax = ctypes.c_double(), ctypes.c_double()
    fn(ctypes.byref(N), Af.ctypes.data_as(ctypes.c_void_p), ctypes.byref(lda), s.ctypes.data_as(ctypes.c_void_p),
       ctypes.byref(scond), ctypes.byref(amax), ctypes.byref(info))
    return s, scond.value, amax.value, info.value


def spd(n, kind, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    A = G @ G.T / n + np.eye(n)
    if kind == "graded":
        s = np.exp2(rng.uniform(-300, 300, n))
        A = A * s[:, None] * s[None, :]
    if kind == "pow2":
        A = np.diag(np.exp2(rng.integers(-60, 60, n).astype(float)))
    return A


@pytest.mark.parametrize("kind", ["plain", "graded", "pow2"])
@pytest.mark.parametrize("seed", [0, 1])
def test_poequb_bit_identical_to_lapack(kind, seed):
    A = spd(48, kind, seed)
    p = xr.poequb(A)
    s, scond, amax, info = lapack_dpoequb(A)
    assert info == p["info"] == 0
    assert _same(s, p["s"]) and (scond, amax) == (p["scond"], p["amax"])
    assert np.all(np.frexp(p["s"])[0] == 0.5)


def test_poequb_non_positive_diagonal():
    A = spd(16, "plain", 6)
    A[4, 4] = 0.0
    A[7, 7] = -1.0
    p = xr.poequb(A)
    s, scond, amax, info = lapack_dpoequb(A)
    assert p["info"] == info == 5 and _same(p["s"], s) and p["amax"] == amax


# ----------------------------------------------------------------------------------------------- pivot growth
def _loop_gerpvgrw(A, U, ncols):
    n = A.shape[0]
    rpvgrw = 1.0
    for j in range(ncols):
        amax = umax = 0.0
        for i in range(n):
            amax = max(abs(A[i, j]), amax)
        for i in range(j + 1):
            umax = max(abs(U[i, j]), umax)
        if umax != 0.0:
            rpvgrw = min(amax / umax, rpvgrw)
    return rpvgrw


def _loop_porpvgrw(A, L, ncols):
    rpvgrw = 1.0
    for j in range(ncols):
        amax = umax = 0.0
        for i in range(j, ncols):
            amax = max(abs(A[i, j]), amax)
            umax = max(abs(L[i, j]), umax)
        if umax != 0.0:
            rpvgrw = min(amax / umax, rpvgrw)
    return rpvgrw


@pytest.mark.parametrize("kind", ["plain", "both", "pow2"])
def test_gerpvgrw_equals_a_plain_loop(kind):
    from scipy.linalg import lu_factor
    A = general(40, kind, 7)
    LU, _ = lu_factor(A)
    for ncols in (40, 17, 1):
        assert xr.gerpvgrw(A, LU, ncols) == _loop_gerpvgrw(A, LU, ncols)
    Z = np.triu(np.abs(general(12, "plain", 8)) + 1.0)
    Z[:, 4] = 0.0                                                     # a column with umax = 0 is skipped
    assert xr.gerpvgrw(Z, Z) == _loop_gerpvgrw(Z, Z, 12)
    # a growth below 1 is found in the column where it happens
    Z2 = Z.copy()
    Z2[:, 6] *= 1e-3
    assert xr.gerpvgrw(Z2, Z) == _loop_gerpvgrw(Z2, Z, 12) < 1e-2


@pytest.mark.parametrize("kind", ["plain", "graded"])
def test_porpvgrw_equals_a_plain_loop(kind):
    A = spd(40, kind, 9)
    L = np.linalg.cholesky(A)
    Al = np.tril(A) + np.triu(np.full(A.shape, np.nan), 1)            # only the lower triangles are read
    Ll = L + np.triu(np.full(A.shape, np.nan), 1)
    for ncols in (40, 23, 1):
        assert xr.porpvgrw(Al, Ll, ncols) == _loop_porpvgrw(A, L, ncols)
    L0 = L.copy()
    L0[:, 3] = 0.0
    assert xr.porpvgrw(A, L0) == _loop_porpvgrw(A, L0, 40)


# ----------------------------------------------------------------------------------------------- the grid pass
LU_GRIDS = [(64, 8, 1, 1, 1), (128, 16, 1, 1, 2), (64, 8, 2, 2, 1), (128, 8, 2, 2, 2), (96, 16, 3, 3, 1),
            (100, 16, 1, 1, 1)]
CHOL_GRIDS = [(256, 32, (2, 2, 1)), (256, 32, (1, 1, 2)), (384, 32, (3, 2, 1)), (384, 32, (1, 3, 2)), (100, 16, (1, 1, 1))]


@pytest.mark.parametrize("N,v,Px,Py,Pz", LU_GRIDS)
def test_growth_cols_grid_lu(N, v, Px, Py, Pz):
    d = layout.dims(N, v, Px, Py, Pz)
    M = d["M"]
    rng = np.random.default_rng(N + Px)
    A = general(M, "both", N)
    F = rng.standard_normal((M, M)) * np.exp2(rng.uniform(-50, 50, (M, M)))
    for ncols in (M, M // 2 + 3):
        An = np.where(np.arange(M)[None, :] < ncols, A, np.nan)       # columns >= ncols: never read
        Fn = np.where((np.arange(M)[:, None] <= np.arange(M)[None, :]) & (np.arange(M)[None, :] < ncols), F, np.nan)
        A_locs, F_locs = layout.scatter(An, v, Px, Py, Pz), layout.scatter(Fn, v, Px, Py, Pz)
        for r in range(d["P"]):
            if r % Pz:
                A_locs[r][...] = np.nan
                F_locs[r][...] = np.nan
        amax, fmax = xr.growth_cols_grid(F_locs, A_locs, N, v, Px, Py, Pz, ncols)
        ref_a = np.array([np.abs(A[:, j]).max() if j < ncols else 0.0 for j in range(M)])
        ref_f = np.array([np.abs(F[:j + 1, j]).max() if j < ncols else 0.0 for j in range(M)])
        assert _same(amax, ref_a) and _same(fmax, ref_f)
        assert xr.rpvgrw_cols(amax, fmax, ncols) == _loop_gerpvgrw(A, F, ncols)


def _chol_locals(A, N, v, grid):
    """the layer-0 shares with NaN in every entry the pass must not read: above the diagonal (whole tiles and inside
    the diagonal tiles), the padding tiles and the other layers"""
    d = chol_ref.dims(N, v, *grid)
    Px, Py, Pz = grid
    locs = chol_solve_ref.scatter(A, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)
    for r, loc in enumerate(locs):
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        if r % Pz == 0:
            for t in range(d["Kappa"]):
                if t % Px == pi and t % Py == pj:
                    blk = loc[(t // Px) * v:(t // Px + 1) * v, (t // Py) * v:(t // Py + 1) * v]
                    blk[np.triu_indices(v, 1)] = np.nan
    return locs


@pytest.mark.parametrize("N,v,grid", CHOL_GRIDS)
def test_growth_cols_grid_chol(N, v, grid):
    n = chol_ref.dims(N, v, *grid)["N"]
    A = spd(n, "graded", N)
    L = np.linalg.cholesky(A)
    amax, fmax = xr.growth_cols_grid(_chol_locals(L, N, v, grid), _chol_locals(A, N, v, grid), N, v, *grid, sym=True)
    assert _same(amax, [np.abs(A[j:, j]).max() for j in range(n)])
    assert _same(fmax, [np.abs(L[j:, j]).max() for j in range(n)])
    assert xr.rpvgrw_cols(amax, fmax, n) == _loop_porpvgrw(A, L, n) == xr.porpvgrw(A, L)


# ----------------------------------------------------------------------------------------------- the drivers
@pytest.mark.parametrize("trans", [False, True])
def test_gesvxx_unscales_the_scaled_solution_exactly(trans):
    from scipy.linalg import lu_factor
    n = 80
    rng = np.random.default_rng(11)                                   # graded by 2^+-20: kappa(A) stays below 1 / (n u)
    A = rng.standard_normal((n, n)) * np.exp2(rng.uniform(-20, 20, n))[:, None] * np.exp2(rng.uniform(-20, 20, n))
    B = np.random.default_rng(12).standard_normal((n, 2))
    g = xr.geequb(A)
    As, equed = sr.laqge(A, g["r"], g["c"], g["rowcnd"], g["colcnd"], g["amax"])
    assert equed == "B" and _same(As, (g["r"][:, None] * A) * g["c"][None, :])
    LU, piv = lu_factor(As)
    perm = np.arange(n)
    for i, p in enumerate(piv):
        perm[i], perm[p] = perm[p], perm[i]
    got = xr.gesvxx(As, LU, perm, B, trans, g["r"], g["c"], equed)
    assert got["info"] == 0
    pre, post = (g["c"], g["r"]) if trans else (g["r"], g["c"])
    solve, solve_t = rr.lu_solvers(LU, perm, trans)
    Bs = pre[:, None] * B
    Y, berr, en, ec, info, _ = rx.gerfsx(As, Bs, solve(Bs), solve, solve_t, got["rcond"], trans, post)
    assert _same(got["X"], post[:, None] * Y) and _same(got["berr"], berr) and _same(got["err_norm"], en)
    assert _same(got["X"] / post[:, None], Y)                         # the unscaling is exact: it divides back
    # the trusted normwise bound holds for the unscaled solution of A x = b
    Ao = A.T if trans else A
    Xt = np.linalg.solve(Ao, B)
    for _ in range(3):
        Xt = Xt + np.linalg.solve(Ao, np.asarray(B - Ao.astype(np.longdouble) @ Xt.astype(np.longdouble), dtype=float))
    err = np.max(np.abs(got["X"] - Xt), 0) / np.max(np.abs(Xt), 0)
    assert np.all(en[:, 0] == 1.0) and np.all(err <= en[:, 1])


def test_posvxx_and_zero_pivot():
    n = 48
    s = np.exp2(np.random.default_rng(13).uniform(-10, 10, n))       # kappa(A) stays below 1 / (n u)
    A = spd(n, "plain", 13) * s[:, None] * s[None, :]
    B = np.random.default_rng(14).standard_normal((n, 2))
    p = xr.poequb(A)
    As, equed = sr.laqsy(A, p["s"], p["scond"], p["amax"])
    assert equed == "Y"
    L = np.linalg.cholesky(chol_ref.lower_sym(As))
    got = xr.posvxx(chol_ref.lower_sym(As), L, B, p["s"], equed)
    assert got["info"] == 0 and _same(got["X"], p["s"][:, None] * got["Y"])
    assert got["rpvgrw"] == _loop_porpvgrw(chol_ref.lower_sym(As), L, n)
    # LU: an exactly zero U(k,k) gives info = k, rcond 0 and the leading-k growth
    Z = np.triu(np.random.default_rng(15).integers(1, 9, (12, 12)).astype(float))
    Z[4, 4] = 0.0
    got = xr.gesvxx(Z, Z.copy(), np.arange(12), np.ones((12, 1)))
    assert got["info"] == 5 and got["rcond"] == 0.0 and got["X"] is None
    assert got["rpvgrw"] == _loop_gerpvgrw(Z, Z, 5)
