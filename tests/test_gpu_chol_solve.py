"""GPU: cflx_chol_solve (A X = B with the Cholesky factor left on the device) and its transposed narrow GEMM, against numpy,
scipy's cho_solve on the device's own factor and the schedule restatement (oracle/chol_solve_ref.py); graded and
ill-conditioned matrices; its state rules; and that it leaves the factorisation untouched.

Tolerances: the backward error ||B - A X||_F / (||A||_F ||X||_F + ||B||_F) <= 1e-13, and X within 1e-10 max|X| of the
host solve and of the restatement on the same factor (the same operations, in other summation orders).  X of integer
right-hand sides is bit for bit the one pinned in tests/golden/solve_bits.json."""
import json
import os

import numpy as np
import pytest
import scipy.linalg

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, hp_ref as hp
from tests._harness import n_gpus, run_ranks
from tests.golden import make_solve_golden

pytestmark = pytest.mark.gpu
ETA_TOL = 1e-13
X_TOL = 1e-10


# ----------------------------------------------------------------------------------------------- gemm_narrow_tn_kernel
@pytest.mark.parametrize("M,N,K", [(1, 1, 4), (37, 3, 8), (1000, 1, 256), (4097, 64, 256), (513, 65, 128),
                                   (16128, 200, 512), (63, 9, 7), (97, 17, 130), (2, 33, 1)])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-1.0, 1.0)])
def test_gemm_narrow_tn_matches_numpy(M, N, K, alpha, beta):
    """odd M, M not a multiple of 32, K not a multiple of 4 or 8, N across the 8 / 16 / 32 / 64-column variants"""
    rng = np.random.default_rng(M + N + K)
    AT = rng.standard_normal((K, M))
    B = rng.standard_normal((K, N))
    C = rng.standard_normal((M, N))
    want = beta * C + alpha * (AT.T @ B)
    tol = 1e-13 * max(K, 1) * np.abs(AT).max() * np.abs(B).max()
    D, ms = cb.dbg.gemm_narrow_tn(AT, B, C, alpha, beta)
    assert ms > 0 and np.abs(D - want).max() <= tol
    Ca = C.copy()
    D2, _ = cb.dbg.gemm_narrow_tn(AT, B, Ca, alpha, beta, out=Ca)       # D aliasing C on the device
    assert D2 is Ca and np.abs(Ca - want).max() <= tol


def test_gemm_narrow_tn_exact_products_and_empty_k():
    """exact integer products come back exactly, and K = 0 gives beta C"""
    rng = np.random.default_rng(3)
    AT = rng.integers(-4, 5, (13, 45)).astype(np.float64)
    B = rng.integers(-4, 5, (13, 11)).astype(np.float64)
    D, _ = cb.dbg.gemm_narrow_tn(AT, B)
    assert np.array_equal(D, AT.T @ B)
    C = rng.standard_normal((45, 11))
    D0, _ = cb.dbg.gemm_narrow_tn(np.zeros((0, 45)), np.zeros((0, 11)), C, 1.0, 2.0)
    assert np.array_equal(D0, 2.0 * C)


def test_gemm_narrow_tn_refuses_bad_shapes():
    with pytest.raises(cb.ConfluxError, match="status -1"):
        cb.dbg.gemm_narrow_tn(np.ones((8, 0)), np.ones((8, 4)))       # M = 0
    with pytest.raises(cb.ConfluxError, match="status -1"):
        cb.dbg.gemm_narrow_tn(np.ones((8, 4)), np.ones((8, 0)))       # N = 0
    with pytest.raises(ValueError):
        cb.dbg.gemm_narrow_tn(np.ones((8, 4)), np.ones((6, 4)))       # K mismatch
    a, b, d = np.ones(64), np.ones(64), np.zeros(64)
    rc = cb.lib().cflx_dbg_gemm_narrow_tn(8, 8, -8, a.ctypes.data, b.ctypes.data, None, 1.0, 0.0, d.ctypes.data, 1, None)
    assert rc == -1                                                   # K < 0


# ----------------------------------------------------------------------------------------------- solves
def _solve_on_grid(N, v, grid, Bs, A=None):
    """Factor once on the grid (A: the global matrix, or None for the library's generator), then solve every B."""
    P = grid[0] * grid[1] * grid[2]
    locs = chol_solve_ref.scatter(A, N, v, *grid) if A is not None else None

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        if locs is not None:
            ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        Xs = [ch.solve(B) for B in Bs]
        res = dict(A=ch.data.copy(), L=ch.local_factor(), X=Xs)
        ch.finalize()
        return res

    rs = run_ranks(P, body)
    return dict(A=[r["A"] for r in rs], L=[r["L"] for r in rs], X=[r["X"] for r in rs])


def _check(g, N, v, grid, Bs):
    S = chol_ref.lower_sym(chol_ref.assemble(g["A"], N, v, *grid))
    L = np.tril(chol_ref.assemble(g["L"], N, v, *grid))
    for i, B in enumerate(Bs):
        X = g["X"][0][i]
        for Xr in g["X"]:
            assert np.array_equal(Xr[i], X)                              # bit-identical on every rank
        assert X.shape == B.shape and np.all(np.isfinite(X))
        assert chol_solve_ref.backward_error(S, X, B) <= ETA_TOL
        scale = np.abs(X).max()
        assert np.abs(X - scipy.linalg.cho_solve((L, True), B)).max() <= X_TOL * scale
        Xo = chol_solve_ref.solve(g["L"], B, N, v, *grid)
        assert np.abs(X - Xo).max() <= X_TOL * scale


SINGLE = [(16, 4), (96, 16), (100, 16), (512, 64), (1024, 128), (1152, 384), (2048, 256), (2048, 512), (4096, 512)]


@pytest.mark.parametrize("kind", ["gen", "int"])
@pytest.mark.parametrize("N,v", SINGLE)
def test_single_gpu_solve(N, v, kind):
    Np = chol_ref.dims(N, v, 1, 1, 1)["N"]
    rng = np.random.default_rng(N + v)
    Bs = [rng.standard_normal((Np, nrhs)) for nrhs in (1, 3, 64, 130)] + [rng.standard_normal(Np)]
    A = chol_ref.bits_case_input(kind, Np)
    g = _solve_on_grid(N, v, (1, 1, 1), Bs, A)
    _check(g, N, v, (1, 1, 1), Bs)


@pytest.mark.parametrize("N,v", [(1024, 128), (1152, 384)])
def test_graded_matrix_bit_for_bit(N, v):
    """A = D S D with D = diag(2^-10 .. 2^10): the solution of A x = D b is D^-1 times that of S y = b.  Scaling by powers
    of two commutes with every rounding (the factor is D L(S) bit for bit, every inverse block and every product of the
    sweeps is scaled by powers of two only), so the two solves must agree bit for bit."""
    rng = np.random.default_rng(N + 3 * v)
    d = 2.0 ** np.round(np.linspace(-10, 10, N))
    S = hp.random_spd(N, 1e2, rng)
    A = d[:, None] * S * d[None, :]
    b = rng.standard_normal((N, 5))
    xa = _solve_on_grid(N, v, (1, 1, 1), [d[:, None] * b], A)["X"][0][0]
    xs = _solve_on_grid(N, v, (1, 1, 1), [b], S)["X"][0][0]
    assert np.array_equal(xa, xs / d[:, None])


def test_ill_conditioned_forward_error():
    """kappa_2(A) = 1e8.  The computed x^ solves (A + dA) x^ = b with ||dA||_F <= gamma_{3n+1} (1 + 4 kappa_max)
    || |L^| |L^T| ||_F: one gamma_{n+1} for the factorisation and one gamma_n for each triangular sweep (Higham Thm 10.4),
    each widened by (1 + 4 kappa_max) for the explicitly inverted nb x nb diagonal blocks, kappa_max their largest
    condition number (the factor of 2 on the first-order 2 kappa_max is a chosen margin, as in oracle/hp_ref.py).  So
        ||x^ - x||_2 / ||x||_2 <= kappa_2(A) eps / (1 - kappa_2(A) eps),   eps = that bound / ||A||_2.
    x is the float64 cho_solve answer refined twice with residuals computed exactly (hp_ref.matmul)."""
    N, v = 1024, 128
    rng = np.random.default_rng(108)
    A = hp.random_spd(N, 1e8, rng)
    b = rng.standard_normal((N, 2))
    g = _solve_on_grid(N, v, (1, 1, 1), [b], A)
    xh = g["X"][0][0]
    Lh = np.tril(g["L"][0])
    x = scipy.linalg.cho_solve((Lh, True), b)
    for _ in range(2):
        r = (b.astype(hp.LD) - hp.matmul(A, x)).astype(np.float64)
        x = x + scipy.linalg.cho_solve((Lh, True), r)
    kmax = hp.diag_block_kappa(Lh, 128)
    ev = np.linalg.eigvalsh(A)
    kappa = ev[-1] / ev[0]
    eps = hp.gamma(3 * N + 1) * (1.0 + 4.0 * kmax) * np.linalg.norm(np.abs(Lh) @ np.abs(Lh).T) / ev[-1]
    assert kappa * eps < 0.5
    assert np.linalg.norm(xh - x) / np.linalg.norm(x) <= kappa * eps / (1.0 - kappa * eps)
    assert chol_solve_ref.backward_error(A, xh, b) <= ETA_TOL


def _not_pd(N, rng):
    A = hp.random_spd(N, 1e2, rng)
    A[N // 2, N // 2] = -1.0
    return A


def test_state_rules():
    N, v = 256, 32
    rng = np.random.default_rng(1)
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    B = rng.standard_normal((ch.N, 2))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.solve(B)                                                     # no factorisation yet
    ch.parallelCholesky()
    S = chol_ref.lower_sym(ch.data)
    X = ch.solve(B)
    assert chol_solve_ref.backward_error(S, X, B) <= ETA_TOL
    with pytest.raises(cb.ConfluxError, match="status -1"):
        ch.solve(np.zeros((ch.N, 0)))                                   # nrhs < 1
    with pytest.raises(ValueError):
        ch.solve(np.zeros((ch.N + 1, 2)))
    b2 = rng.standard_normal(ch.N)
    x2 = ch.solve(b2)                                                   # a second B after the same factorisation
    assert chol_solve_ref.backward_error(S, x2, b2) <= ETA_TOL
    a = np.ascontiguousarray(ch.data)
    cb.check(cb.lib().cflx_chol_set_local(ch._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.solve(B)                                                     # new input, not factored yet
    ch.data = _not_pd(N, rng)
    with pytest.raises(cb.ConfluxError, match="positive definite"):
        ch.parallelCholesky()
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.solve(B)                                                     # the factorisation failed
    A2 = hp.random_spd(N, 1e3, rng)
    ch.data = A2.copy()
    ch.parallelCholesky()                                               # a good one after the failed one, another matrix
    X3 = ch.solve(B)
    assert chol_solve_ref.backward_error(A2, X3, B) <= ETA_TOL          # the cache follows the new matrix
    assert not np.allclose(X3, X)
    ch.finalize()
    comm.close()


def _launches(ch):
    """kernels counted since the last call (and reset)"""
    import ctypes
    n = ctypes.c_int64()
    cb.check(cb.lib().cflx_chol_launch_count(ch._h, ctypes.byref(n), 1), "launch_count")
    return n.value


def test_no_side_effects_on_factor_and_validation():
    N, v = 1024, 128

    def run(solve):
        comm = cb.Comm(1, 0, None, 0)
        ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
        ch.parallelCholesky()
        n1 = _launches(ch)
        if solve:
            ch.solve(np.random.default_rng(0).standard_normal((ch.N, 7)))
        n_solve = _launches(ch)
        L, resid = ch.local_factor(), ch.validate()
        _launches(ch)
        ch.parallelCholesky()                                           # a second factorisation after the solve
        L2, n2 = ch.local_factor(), _launches(ch)
        data = ch.data.copy()
        ch.finalize()
        comm.close()
        return L, resid, L2, n1, n_solve, n2, data

    L0, r0, _, n10, _, _, d0 = run(False)
    L1, r1, L2, n11, ns, n2, d1 = run(True)
    assert np.array_equal(L0, L1) and r0 == r1
    assert np.array_equal(L2, L1) and n2 == n11 == n10
    assert ns == 0                                                      # the solve adds nothing to the launch count
    assert np.array_equal(d0, d1)


def test_solve_is_deterministic():
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(2048, 256, (1, 1, 1), comm)
    ch.parallelCholesky()
    B = np.random.default_rng(8).standard_normal((ch.N, 9))
    assert np.array_equal(ch.solve(B), ch.solve(B))
    ch.finalize()
    comm.close()


def test_solve_bits_are_pinned(golden_dir):
    """X of integer right-hand sides is the one recorded by tests/golden/make_solve_golden.py"""
    with open(os.path.join(golden_dir, "solve_bits.json")) as f:
        want = json.load(f)
    for kind, N, v in make_solve_golden.CHOL_CASES:
        assert make_solve_golden.chol_solve_bits(kind, N, v) == want[f"chol_{kind}_{N}_{v}"], (kind, N, v)


@pytest.mark.parametrize("v", [128, 512])
def test_ozaki_update_factor_solves(v, monkeypatch):
    N = 4 * v
    monkeypatch.setenv("CFLX_GEMM", "ozaki")                             # read when the object is created
    rng = np.random.default_rng(v)
    Bs = [rng.standard_normal((N, 3)), rng.standard_normal(N)]
    g = _solve_on_grid(N, v, (1, 1, 1), Bs)
    _check(g, N, v, (1, 1, 1), Bs)


GRIDS = [(2, 1, 1), (1, 2, 1), (2, 2, 1), (4, 2, 1), (2, 2, 2)]


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "%dx%dx%d" % g)
@pytest.mark.parametrize("N,v", [(1000, 48), (1024, 128)])   # Kappa = 21 (odd) and 8
def test_multi_gpu_solve(grid, N, v):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    Np = chol_ref.dims(N, v, *grid)["N"]
    rng = np.random.default_rng(N + P)
    Bs = [rng.standard_normal((Np, 3)), rng.standard_normal((Np, 70)), rng.standard_normal(Np)]
    g = _solve_on_grid(N, v, grid, Bs)
    _check(g, N, v, grid, Bs)
    g2 = _solve_on_grid(N, v, grid, Bs[:1])
    assert np.array_equal(g2["X"][0][0], g["X"][0][0])
