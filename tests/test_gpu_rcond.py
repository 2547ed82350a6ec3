"""GPU: cflx_lu_rcond / cflx_chol_rcond (LAPACK dgecon / dpocon on the grid).

  * anorm is the 1-norm of the assembled input (the padded LU matrix, the symmetric completion of the Cholesky input's
    lower triangle) to 1e-15 relative.  The reference column sums run in long double: numpy's float64 sum down a
    row-major column is a sequential one, in error by up to n u, and the device's sums are compensated;
  * rcond equals scipy's dgecon / dpocon on the device's own factors with the same anorm, to n u kappa_1(A) relative
    (u = 2^-53; a bound on the forward error of the solves that feed the estimator);
  * rcond >= (1 - 1e-10) / (||A||_1 ||A^-1||_1): the estimate of ||A^-1||_1 never exceeds it;
  * an exactly singular U gives rcond 0 with success, a failed Cholesky and the state rules give CFLX_ERR_STATE;
  * the factors, permutation, residual, launch count and a later solve are unchanged, and rcond is the same on every rank.
The largest observed |rcond - LAPACK| / (LAPACK n u kappa_1) is printed with -s."""
import numpy as np
import pytest
from scipy.linalg import lapack

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, layout
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
LU_GRIDS = [(64, 8, 2, 2, 1), (128, 16, 1, 1, 2), (128, 8, 2, 2, 2), (512, 64, 2, 2, 2)]
CHOL_GRIDS = [(256, 32, (2, 2, 1)), (256, 32, (1, 1, 2)), (384, 32, (3, 2, 1)), (512, 64, (2, 2, 2))]


def _kappa_matrix(n, kappa, seed):
    rng = np.random.default_rng(seed)
    Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
    Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
    return (Q1 * np.logspace(0, -np.log10(kappa), n)) @ Q2.T


def _norm1(A):
    return float(np.abs(A).astype(np.longdouble).sum(0).max())


def _check_rcond(A, rcond, anorm, want, what):
    n = A.shape[0]
    assert abs(anorm - _norm1(A)) <= 1e-15 * anorm, what
    ainv1 = np.abs(np.linalg.inv(A)).sum(0).max()
    kappa = anorm * ainv1
    margin = abs(rcond - want) / (want * n * U * kappa)
    print(f"rcond {what}: n={n} kappa_1={kappa:.2e} rcond={rcond:.6e} lapack={want:.6e} margin={margin:.2e}")
    assert margin <= 1.0, what
    assert rcond >= (1 - 1e-10) / kappa, what


# ----------------------------------------------------------------------------------------------- LU
def _lu_on_grid(N, v, Px, Py, Pz, A_locals=None, extra=None):
    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        if A_locals is not None:
            gv.data[...] = np.asarray(A_locals[gv.rank]).reshape(gv.Ml, gv.Nl)
        C = np.zeros((gv.Ml, gv.Nl))
        perm = np.zeros(gv.M, dtype=np.int32)
        cb.LU_rep(gv, C, perm)
        r = cb.lu_rcond(gv)
        out = dict(A=gv.data.copy(), C=C, perm=perm, r=r, r2=cb.lu_rcond(gv))
        if extra:
            out.update(extra(gv))
        gv.free_comms()
        return out

    return run_ranks(Px * Py * Pz, body)


def _check_lu(rs, N, v, Px, Py, Pz, what):
    A = layout.assemble([r["A"] for r in rs], N, v, Px, Py, Pz)
    LU = layout.assemble([r["C"] for r in rs], N, v, Px, Py, Pz)
    rcond, anorm = rs[0]["r"]
    for r in rs:
        assert r["r"] == (rcond, anorm) and r["r2"] == (rcond, anorm)  # every rank, every call: the same bits
    want, info = lapack.dgecon(LU, anorm, norm="1")
    assert info == 0
    _check_rcond(A, rcond, anorm, want, what)


@pytest.mark.parametrize("N,v", [(16, 4), (96, 16), (512, 64), (1024, 128), (100, 16)])
def test_lu_rcond_generator(N, v):
    _check_lu(_lu_on_grid(N, v, 1, 1, 1), N, v, 1, 1, 1, f"lu gen {N}/{v}")


@pytest.mark.parametrize("N,v", [(256, 32), (1024, 128)])
def test_lu_rcond_standard_normal(N, v):
    A = np.random.default_rng(N).standard_normal((N, N))
    _check_lu(_lu_on_grid(N, v, 1, 1, 1, [A]), N, v, 1, 1, 1, f"lu normal {N}")


def test_lu_rcond_ill_conditioned():
    N, v = 512, 64
    A = _kappa_matrix(N, 1e8, 7)
    _check_lu(_lu_on_grid(N, v, 1, 1, 1, [A]), N, v, 1, 1, 1, "lu kappa 1e8")


def test_lu_rcond_singular_is_zero():
    N, v = 256, 32
    A = np.random.default_rng(2).standard_normal((N, N))
    A[:, -1] = 0.0                                                       # U[N-1, N-1] = 0 exactly
    rs = _lu_on_grid(N, v, 1, 1, 1, [A])
    rcond, anorm = rs[0]["r"]
    assert rcond == 0.0 and abs(anorm - _norm1(A)) <= 1e-15 * anorm


def test_lu_rcond_state_rules_and_side_effects():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(512, 512, 64, 1, 1, 1, comm)
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_rcond(gv)                                                  # no factorisation yet
    cb.LU_rep(gv)
    B = np.random.default_rng(3).standard_normal((gv.M, 5))
    X0, Xt0 = cb.lu_solve(gv, B), cb.lu_solve(gv, B, trans=True)
    C0, p0 = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C0.ctypes.data, p0.ctypes.data), "get_factors")
    r0 = cb.validate(gv)
    import ctypes
    n0, n1 = ctypes.c_int64(), ctypes.c_int64()
    cb.check(cb.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n0), 0), "launch_count")
    cb.lu_rcond(gv)
    cb.check(cb.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n1), 0), "launch_count")
    assert n0.value == n1.value
    C1, p1 = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C1.ctypes.data, p1.ctypes.data), "get_factors")
    assert np.array_equal(C0, C1) and np.array_equal(p0, p1) and cb.validate(gv) == r0
    assert np.array_equal(cb.lu_solve(gv, B), X0) and np.array_equal(cb.lu_solve(gv, B, trans=True), Xt0)
    a = np.ascontiguousarray(gv.data)
    cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_rcond(gv)                                                  # new input, not factored yet
    gv.free_comms()
    comm.close()


def test_lu_rcond_refused_when_input_was_handed_on():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(256, 256, 32, 1, 1, 1, comm)
    mats = [cb.pinned_empty((gv.Ml, gv.Nl)) for _ in range(2)]
    rng = np.random.default_rng(4)
    for m in mats:
        m[...] = rng.standard_normal((gv.Ml, gv.Nl))
    gv.data = mats[0]
    cb.LU_rep(gv, next_data=mats[1])
    with pytest.raises(cb.ConfluxError, match="queued next matrix"):
        cb.lu_rcond(gv)
    cb.LU_rep(gv, upload=False)
    rcond, anorm = cb.lu_rcond(gv)                                       # the streamed matrix's own run: allowed
    assert rcond > 0 and abs(anorm - _norm1(mats[1])) <= 1e-15 * anorm
    for m in mats:
        cb.pinned_free(m)
    gv.free_comms()
    comm.close()


@pytest.mark.parametrize("N,v,Px,Py,Pz", LU_GRIDS)
def test_multi_gpu_lu_rcond(N, v, Px, Py, Pz):
    if n_gpus() < Px * Py * Pz:
        pytest.skip(f"needs {Px * Py * Pz} GPUs")
    _check_lu(_lu_on_grid(N, v, Px, Py, Pz), N, v, Px, Py, Pz, f"lu grid {Px}x{Py}x{Pz}")


# ----------------------------------------------------------------------------------------------- Cholesky
def _chol_on_grid(N, v, grid, A=None):
    locs = chol_solve_ref.scatter(A, N, v, *grid) if A is not None else None

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        if locs is not None:
            ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        import ctypes
        n0, n1 = ctypes.c_int64(), ctypes.c_int64()
        cb.check(cb.lib().cflx_chol_launch_count(ch._h, ctypes.byref(n0), 0), "launch_count")
        L0 = ch.local_factor()
        r = ch.rcond()
        cb.check(cb.lib().cflx_chol_launch_count(ch._h, ctypes.byref(n1), 0), "launch_count")
        out = dict(A=ch.data.copy(), L=ch.local_factor(), r=r, r2=ch.rcond(), same=np.array_equal(L0, ch.local_factor()),
                   launches=(n0.value, n1.value))
        ch.finalize()
        return out

    return run_ranks(grid[0] * grid[1] * grid[2], body)


def _check_chol(rs, N, v, grid, what):
    As = chol_ref.assemble([r["A"] for r in rs], N, v, *grid)
    A = chol_ref.lower_sym(As)
    L = np.tril(chol_ref.assemble([r["L"] for r in rs], N, v, *grid))
    rcond, anorm = rs[0]["r"]
    for r in rs:
        assert r["r"] == (rcond, anorm) and r["r2"] == (rcond, anorm)
        assert r["same"] and r["launches"][0] == r["launches"][1]
    want, info = lapack.dpocon(L, anorm, uplo="L")
    assert info == 0
    _check_rcond(A, rcond, anorm, want, what)


@pytest.mark.parametrize("N,v", [(100, 16), (256, 32), (512, 128), (1024, 256)])
def test_chol_rcond_generator(N, v):
    _check_chol(_chol_on_grid(N, v, (1, 1, 1)), N, v, (1, 1, 1), f"chol gen {N}/{v}")


def test_chol_rcond_normal_and_ill_conditioned():
    N, v = 512, 64
    G = np.random.default_rng(5).standard_normal((N, N))
    _check_chol(_chol_on_grid(N, v, (1, 1, 1), G @ G.T + N * np.eye(N)), N, v, (1, 1, 1), "chol normal")
    Q, _ = np.linalg.qr(np.random.default_rng(6).standard_normal((N, N)))
    A = (Q * np.logspace(0, -8, N)) @ Q.T
    A = (A + A.T) / 2
    _check_chol(_chol_on_grid(N, v, (1, 1, 1), A), N, v, (1, 1, 1), "chol kappa 1e8")


def test_chol_rcond_state_rules():
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(256, 32, (1, 1, 1), comm)
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.rcond()                                                       # no factorisation yet
    ch.parallelCholesky()
    ch.rcond()
    a = np.ascontiguousarray(ch.data)
    cb.check(cb.lib().cflx_chol_set_local(ch._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.rcond()
    ch.finalize()
    ch = cb.cholesky.initialize(256, 32, (1, 1, 1), comm)
    ch.data[...] = -np.eye(256)                                          # not positive definite
    with pytest.raises(cb.ConfluxError):
        ch.parallelCholesky()
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.rcond()
    ch.finalize()
    comm.close()


@pytest.mark.parametrize("N,v,grid", CHOL_GRIDS)
def test_multi_gpu_chol_rcond(N, v, grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    _check_chol(_chol_on_grid(N, v, grid), N, v, grid, f"chol grid {grid}")
