"""GPU: cflx_lu_refine / cflx_chol_refine (LAPACK dgerfs / dporfs on the grid) and their residual kernels.

  * dbg.residual in every mode against exact products (hp_ref.matmul): |P - op(A) X| <= gamma_K |op(A)| |X| and
    |Q - |op(A)| |X|| <= gamma_K |op(A)| |X| componentwise, K the reduction length; the symmetric mode with NaN in every
    entry it must not read (above the diagonal, beyond Kappa);
  * refinement from the X of the plain solve, on the device's own factors:
      - berr <= max(2 berr_LAPACK, BERR_FLOOR), berr_LAPACK from scipy's dgesvx / dposvx (fact='F') on the same factors,
        and the long-double backward error of the returned X meets the same bound.  BERR_FLOOR = 4u, not u: once
        refinement has converged, the berr either side reports is the rounding of its own residual evaluation (its
        products' summation order), a few u for any order; on the H100 the device reported up to 2.4u where LAPACK
        reported 0.8u on the same row-scaled matrix, while the long-double backward errors of both X were about 1u;
      - ferr within a factor FERR_RATIO = 2 of LAPACK's (the estimator takes LAPACK's steps; its products are solves whose
        rounding differs from LAPACK's, which moves the estimate by far less than 2x on these matrices);
      - ferr >= the true relative forward error against a long-double solution;
      - on row- and column-scaled matrices, the refined backward error is at least 5x below the unrefined one.
    For trans = 1, scipy's dgesvx(trans='T', fact='F') on the device's factors returned berr near 1 (an X that does not
    solve A^T X = B), so the trans = 1 cases take the LAPACK numbers from oracle.refine_ref.gerfs on the same factors: the
    numpy restatement of dgerfs that tests/test_refine_ref.py checks against dgesvx;
  * determinism and side effects, ferr=None, the state and argument rules, and the multi-GPU grids of test_gpu_rcond.py.
The observed margins are printed with -s."""
import ctypes

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, hp_ref, layout
from oracle import refine_ref as rr
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -53
FERR_RATIO = 2.0
BERR_FLOOR = 4 * EPS
LU_GRIDS = [(64, 8, 2, 2, 1), (128, 16, 1, 1, 2), (128, 8, 2, 2, 2), (512, 64, 2, 2, 2)]
CHOL_GRIDS = [(256, 32, (2, 2, 1)), (256, 32, (1, 1, 2)), (384, 32, (3, 2, 1)), (512, 64, (2, 2, 2))]


# ----------------------------------------------------------------------------------------------- the kernel
def _check_kernel(P, Q, Aop, X, what):
    K = Aop.shape[1]
    Pe = hp_ref.matmul(Aop, X)
    Qe = hp_ref.matmul(np.abs(Aop), np.abs(X))
    g = hp_ref.gamma(K)
    tol = g * np.asarray(Qe, dtype=np.float64)
    assert np.all(np.abs(P - np.asarray(Pe, dtype=np.float64)) <= tol), what
    assert np.all(np.abs(Q - np.asarray(Qe, dtype=np.float64)) <= tol), what


@pytest.mark.parametrize("Ml,Nl,v", [(36, 44, 4), (100, 48, 16), (200, 520, 4), (512, 256, 256)])
@pytest.mark.parametrize("nrhs", [1, 7, 64, 200])
def test_residual_kernel_nn_tn(Ml, Nl, v, nrhs):
    rng = np.random.default_rng(Ml * 1000 + nrhs)
    A = rng.standard_normal((Ml, Nl)) * np.exp(rng.uniform(-5, 5, (Ml, Nl)))
    Xc, Xr = rng.standard_normal((Nl, nrhs)), rng.standard_normal((Ml, nrhs))
    P, Q, _ = cb.dbg.residual(A, "nn", v, Xc=Xc)
    _check_kernel(P, Q, A, Xc, f"nn {Ml}x{Nl} nrhs={nrhs}")
    P, Q, _ = cb.dbg.residual(A, "tn", v, Xr=Xr)
    _check_kernel(P, Q, A.T, Xr, f"tn {Ml}x{Nl} nrhs={nrhs}")
    P2, Q2, _ = cb.dbg.residual(A, "tn", v, Xr=Xr)
    assert np.array_equal(P, P2) and np.array_equal(Q, Q2)                 # the same call, the same bits


@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj,mt,nt", [(4, 9, 2, 3, 1, 2, 5, 3), (16, 5, 2, 2, 0, 1, 3, 3),
                                                         (16, 3, 1, 1, 0, 0, 4, 4), (256, 2, 1, 1, 0, 0, 2, 2)])
@pytest.mark.parametrize("nrhs", [1, 7, 64, 200])
def test_residual_kernel_symmetric_masks(v, Kappa, Px, Py, pi, pj, mt, nt, nrhs):
    Ml, Nl = mt * v, nt * v
    rng = np.random.default_rng(v * 100 + nrhs)
    A = rng.standard_normal((Ml, Nl))
    mnn, mtn = rr.sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj)
    A[~mnn] = np.nan                                                   # everything the kernel must not read
    Xc, Xr = rng.standard_normal((Nl, nrhs)), rng.standard_normal((Ml, nrhs))
    P, Q, _ = cb.dbg.residual(A, "sym", v, Kappa, (Px, Py), (pi, pj), Xc=Xc, Xr=Xr)
    An, At = np.where(mnn, A, 0.0), np.where(mtn, A, 0.0)
    _check_kernel(P[:Ml], Q[:Ml], An, Xc, "sym nn")
    _check_kernel(P[Ml:], Q[Ml:], At.T, Xr, "sym tn")


# ----------------------------------------------------------------------------------------------- LU
def _scaled(n, kind, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    s = np.logspace(0, 12, n)
    rng.shuffle(s)
    if kind == "rows":
        return A * s[:, None]
    if kind == "cols":
        return A * s[None, :]
    if kind == "kappa":
        Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
        Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
        return (Q1 * np.logspace(0, -8, n)) @ Q2.T
    return A


def _lu_run(N, v, Px, Py, Pz, A=None, nrhs=5, seed=0):
    d = layout.dims(N, v, Px, Py, Pz)
    locs = layout.scatter(A, v, Px, Py, Pz) if A is not None else None    # A: N a multiple of v * Px
    B = np.random.default_rng(seed).standard_normal((d["M"], nrhs))

    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        if locs is not None:
            gv.data[...] = locs[gv.rank]
        C = np.zeros((gv.Ml, gv.Nl))
        perm = np.zeros(gv.M, dtype=np.int32)
        cb.LU_rep(gv, C, perm)
        out = dict(A=gv.data.copy(), C=C, perm=perm)
        for t in (False, True):
            X0 = cb.lu_solve(gv, B, trans=t)
            X, fe, be = cb.lu_refine(gv, B, X0, trans=t)
            X2, fe2, be2 = cb.lu_refine(gv, B, X0, trans=t)
            X3, fe3, be3 = cb.lu_refine(gv, B, X0, trans=t, ferr=False)
            assert np.array_equal(X, X2) and np.array_equal(fe, fe2) and np.array_equal(be, be2)
            assert fe3 is None and np.array_equal(X, X3) and np.array_equal(be, be3)
            out[t] = (X0, X, fe, be)
        gv.free_comms()
        return out

    rs = run_ranks(Px * Py * Pz, body)
    for r in rs[1:]:
        for t in (False, True):
            assert all(np.array_equal(a, b) for a, b in zip(r[t], rs[0][t]))   # every rank: the same bits
    return rs, B, d


def _check_refined(Ag, B, X0, X, fe, be, lap, trans, what, scaled):
    Xl, fe_l, be_l = lap
    bound = np.maximum(2 * be_l, BERR_FLOOR)
    bw = rr.backward_error(Ag, B, X, trans)
    bw0 = rr.backward_error(Ag, B, X0, trans)
    Ao = (Ag.T if trans else Ag).astype(np.longdouble)
    Xt = np.linalg.solve(Ag.T if trans else Ag, B)
    for _ in range(3):                                                   # long-double refinement of the true solution
        Xt = Xt + np.linalg.solve(Ag.T if trans else Ag, np.asarray(B - Ao @ Xt.astype(np.longdouble), dtype=np.float64))
    fwd = np.asarray(np.max(np.abs(X.astype(np.longdouble) - Xt), 0) / np.max(np.abs(X), 0), dtype=np.float64)
    ratio = np.maximum(fe / fe_l, fe_l / fe)
    print(f"refine {what}: berr={be.max():.2e} lapack={be_l.max():.2e} host={bw.max():.2e} unrefined={bw0.max():.2e} "
          f"ferr={fe.max():.2e} lapack={fe_l.max():.2e} ratio={ratio.max():.3f} fwd/ferr={(fwd / fe).max():.2e}")
    assert np.all(be <= bound) and np.all(bw <= bound), what
    assert np.all(ratio <= FERR_RATIO), what
    assert np.all(fe >= fwd), what
    if scaled:
        assert np.all(bw * 5 <= bw0), what


def _check_lu(rs, B, d, N, v, Px, Py, Pz, kind, what):
    Ag = layout.assemble([r["A"] for r in rs], N, v, Px, Py, Pz)
    LU = layout.assemble([r["C"] for r in rs], N, v, Px, Py, Pz)
    perm = rs[0]["perm"]
    ipiv = rr.perm_to_ipiv(perm)
    for t in (False, True):
        X0, X, fe, be = rs[0][t]
        Xl, fe_l, be_l, info = rr.lapack_gesvx(Ag, LU, ipiv, B, t)
        assert info == 0, what
        if t:
            s, st = rr.lu_solvers(LU, perm, t)
            _, fe_l, be_l = rr.gerfs(Ag, B, s(B), s, st, t)
        _check_refined(Ag, B, X0, X, fe, be, (Xl, fe_l, be_l), t, f"{what} trans={int(t)}", kind in ("rows", "cols"))


@pytest.mark.parametrize("N,v", [(16, 4), (96, 16), (512, 64), (1024, 128), (100, 16)])
@pytest.mark.parametrize("nrhs", [1, 5])
def test_lu_refine_generator(N, v, nrhs):
    rs, B, d = _lu_run(N, v, 1, 1, 1, nrhs=nrhs, seed=N)
    _check_lu(rs, B, d, N, v, 1, 1, 1, "gen", f"lu gen {N}/{v} nrhs={nrhs}")


@pytest.mark.parametrize("kind", ["rows", "cols", "kappa"])
def test_lu_refine_scaled_and_ill_conditioned(kind):
    N, v = 256, 32
    rs, B, d = _lu_run(N, v, 1, 1, 1, A=_scaled(N, kind, 11), nrhs=3, seed=5)
    _check_lu(rs, B, d, N, v, 1, 1, 1, kind, f"lu {kind}")


def test_lu_refine_state_rules_and_side_effects():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(512, 512, 64, 1, 1, 1, comm)
    B = np.random.default_rng(3).standard_normal((gv.M, 5))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_refine(gv, B, B)                                           # no factorisation yet
    cb.LU_rep(gv)
    X0, Xt0 = cb.lu_solve(gv, B), cb.lu_solve(gv, B, trans=True)
    C0, p0 = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C0.ctypes.data, p0.ctypes.data), "get_factors")
    r0, rc0 = cb.validate(gv), cb.lu_rcond(gv)
    n0, n1 = ctypes.c_int64(), ctypes.c_int64()
    cb.check(cb.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n0), 0), "launch_count")
    cb.lu_refine(gv, B, X0)
    cb.lu_refine(gv, B, Xt0, trans=True)
    cb.check(cb.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n1), 0), "launch_count")
    assert n0.value == n1.value
    C1, p1 = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C1.ctypes.data, p1.ctypes.data), "get_factors")
    assert np.array_equal(C0, C1) and np.array_equal(p0, p1) and cb.validate(gv) == r0 and cb.lu_rcond(gv) == rc0
    assert np.array_equal(cb.lu_solve(gv, B), X0) and np.array_equal(cb.lu_solve(gv, B, trans=True), Xt0)
    h, Bc, Xc = gv._h, np.ascontiguousarray(B), X0.copy()
    fe, be = np.empty(5), np.empty(5)
    args = lambda trans, n, ldb, ldx, b, x: (h, trans, n, b, ldb, x, ldx, fe.ctypes.data, be.ctypes.data)
    for bad in [args(2, 5, 5, 5, Bc.ctypes.data, Xc.ctypes.data), args(0, 0, 5, 5, Bc.ctypes.data, Xc.ctypes.data),
                args(0, 5, 4, 5, Bc.ctypes.data, Xc.ctypes.data), args(0, 5, 5, 4, Bc.ctypes.data, Xc.ctypes.data),
                args(0, 5, 5, 5, None, Xc.ctypes.data), args(0, 5, 5, 5, Bc.ctypes.data, None)]:
        assert cb.lib().cflx_lu_refine(*bad) == -1
    a = np.ascontiguousarray(gv.data)
    cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_refine(gv, B, X0)                                          # new input, not factored yet
    gv.free_comms()
    comm.close()


def test_lu_refine_refused_when_input_was_handed_on():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(256, 256, 32, 1, 1, 1, comm)
    mats = [cb.pinned_empty((gv.Ml, gv.Nl)) for _ in range(2)]
    rng = np.random.default_rng(4)
    for m in mats:
        m[...] = rng.standard_normal((gv.Ml, gv.Nl))
    gv.data = mats[0]
    B = rng.standard_normal((gv.M, 2))
    cb.LU_rep(gv, next_data=mats[1])
    with pytest.raises(cb.ConfluxError, match="queued next matrix"):
        cb.lu_refine(gv, B, cb.lu_solve(gv, B))
    cb.LU_rep(gv, upload=False)
    X, fe, be = cb.lu_refine(gv, B, cb.lu_solve(gv, B))                 # the streamed matrix's own run: allowed
    assert np.all(be <= 1e-14) and np.all(np.isfinite(fe))
    for m in mats:
        cb.pinned_free(m)
    gv.free_comms()
    comm.close()


@pytest.mark.parametrize("N,v,Px,Py,Pz", LU_GRIDS)
def test_multi_gpu_lu_refine(N, v, Px, Py, Pz):
    if n_gpus() < Px * Py * Pz:
        pytest.skip(f"needs {Px * Py * Pz} GPUs")
    rs, B, d = _lu_run(N, v, Px, Py, Pz, nrhs=3, seed=N)
    _check_lu(rs, B, d, N, v, Px, Py, Pz, "gen", f"lu grid {Px}x{Py}x{Pz}")


# ----------------------------------------------------------------------------------------------- Cholesky
def _chol_run(N, v, grid, A=None, nrhs=5, seed=0, nan=False):
    locs = None
    if A is not None:
        nan_or = lambda x: np.nan if nan else x
        locs = chol_solve_ref.scatter(A, N, v, *grid, upper=nan_or(None), pad=nan_or(0.0), layers=nan_or(0.0))
    B = np.random.default_rng(seed).standard_normal((chol_ref.dims(N, v, *grid)["N"], nrhs))

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        if locs is not None:
            ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        n0, n1 = ctypes.c_int64(), ctypes.c_int64()
        cb.check(cb.lib().cflx_chol_launch_count(ch._h, ctypes.byref(n0), 0), "launch_count")
        L0 = ch.local_factor()
        X0 = ch.solve(B)
        X, fe, be = ch.refine(B, X0)
        X2, fe2, be2 = ch.refine(B, X0)
        X3, fe3, be3 = ch.refine(B, X0, ferr=False)
        cb.check(cb.lib().cflx_chol_launch_count(ch._h, ctypes.byref(n1), 0), "launch_count")
        assert np.array_equal(X, X2) and np.array_equal(fe, fe2) and np.array_equal(be, be2)
        assert fe3 is None and np.array_equal(X, X3) and np.array_equal(be, be3)
        assert np.array_equal(L0, ch.local_factor(), equal_nan=True) and n0.value == n1.value and np.array_equal(ch.solve(B), X0)
        out = dict(A=ch.data.copy(), L=L0, res=(X0, X, fe, be))
        ch.finalize()
        return out

    rs = run_ranks(grid[0] * grid[1] * grid[2], body)
    for r in rs[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(r["res"], rs[0]["res"]))
    return rs, B


def _check_chol(rs, B, N, v, grid, what, scaled=False):
    As = chol_ref.assemble([np.nan_to_num(r["A"], nan=0.0) for r in rs], N, v, *grid)
    A = chol_ref.lower_sym(As)
    L = np.tril(chol_ref.assemble([r["L"] for r in rs], N, v, *grid))
    X0, X, fe, be = rs[0]["res"]
    Xl, fe_l, be_l, info = rr.lapack_posvx(A, L, B)
    assert info == 0, what
    _check_refined(A, B, X0, X, fe, be, (Xl, fe_l, be_l), False, what, scaled)


@pytest.mark.parametrize("N,v", [(100, 16), (256, 32), (512, 128), (1024, 256)])
def test_chol_refine_generator(N, v):
    rs, B = _chol_run(N, v, (1, 1, 1), nrhs=5, seed=N)
    _check_chol(rs, B, N, v, (1, 1, 1), f"chol gen {N}/{v}")


def test_chol_refine_matrices():
    N, v = 512, 64
    G = np.random.default_rng(5).standard_normal((N, N))
    rs, B = _chol_run(N, v, (1, 1, 1), G @ G.T + N * np.eye(N), nrhs=1)
    _check_chol(rs, B, N, v, (1, 1, 1), "chol G G^T + N I")
    Q, _ = np.linalg.qr(np.random.default_rng(6).standard_normal((N, N)))
    A = (Q * np.logspace(0, -8, N)) @ Q.T
    rs, B = _chol_run(N, v, (1, 1, 1), (A + A.T) / 2, nrhs=3)
    _check_chol(rs, B, N, v, (1, 1, 1), "chol kappa 1e8")
    s = np.logspace(0, 6, N)
    np.random.default_rng(7).shuffle(s)
    A = (G @ G.T / N + np.eye(N)) * s[:, None] * s[None, :]
    rs, B = _chol_run(N, v, (1, 1, 1), A, nrhs=3)
    _check_chol(rs, B, N, v, (1, 1, 1), "chol diagonally scaled")


def test_chol_refine_nan_outside_the_lower_triangle():
    N, v = 384, 32
    G = np.random.default_rng(8).standard_normal((N, N))
    rs, B = _chol_run(N, v, (1, 1, 1), G @ G.T + N * np.eye(N), nrhs=3, nan=True)
    _check_chol(rs, B, N, v, (1, 1, 1), "chol NaN above the diagonal")


def test_chol_refine_state_rules():
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(256, 32, (1, 1, 1), comm)
    B = np.random.default_rng(9).standard_normal((ch.N, 2))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.refine(B, B)                                                  # no factorisation yet
    ch.parallelCholesky()
    X0 = ch.solve(B)
    ch.refine(B, X0)
    fe, be, Bc, Xc = np.empty(2), np.empty(2), np.ascontiguousarray(B), X0.copy()
    for n, ldb, ldx, b, x in [(0, 2, 2, Bc.ctypes.data, Xc.ctypes.data), (2, 1, 2, Bc.ctypes.data, Xc.ctypes.data),
                              (2, 2, 1, Bc.ctypes.data, Xc.ctypes.data), (2, 2, 2, None, Xc.ctypes.data),
                              (2, 2, 2, Bc.ctypes.data, None)]:
        assert cb.lib().cflx_chol_refine(ch._h, n, b, ldb, x, ldx, fe.ctypes.data, be.ctypes.data) == -1
    a = np.ascontiguousarray(ch.data)
    cb.check(cb.lib().cflx_chol_set_local(ch._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.refine(B, X0)
    ch.finalize()
    ch = cb.cholesky.initialize(256, 32, (1, 1, 1), comm)
    ch.data[...] = -np.eye(256)                                          # not positive definite
    with pytest.raises(cb.ConfluxError):
        ch.parallelCholesky()
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.refine(B, X0)
    ch.finalize()
    comm.close()


@pytest.mark.parametrize("N,v,grid", CHOL_GRIDS)
def test_multi_gpu_chol_refine(N, v, grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    rs, B = _chol_run(N, v, grid, nrhs=3, seed=N)
    _check_chol(rs, B, N, v, grid, f"chol grid {grid}")
