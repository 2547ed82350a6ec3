"""GPU: cflx_lu_refine_x / cflx_chol_refine_x (LAPACK dgerfsx / dporfsx on the grid) and their double-double residual
kernels.

  * dbg.residual_x in every mode, at off-origin grid positions, with Kappa short of the share and NaN wherever the
    kernel must not read: b - (Hi + Lo), rounded as the assembly rounds it, meets |r^ - r| <= 2u|r| + (K u)^2 (|op A|
    (|y| + |y_tail|) + |b|) against the correctly rounded r, on inputs where b is op(A) y rounded -- where the FP64
    residual kernel (dbg.residual) violates the same bound, so the test discriminates;
  * lu_refine_x (trans 0 and 1) and cholesky.refine_x from the plain solve's X on Q1 diag(sigma) Q2 matrices with kappa
    from 1e2 to 1e17 (and the generator at N = 100): trusted bounds hold against the double-double solution of
    tests/test_refinex_ref.py, kappa M u <= 1e-2 gives trusted bounds at ERR_LBND, kappa >= 100 / (M u) untrusted ones
    and info = M + 1; for 1e10 <= kappa <= 1e-2 / (M u) the error is at least 100x below lu_refine's.  The trust flags
    and info equal oracle.refinex_ref's on the device's own factors away from the thresholds;
  * an equilibrated (column-scaled) input, cwise=False, the zero pivot, determinism, no side effects, the argument and
    state rules, and the multi-GPU grids (skipped on fewer GPUs).  Observed errors are printed with -s."""
import ctypes
import math

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, layout
from oracle import refine_ref as rr
from oracle import refinex_ref as rx
from tests._harness import n_gpus, run_ranks
from tests.test_refinex_ref import errors, true_solution

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
CFLX_ERR_ARG, CFLX_ERR_STATE = -1, -5                                     # include/conflux_b200.h


# ----------------------------------------------------------------------------------------------- the kernel
def _round_residual(b, H, L):
    s = b - H
    bb = s - b
    e = (b - (s - bb)) + (-H - bb)
    return s + (e - L)


@pytest.mark.parametrize("mode,v,Kappa,Px,Py,pi,pj,mt,nt", [("nn", 16, 1 << 30, 2, 3, 1, 2, 5, 4),
                                                             ("tn", 16, 1 << 30, 3, 2, 2, 1, 4, 6),
                                                             ("sym", 16, 5, 2, 2, 1, 0, 3, 3),
                                                             ("sym", 8, 9, 2, 3, 0, 2, 5, 3)])
@pytest.mark.parametrize("nrhs", [1, 3, 8, 13])
def test_residual_x_kernel(mode, v, Kappa, Px, Py, pi, pj, mt, nt, nrhs):
    Ml, Nl = mt * v, nt * v
    rng = np.random.default_rng(mt * 100 + nrhs)
    A = rng.standard_normal((Ml, Nl)) * np.exp(rng.uniform(-3, 3, (Ml, Nl)))
    Xc, Xr = rng.standard_normal((Nl, nrhs)), rng.standard_normal((Ml, nrhs))
    Xct, Xrt = Xc * 1e-17 * rng.standard_normal(Xc.shape), Xr * 1e-17 * rng.standard_normal(Xr.shape)
    if mode == "sym":
        mnn, mtn = rr.sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj)
        A[~mnn] = np.nan
        ops = [(np.where(mnn, A, 0.0), Xc, Xct, slice(0, Ml)), (np.where(mtn, A, 0.0).T, Xr, Xrt, slice(Ml, Ml + Nl))]
    elif mode == "nn":
        ops = [(A, Xc, Xct, slice(0, Ml))]
    else:
        ops = [(A.T, Xr, Xrt, slice(0, Nl))]
    args = dict(Kappa=Kappa, grid=(Px, Py), pos=(pi, pj), Xc=Xc, Xr=Xr)
    H, L, _ = cb.dbg.residual_x(A, mode, v, Xc_tail=Xct, Xr_tail=Xrt, **args)
    H2, L2, _ = cb.dbg.residual_x(A, mode, v, Xc_tail=Xct, Xr_tail=Xrt, **args)
    assert np.array_equal(H, H2) and np.array_equal(L, L2)
    P, _, _ = cb.dbg.residual(A, mode, v, **args)
    violated = False
    for Aop, Y, T, rows in ops:
        B = -rx.exact_residual(Aop, np.zeros((Aop.shape[0], nrhs)), Y)          # op(A) y rounded: r is tiny
        r = rx.exact_residual(Aop, B, Y, T)
        K = Aop.shape[1]
        tol = 2 * U * np.abs(r) + (K * U) ** 2 * (np.abs(Aop) @ (np.abs(Y) + np.abs(T)) + np.abs(B))
        rh = _round_residual(B, H[rows], L[rows])
        assert np.all(np.abs(rh - r) <= tol), (mode, np.max(np.abs(rh - r) / tol))
        violated |= bool(np.any(np.abs((B - P[rows]) - r) > tol))
    assert violated                                                      # the FP64 kernel does not meet it


def test_residual_x_tail_none_is_zero():
    rng = np.random.default_rng(1)
    A, Xc = rng.standard_normal((32, 48)), rng.standard_normal((48, 2))
    H, L, _ = cb.dbg.residual_x(A, "nn", 16, Xc=Xc)
    H2, L2, _ = cb.dbg.residual_x(A, "nn", 16, Xc=Xc, Xc_tail=np.zeros_like(Xc))
    assert np.array_equal(H, H2) and np.array_equal(L, L2)


# ----------------------------------------------------------------------------------------------- LU
def _kappa_matrix(n, kappa, seed, col_scale=None):
    rng = np.random.default_rng(seed)
    Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
    Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q1 * np.logspace(0, -math.log10(kappa), n)) @ Q2.T
    return A if col_scale is None else A * col_scale[None, :]


def _lu_case(N, v, A=None, nrhs=3, seed=0, equilibrate=False, grid=(1, 1, 1)):
    Px, Py, Pz = grid
    d = layout.dims(N, v, Px, Py, Pz)
    locs = layout.scatter(A, v, Px, Py, Pz) if A is not None else None
    B = np.random.default_rng(seed).standard_normal((d["M"], nrhs))

    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        if locs is not None:
            gv.data[...] = locs[gv.rank]
        eq = None
        if equilibrate:
            eq = cb.lu_equilibrate(gv)
            cb.LU_rep(gv, upload=False)
        C = np.zeros((gv.Ml, gv.Nl))
        perm = np.zeros(gv.M, dtype=np.int32)
        if not equilibrate:
            cb.LU_rep(gv, C, perm)
        else:
            cb.check(cb.lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "get_factors")
        n0, n1 = ctypes.c_int64(), ctypes.c_int64()
        out = dict(C=C, perm=perm, eq=eq)
        for t in (False, True):
            X0 = cb.lu_solve(gv, B, trans=t)
            cb.check(cb.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n0), 0), "launch_count")
            X, r = cb.lu_refine_x(gv, B, X0, trans=t)
            cb.check(cb.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n1), 0), "launch_count")
            X2, r2 = cb.lu_refine_x(gv, B, X0, trans=t)
            X3, r3 = cb.lu_refine_x(gv, B, X0, trans=t, cwise=False)
            assert n0.value == n1.value
            assert np.array_equal(X, X2) and all(np.array_equal(r[k], r2[k]) for k in r)
            assert r3["err_comp"] is None and r3["err_norm"].shape == (nrhs, 3)
            assert np.array_equal(cb.lu_solve(gv, B, trans=t), X0)      # later solves: the same bits
            Xw = cb.lu_refine(gv, B, X0, trans=t, ferr=False)[0]
            out[t] = (X0, X, r, Xw)
        C2 = np.zeros_like(C)
        cb.check(cb.lib().cflx_lu_get_factors(gv._h, C2.ctypes.data, None), "get_factors")
        assert np.array_equal(C, C2)
        out["A"] = gv.data.copy()
        gv.free_comms()
        return out

    rs = run_ranks(Px * Py * Pz, body)
    for r in rs[1:]:
        for t in (False, True):
            assert np.array_equal(r[t][1], rs[0][t][1])
            assert all(np.array_equal(r[t][2][k], rs[0][t][2][k]) for k in ("berr", "err_norm", "err_comp"))
    return rs, B, d


def _check_lu(rs, B, d, N, v, kappa, what, grid=(1, 1, 1)):
    M = d["M"]
    LU = layout.assemble([r["C"] for r in rs], N, v, *grid)
    As = layout.assemble([r["A"] for r in rs], N, v, *grid)
    eq = rs[0]["eq"]
    if eq is not None:                                                   # the matrix the factors represent, as dlaqge
        r_ = eq["r"] if eq["equed"] in ("R", "B") else np.ones(M)        # rounds it: (c_j r_i) a_ij
        c_ = eq["c"] if eq["equed"] in ("C", "B") else np.ones(M)
        As = (c_[None, :] * r_[:, None]) * As
    perm = rs[0]["perm"]
    for t in (False, True):
        X0, X, r, Xw = rs[0][t]
        dvec = None
        if eq is not None and eq["equed"] in ("C", "B") and not t:
            dvec = eq["c"]
        if eq is not None and eq["equed"] in ("R", "B") and t:
            dvec = eq["r"]
        solve, solve_t = rr.lu_solvers(LU, perm, t)
        Aop = As.T if t else As
        Xt, Tt = true_solution(Aop, B, solve)
        nw, cw = errors(X, Xt, Tt, dvec)
        nww, _ = errors(Xw, Xt, Tt, dvec)
        en, ec, info = r["err_norm"], r["err_comp"], r["info"]
        print(f"refine_x {what} trans={int(t)}: err={nw.max():.2e} (refine {nww.max():.2e}) bound={en[:, 1].max():.2e} "
              f"trust={en[:, 0].min():.0f} rcond_norm={en[0, 2]:.2e} info={info}")
        for j in range(B.shape[1]):
            if en[j, 0] == 1:
                assert nw[j] <= en[j, 1], (what, t, j)
            if ec[j, 0] == 1:
                assert cw[j] <= ec[j, 1], (what, t, j)
        if kappa is not None and kappa * M * U <= 1e-2:
            assert np.all(en[:, 0] == 1) and np.all(nw <= max(10, math.sqrt(M)) * U), (what, t)
        if kappa is not None and kappa >= 100 / (M * U):
            assert np.all(en[:, 0] == 0) and info == M + 1, (what, t)
        if kappa is not None and 1e10 <= kappa <= 1e-2 / (M * U):
            assert np.all(nw * 100 <= nww), (what, t, nw, nww)
        # the restatement on the device's factors: the same trust flags and info away from the thresholds
        rcond = r["rcond"]
        ref = rx.gerfsx(As, B, X0, solve, solve_t, rcond, t, dvec)
        rn = en[0, 2]
        if not (0.1 < rn / (M * U) < 10):
            assert np.array_equal(ref[2][:, 0], en[:, 0]), (what, t)
            if info == 0 or info == M + 1:
                assert (ref[4] == 0) == (info == 0), (what, t, ref[4], info)


@pytest.mark.parametrize("N,v,kappa", [(100, 16, None), (512, 64, 1e2), (512, 64, 1e10), (512, 64, 1e17),
                                       (1024, 128, 1e6), (1024, 128, 1e10), (1024, 128, 1e15)])
def test_lu_refine_x(N, v, kappa):
    A = _kappa_matrix(N, kappa, N + int(math.log10(kappa))) if kappa else None
    rs, B, d = _lu_case(N, v, A, seed=N)
    _check_lu(rs, B, d, N, v, kappa, f"lu {N}/{v} kappa={kappa}")


def test_lu_refine_x_equilibrated():
    N, v = 512, 64
    s = np.logspace(0, 10, N)
    np.random.default_rng(2).shuffle(s)
    A = _kappa_matrix(N, 1e6, 9, col_scale=s)
    rs, B, d = _lu_case(N, v, A, seed=3, equilibrate=True)
    assert rs[0]["eq"]["equed"] in ("C", "B")
    _check_lu(rs, B, d, N, v, None, "lu equilibrated")
    # trans 0: the bound is for x = diag(c) y, whose condition is that of the unscaled, column-scaled input
    assert rs[0][False][2]["info"] == d["M"] + 1 and np.all(rs[0][True][2]["err_norm"][:, 0] == 1)


def test_lu_refine_x_zero_pivot_and_rules():
    N, v = 64, 16
    A = np.random.default_rng(5).standard_normal((N, N))
    A[:, 7] = 0.0

    def body(comm):
        gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
        B = np.ones((gv.M, 2))
        X = np.full((gv.M, 2), 3.0)
        L = cb.lib()
        info, rc = ctypes.c_int(), ctypes.c_double()
        en = np.zeros((2, 3))
        # before any factorisation: a state error
        rcode = L.cflx_lu_refine_x(gv._h, 0, 2, B.ctypes.data, 2, X.ctypes.data, 2, None, None, en.ctypes.data, None,
                                   ctypes.byref(info))
        assert rcode == CFLX_ERR_STATE
        gv.data[...] = layout.scatter(A, v, 1, 1, 1)[0]
        cb.LU_rep(gv)
        Xr, r = cb.lu_refine_x(gv, B, X)
        assert r["info"] == 8 and np.array_equal(Xr, X) and r["rcond"] == 0.0
        for bad in (dict(trans=2), dict(nrhs=0), dict(info=None), dict(en=None)):
            rcode = L.cflx_lu_refine_x(gv._h, bad.get("trans", 0), bad.get("nrhs", 2), B.ctypes.data, 2, X.ctypes.data,
                                       2, None, None, None if "en" in bad else en.ctypes.data, None,
                                       None if "info" in bad else ctypes.byref(info))
            assert rcode == CFLX_ERR_ARG, bad
        gv.free_comms()

    run_ranks(1, body)


# ----------------------------------------------------------------------------------------------- Cholesky
def _chol_case(N, v, kappa, grid=(1, 1, 1), nrhs=3, seed=0):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((N, N)))
    A = (Q * np.logspace(0, -math.log10(kappa), N)) @ Q.T
    A = (A + A.T) / 2
    locs = chol_solve_ref.scatter(A, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)
    n = chol_ref.dims(N, v, *grid)["N"]
    B = rng.standard_normal((n, nrhs))

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        L0 = ch.local_factor()
        X0 = ch.solve(B)
        X, r = ch.refine_x(B, X0)
        X2, r2 = ch.refine_x(B, X0)
        assert np.array_equal(X, X2) and all(np.array_equal(r[k], r2[k]) for k in r)
        assert np.array_equal(L0, ch.local_factor(), equal_nan=True) and np.array_equal(ch.solve(B), X0)
        Xw = ch.refine(B, X0, ferr=False)[0]
        out = dict(A=ch.data.copy(), L=L0, res=(X0, X, r, Xw))
        ch.finalize()
        return out

    rs = run_ranks(grid[0] * grid[1] * grid[2], body)
    for r in rs[1:]:
        assert np.array_equal(r["res"][1], rs[0]["res"][1])
    return rs, B, n


@pytest.mark.parametrize("N,v,kappa", [(512, 64, 1e2), (512, 64, 1e10), (1024, 128, 1e6)])
def test_chol_refine_x(N, v, kappa):
    grid = (1, 1, 1)
    rs, B, n = _chol_case(N, v, kappa, grid, seed=N)
    A = chol_ref.lower_sym(chol_ref.assemble([np.nan_to_num(r["A"], nan=0.0) for r in rs], N, v, *grid))
    L = np.tril(chol_ref.assemble([np.nan_to_num(r["L"], nan=0.0) for r in rs], N, v, *grid))
    X0, X, r, Xw = rs[0]["res"]
    solve = rr.chol_solver(L)
    Xt, Tt = true_solution(A, B, solve)
    nw, cw = errors(X, Xt, Tt)
    nww, _ = errors(Xw, Xt, Tt)
    en = r["err_norm"]
    print(f"chol refine_x {N}/{v} kappa={kappa:g}: err={nw.max():.2e} (refine {nww.max():.2e}) bound={en[:, 1].max():.2e}")
    assert np.all(en[:, 0] == 1) and np.all(nw <= en[:, 1])
    if 1e10 <= kappa <= 1e-2 / (n * U):
        assert np.all(nw * 100 <= nww)
    ref = rx.porfsx(A, B, X0, solve, r["rcond"])
    assert np.array_equal(ref[2][:, 0], en[:, 0])


# ----------------------------------------------------------------------------------------------- multi-GPU
@pytest.mark.parametrize("N,v,grid", [(256, 32, (2, 2, 1)), (256, 32, (2, 2, 2))])
def test_multi_gpu_lu_refine_x(N, v, grid):
    if n_gpus() < grid[0] * grid[1] * grid[2]:
        pytest.skip(f"needs {grid[0] * grid[1] * grid[2]} GPUs")
    A = _kappa_matrix(N, 1e10, 4)
    rs, B, d = _lu_case(N, v, A, seed=1, grid=grid)
    _check_lu(rs, B, d, N, v, 1e10, f"lu grid {grid}", grid)
