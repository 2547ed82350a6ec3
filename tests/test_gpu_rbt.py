"""GPU: random butterfly transforms (cflx_lu_rbt, cflx_lu_rbt_solve, cflx_lu_rbt_apply_local, cflx_dbg_rbt_share)
against the restatement (oracle/rbt_ref.py), numpy's solve, and the state and argument rules."""
import ctypes

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import layout, rbt_ref
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
EPS = np.finfo(float).eps
FACTOR_TOL = 1e-12        # ||L U - W||_F / ||W||_F, the bound of the fixed-order tests
BERR_TOL = 1e-13


def _one(N, v, body):
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    try:
        return body(gv)
    finally:
        gv.free_comms()
        comm.close()


def _count(gv):
    n = ctypes.c_int64()
    cb._lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n), 1)
    return n.value


def zero_leading_pivot(M, rng):
    """well conditioned with A[0, 0] = 0 exactly: a diagonally dominant D with D[1, 0] = 0, rows 0 and 1 swapped"""
    D = rng.standard_normal((M, M)) + 2.0 * M * np.eye(M)
    D[1, 0] = 0.0
    return D[[1, 0] + list(range(2, M))]


def _rel(X, Y):
    return np.abs(X - Y).max() / np.abs(Y).max()


# --------------------------------------------------------------------------------------------------------- the hook
@pytest.mark.parametrize("depth", [1, 2])
@pytest.mark.parametrize("op", [0, 1, 2, 3, 4])
def test_hook_matches_the_restatement_off_origin(op, depth):
    """grid position (1, 2) of a 2 x 3 layout: global rows and columns interleave with the other ranks'"""
    v, Ml, Nl = 8, 64, 64
    grid, pos = (2, 3), (1, 2)
    M = max(Ml * grid[0], Nl * grid[1])
    rng = np.random.default_rng(10 * op + depth)
    u, vv = cb.rbt_multipliers(M, depth, 77 + depth)
    X = rng.standard_normal((Ml, Nl if op == 4 else 7))
    got = cb.dbg.rbt_share(op, X, v, depth, u=u, vv=vv, grid=grid, pos=pos, M=M)
    want = rbt_ref.share_op(op, X, v, depth, u, vv, grid, pos)
    assert np.array_equal(got, want)


def test_hook_refusals():
    u, vv = cb.rbt_multipliers(64, 2, 0)
    X = np.ones((32, 32))
    for args in [dict(op=5), dict(op=4, M=16), dict(op=0, v=16), dict(op=4, vv=None), dict(op=0, u=None)]:
        kw = dict(op=0, X=X, v=8, depth=2, u=u, vv=vv, M=64)
        kw.update(args)
        with pytest.raises(cb.ConfluxError, match="refused"):
            cb.dbg.rbt_share(**kw)
    cb.dbg.rbt_share(1, X, 8, 2, u=None, vv=vv, M=64)          # V needs only v


# ----------------------------------------------------------------------------------------------- the factorisation
def test_multipliers_and_factors_of_w():
    N, v, depth, seed = 512, 32, 2, 12345

    def body(gv):
        A = zero_leading_pivot(N, np.random.default_rng(1))
        gv.data[...] = A
        u, vv = np.zeros((depth, N)), np.zeros((depth, N))
        C = np.zeros((gv.Ml, gv.Nl))
        _, nrepl, info = cb.LU_rep_rbt(gv, depth, seed, C=C, u_out=u, v_out=vv)
        ru, rv = cb.rbt_multipliers(N, depth, seed)
        assert np.array_equal(u, ru) and np.array_equal(vv, rv)
        assert (nrepl, info) == (0, 0)
        W = rbt_ref.global_w(A, u, vv)
        L, U = np.tril(C, -1) + np.eye(N), np.triu(C)
        rel = np.linalg.norm(L @ U - W) / np.linalg.norm(W)
        assert rel <= FACTOR_TOL, rel
        rel = cb.validate(gv)[1]                                # validate refers to W
        assert rel <= FACTOR_TOL, rel
    _one(N, v, body)


@pytest.mark.parametrize("N,v", [(1024, 64), (1024, 256), (4096, 64), (4096, 256)])
def test_zero_leading_pivot_needs_no_pivoting_after_the_transform(N, v):
    def body(gv):
        rng = np.random.default_rng(N + v)
        A = zero_leading_pivot(N, rng)
        assert A[0, 0] == 0.0
        gv.data[...] = A
        _, _, info = cb.LU_rep_fixed(gv, perm=np.arange(N))
        assert info == 1
        _, nrepl, info = cb.LU_rep_rbt(gv)
        assert (nrepl, info) == (0, 0)
        for trans in (False, True):
            for nrhs in (1, 7, 64):
                B = rng.standard_normal((N, nrhs))
                X, ferr, berr = cb.lu_rbt_solve(gv, B, trans=trans, refine=True)
                want = np.linalg.solve(A.T if trans else A, B)
                assert berr.max() <= BERR_TOL and np.isfinite(ferr).all()
                assert _rel(X, want) <= 1e-10
    _one(N, v, body)


@pytest.mark.parametrize("kind", ["normal", "init"])
def test_forward_error_within_the_condition_bound(kind):
    N, v = 1024, 64

    def body(gv):
        rng = np.random.default_rng(3)
        if kind == "normal":
            gv.data[...] = rng.standard_normal((N, N))
        A = gv.data.copy()
        cb.LU_rep(gv)
        rcond, _ = cb.lu_rcond(gv)
        _, _, info = cb.LU_rep_rbt(gv)
        assert info == 0
        B = rng.standard_normal((N, 7))
        for trans in (False, True):
            X, _, berr = cb.lu_rbt_solve(gv, B, trans=trans)
            want = np.linalg.solve(A.T if trans else A, B)
            assert berr.max() <= BERR_TOL
            err = np.abs(X - want).max(axis=0) / np.abs(want).max(axis=0)
            assert err.max() <= 100 * EPS / rcond
    _one(N, v, body)


# ---------------------------------------------------------------------------------------- distributed right-hand sides
@pytest.mark.parametrize("device", [False, True], ids=["host", "torch"])
@pytest.mark.parametrize("trans", [False, True])
def test_apply_local_around_solve_local_is_the_solve(trans, device):
    N, v, nrhs = 512, 32, 40

    def body(gv):
        rng = np.random.default_rng(5)
        gv.data[...] = rng.standard_normal((N, N))
        cb.LU_rep_rbt(gv, depth=2, seed=9)
        B = rng.standard_normal((N, nrhs))
        want, _, _ = cb.lu_rbt_solve(gv, B, trans=trans, refine=False)
        ncl = cb.rhs_local_cols(nrhs, v, 1)
        S = np.full((N, ncl), 7.0)
        S[:, :nrhs] = B
        if device:
            import torch
            S = torch.from_numpy(S).cuda()
        pre, post = (2, 3) if trans else (0, 1)
        cb.lu_rbt_apply_local(gv, pre, S, nrhs)
        X = cb.lu_solve_local(gv, S, nrhs, trans=trans, out=S)
        cb.lu_rbt_apply_local(gv, post, X, nrhs)
        X = X.cpu().numpy() if device else X
        assert np.array_equal(X[:, :nrhs], want)
        assert (X[:, nrhs:] == 7.0).all()                       # columns past nrhs are left as they are
    _one(N, v, body)


def test_repeated_calls_and_launch_count():
    N, v = 512, 64

    def body(gv):
        rng = np.random.default_rng(6)
        gv.data[...] = rng.standard_normal((N, N))
        B = rng.standard_normal((N, 3))
        C0, C1 = np.zeros((N, N)), np.zeros((N, N))
        cb.LU_rep_rbt(gv, seed=4, C=C0)
        X0 = cb.lu_rbt_solve(gv, B)
        _count(gv)
        X1 = cb.lu_rbt_solve(gv, B)
        assert _count(gv) == 0                                  # the solve launches nothing the count sees
        cb.LU_rep_rbt(gv, seed=4, C=C1)
        X2 = cb.lu_rbt_solve(gv, B)
        assert np.array_equal(C0, C1)
        for a, b in ((X0, X1), (X0, X2)):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    _one(N, v, body)


# ------------------------------------------------------------------------------------------------- state and arguments
def test_state_and_argument_rules():
    N, v = 256, 32

    def body(gv):
        L = cb._lib.lib()
        rbt = lambda depth=2, seed=0: L.cflx_lu_rbt(gv._h, depth, ctypes.c_uint64(seed), None, None)
        B = np.ones((N, 1))
        assert rbt() == -5                                      # nothing uploaded yet
        a = np.ascontiguousarray(gv.data)
        L.cflx_lu_set_local(gv._h, a.ctypes.data)
        assert rbt(0) == -1 and rbt(5) == -1
        assert rbt(4) == -4                                     # 2^4 * 32 > 256
        assert "512" in L.cflx_last_error().decode()            # the smallest order that works
        cb.LU_rep(gv, upload=False)
        with pytest.raises(cb.ConfluxError, match="status -5"):  # factors without a transform
            cb.lu_rbt_solve(gv, B)
        with pytest.raises(cb.ConfluxError, match="status -5"):
            cb.lu_rbt_apply_local(gv, 0, np.ones((N, v)), 1)
        assert rbt() == 0
        with pytest.raises(cb.ConfluxError, match="status -5"):  # the transform dropped the factors
            cb.lu_solve(gv, B)
        assert rbt() == -5                                      # already transformed
        with pytest.raises(cb.ConfluxError, match="status -5"):
            cb.lu_equilibrate(gv, apply=True, upload=False)
        cb.lu_equilibrate(gv, apply=False, upload=False)        # a query stays allowed
        cb.LU_rep_fixed(gv, perm=np.arange(N), upload=False)
        X = np.empty((N, 1))
        for args in [(2, 1, B, 1, X, 1, 1), (0, 1, B, 1, X, 1, 2), (0, 0, B, 1, X, 1, 1), (0, 1, None, 1, X, 1, 1)]:
            t, n, b, lb, x, lx, r = args
            assert L.cflx_lu_rbt_solve(gv._h, t, n, cb._ptr(b), lb, cb._ptr(x), lx, r, None, None) == -1
        for op in (-1, 4):
            assert L.cflx_lu_rbt_apply_local(gv._h, op, 1, np.ones((N, v)).ctypes.data, v) == -1
        assert L.cflx_lu_rbt_apply_local(gv._h, 0, 1, np.ones((N, v)).ctypes.data, v - 1) == -1
        cb.lu_rbt_solve(gv, B)
        L.cflx_lu_set_local(gv._h, a.ctypes.data)               # a new input: plain, and no factors
        with pytest.raises(cb.ConfluxError, match="status -5"):
            cb.lu_rbt_solve(gv, B, refine=False)
        scaled = a.copy()
        scaled[3] *= 1e-12
        L.cflx_lu_set_local(gv._h, scaled.ctypes.data)
        assert cb.lu_equilibrate(gv, apply=True, upload=False)["equed"] != "N"
        assert rbt() == -5                                      # a scaled input
    _one(N, v, body)


def test_queued_next_input_is_plain():
    N, v = 256, 32

    def body(gv):
        rng = np.random.default_rng(8)
        A, A2 = zero_leading_pivot(N, rng), zero_leading_pivot(N, rng)
        nxt = cb.pinned_empty((N, N))
        nxt[...] = A2
        gv.data[...] = A
        L = cb._lib.lib()
        L.cflx_lu_set_local(gv._h, np.ascontiguousarray(A).ctypes.data)
        assert L.cflx_lu_rbt(gv._h, 2, ctypes.c_uint64(1), None, None) == 0
        L.cflx_lu_queue_next_local(gv._h, nxt.ctypes.data)
        cb.LU_rep_fixed(gv, perm=np.arange(N), upload=False)
        B = rng.standard_normal((N, 2))
        X, _, _ = cb.lu_rbt_solve(gv, B, refine=False)          # the factors carry the transform
        assert _rel(X, np.linalg.solve(A, B)) <= 1e-10
        assert L.cflx_lu_rbt(gv._h, 2, ctypes.c_uint64(1), None, None) == 0   # the queued input arrived plain
        cb.LU_rep_fixed(gv, perm=np.arange(N), upload=False)
        X, _, _ = cb.lu_rbt_solve(gv, B)
        assert _rel(X, np.linalg.solve(A2, B)) <= 1e-10
        cb.pinned_free(nxt)
    _one(N, v, body)


# ------------------------------------------------------------------------------------------------------- multi-GPU
def test_multi_gpu_matches_one_gpu():
    grid = (2, 2, 1)
    P = 4
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 512, 32
    rng = np.random.default_rng(11)
    A = zero_leading_pivot(N, rng)
    B = rng.standard_normal((N, 5))
    shares = layout.scatter(A, v, *grid)

    def one(gv):
        gv.data[...] = A
        cb.LU_rep_rbt(gv, seed=3)
        return cb.lu_rbt_solve(gv, B)[0]
    X1 = _one(N, v, one)

    def body(comm):
        gv = cb.lu_params(N, N, v, *grid, comm)
        gv.data[...] = shares[gv.rank]
        _, _, info = cb.LU_rep_rbt(gv, seed=3)
        X = cb.lu_rbt_solve(gv, B)[0]
        bad = _rbt_refused(gv)
        gv.free_comms()
        return info, X, bad
    for info, X, bad in run_ranks(P, body):
        assert info == 0 and _rel(X, X1) <= 1e-12 and bad


def _rbt_refused(gv):
    """rank 1 passes another seed: every rank returns the error"""
    cb._lib.lib().cflx_lu_set_local(gv._h, np.ascontiguousarray(gv.data).ctypes.data)
    return cb._lib.lib().cflx_lu_rbt(gv._h, 2, ctypes.c_uint64(5 + (gv.rank == 1)), None, None) == -1
