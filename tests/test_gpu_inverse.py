"""GPU: cflx_lu_inverse and cflx_chol_inverse (the explicit inverse from the factors left on the device, by block solves with
the identity) against numpy / scipy on the device's own factors and against the schedule restatement
(oracle/inverse_ref.py); the per-share seed, scatter and zero kernels at grid positions a one-GPU run never reaches;
determinism, host and device output; the state and zero-pivot rules; and that nothing else changes.

Tolerances: ||A X - I||_F / (||A||_F ||X||_F + sqrt(M)) <= 1e-13 (the solve tests' bound with B = I), and X within
1e-10 max|X| of the host inverse from the same factors."""
import ctypes

import numpy as np
import pytest
import scipy.linalg

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, hp_ref, inverse_ref, layout, solve_ref
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
ETA_TOL = 1e-13
X_TOL = 1e-10


def _eta(A, X):
    M = A.shape[0]
    return float(np.linalg.norm(A @ X - np.eye(M)) / (np.linalg.norm(A) * np.linalg.norm(X) + np.sqrt(M)))


def _nc(M, v):
    """the library's block width: the whole number of tiles nearest 2048 columns, all of M when M is smaller"""
    return min(max(1, (2048 + v // 2) // v) * v, M)


# ----------------------------------------------------------------------------------------------- per-share kernels
def _hook_case(mode, perm, rng):
    v, Px, Py, pos, M = 8, 2, 3, (1, 2), 96
    Ml, Nl = (M // v // Px) * v, (M // v // Py) * v
    Kappa = 10 if mode == "chol" else M // v                         # the Cholesky's real tiles stop short of the share
    rows = Ml if mode == "lu" else inverse_ref.flt(Kappa, pos[0], Px) * v
    for c0, nc in [(0, 24), (16, 40), (56, 40), (88, 8)]:
        X = rng.standard_normal((M, nc))
        share = np.full((Ml, Nl), 7777.0)                            # a sentinel in every entry the scatter must not write
        W, out = cb.dbg.inverse_share(mode, v, (Px, Py), pos, M, c0, nc, Ml, Nl, Kappa=Kappa, rows=rows, X=X, perm=perm,
                                      share=share)
        assert np.array_equal(W, inverse_ref.seed_share(Ml, v, Px, pos[0], rows, c0, nc))
        want = inverse_ref.scatter_share(mode, X, c0, nc, perm, share.copy(), v, Px, Py, *pos, Kappa)
        assert np.array_equal(out, want)
        if mode == "chol":
            _, z = cb.dbg.inverse_share(mode, v, (Px, Py), pos, M, c0, nc, Ml, Nl, Kappa=Kappa, X=X, share=share,
                                        zero_fill=True)
            assert np.array_equal(z, inverse_ref.zero_share(want, v, Px, Py, *pos, Kappa))


def test_share_kernels_match_restatement():
    rng = np.random.default_rng(21)
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(96, 96, 8, 1, 1, 1, comm)
    gv.data[...] = rng.standard_normal((96, 96))
    perm = np.empty(96, dtype=np.int32)
    cb.LU_rep(gv, None, perm)                                        # a permutation from a real factorisation
    assert not np.array_equal(perm, np.arange(96))
    gv.free_comms()
    comm.close()
    _hook_case("lu", perm, rng)
    _hook_case("chol", None, rng)


# ----------------------------------------------------------------------------------------------- LU
def _lu_run(A, v):
    """factor A on one GPU; returns dict(C, perm, inv = lu_inverse's result, and the handles)"""
    N = A.shape[0]
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    gv.data[...] = A
    C = np.zeros((gv.Ml, gv.Nl))
    perm = np.empty(gv.M, dtype=np.int32)
    cb.LU_rep(gv, C, perm)
    res = dict(C=C, perm=perm, gv=gv, comm=comm)
    res["inv"] = cb.lu_inverse(gv)
    return res


def _close(res):
    res["gv"].free_comms()
    res["comm"].close()


LU_SIZES = [(16, 4), (96, 16), (100, 16), (512, 64), (1024, 128), (4096, 256), (5120, 256)]


@pytest.mark.parametrize("N,v", LU_SIZES)
def test_lu_inverse(N, v):
    M = layout.dims(N, v, 1, 1, 1)["M"]
    if (N, v) == (5120, 256):
        nc = _nc(M, v)
        assert -(-M // nc) >= 3 and M % nc                           # three blocks or more, the last one narrower
    A = np.random.default_rng(N + v).standard_normal((M, M))
    r = _lu_run(A, v)
    X, info = r["inv"]
    assert info == 0 and X.shape == (M, M) and np.all(np.isfinite(X))
    assert _eta(A, X) <= ETA_TOL
    Xh = solve_ref.host_solve(r["C"], r["perm"], np.eye(M))
    assert np.abs(X - Xh).max() <= X_TOL * np.abs(X).max()
    _close(r)


def test_lu_inverse_matches_restatement():
    N, v = 100, 16
    M = layout.dims(N, v, 1, 1, 1)["M"]
    A = np.random.default_rng(5).standard_normal((M, M))
    r = _lu_run(A, v)
    X, _ = r["inv"]
    Xo = inverse_ref.lu_inverse([r["C"]], r["perm"], N, v, nc=_nc(M, v))[0]
    assert np.abs(X - Xo).max() <= X_TOL * np.abs(X).max()
    _close(r)


def test_lu_zero_pivot_and_state_rules():
    n, v = 64, 16
    rng = np.random.default_rng(12)
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    out = np.full((n, n), 3.0)
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_inverse(gv, out)                                       # no factorisation yet
    A = np.triu(rng.integers(1, 9, (n, n)).astype(float)) + np.diag(np.full(n, 50.0))
    A[20, 20] = 0.0                                                  # partial pivoting keeps every row: U(21, 21) = 0
    gv.data[...] = A
    cb.LU_rep(gv)
    X, info = cb.lu_inverse(gv, out)
    assert X is None and info == 21 and np.all(out == 3.0)           # nothing written
    A[20, 20] = 5.0
    gv.data[...] = A
    cb.LU_rep(gv)
    X, info = cb.lu_inverse(gv, out)
    assert info == 0 and X is out and _eta(A, X) <= ETA_TOL
    a = np.ascontiguousarray(gv.data)
    cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_inverse(gv)                                            # new input, not factored yet
    assert cb.lib().cflx_lu_inverse(gv._h, None, None) == -1         # NULL info_out
    with pytest.raises(ValueError):
        cb.lu_inverse(gv, np.zeros((n, n + 1)))
    with pytest.raises(ValueError):
        cb.lu_inverse(gv, np.zeros((n, n), dtype=np.float32))
    with pytest.raises(ValueError):
        cb.lu_inverse(gv, np.zeros((n, 2 * n))[:, ::2])
    gv.free_comms()
    comm.close()


def _launches(fn, h):
    n = ctypes.c_int64()
    cb.check(fn(h, ctypes.byref(n), 1), "launch_count")
    return n.value


def test_lu_no_side_effects_deterministic_and_device_output():
    import torch
    N, v = 2048, 256
    rng = np.random.default_rng(9)
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    C0 = np.zeros((gv.Ml, gv.Nl))
    perm0 = np.empty(gv.M, dtype=np.int32)
    cb.LU_rep(gv, C0, perm0)
    B = rng.standard_normal((gv.M, 5))
    x0 = cb.lu_solve(gv, B)
    _launches(cb.lib().cflx_lu_launch_count, gv._h)
    X1, _ = cb.lu_inverse(gv)
    X2, _ = cb.lu_inverse(gv)
    assert np.array_equal(X1, X2)                                    # two calls, the same bits
    t = torch.full((gv.Ml, gv.Nl), float("nan"), dtype=torch.float64, device="cuda")
    Xt, info = cb.lu_inverse(gv, t)
    assert info == 0 and Xt is t
    assert np.array_equal(t.cpu().numpy(), X1)                       # device output: the bits of host output
    assert _launches(cb.lib().cflx_lu_launch_count, gv._h) == 0
    assert np.array_equal(cb.lu_solve(gv, B), x0)                    # a later solve: the same bits
    C1 = np.zeros_like(C0)
    perm1 = np.empty_like(perm0)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C1.ctypes.data, perm1.ctypes.data), "get_factors")
    assert np.array_equal(C1, C0) and np.array_equal(perm1, perm0)
    gv.free_comms()
    comm.close()


# ----------------------------------------------------------------------------------------------- Cholesky
def _chol_check(N, v, grid, X_shares, L_shares, S):
    d = chol_ref.dims(N, v, *grid)
    K = d["Kappa"]
    X = chol_ref.assemble(X_shares, N, v, *grid)
    L = np.tril(chol_ref.assemble(L_shares, N, v, *grid))
    tr = np.arange(X.shape[0]) // v
    low = (tr[:, None] >= tr[None, :]) & (tr[:, None] < K) & (tr[None, :] < K)
    inv, info = scipy.linalg.lapack.dpotri(L, lower=1)
    assert info == 0
    inv = np.tril(inv) + np.tril(inv, -1).T
    scale = np.abs(X).max()
    assert np.abs(np.where(low, X - inv, 0.0)).max() <= X_TOL * scale
    assert np.all(X[~low] == 0.0)
    Xs = np.tril(X) + np.tril(X, -1).T                               # the symmetric completion
    assert _eta(S, Xs) <= ETA_TOL


CHOL_SIZES = [(16, 4), (96, 16), (100, 16), (512, 64), (1024, 128), (2048, 512), (4096, 256), (5120, 512)]


@pytest.mark.parametrize("N,v", CHOL_SIZES)
def test_chol_inverse(N, v):
    Np = chol_ref.dims(N, v, 1, 1, 1)["N"]
    if (N, v) == (5120, 512):
        nc = _nc(Np, v)
        assert -(-Np // nc) >= 3 and Np % nc
    S = hp_ref.random_spd(Np, 1e3, np.random.default_rng(N + v))
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    ch.data[...] = S
    ch.parallelCholesky()
    X = ch.inverse()
    _chol_check(N, v, (1, 1, 1), [X], [ch.local_factor()], S)
    if (N, v) == (100, 16):
        Xo = inverse_ref.chol_inverse([ch.local_factor()], N, v, nc=_nc(Np, v))[0]
        assert np.abs(X - Xo).max() <= X_TOL * np.abs(X).max()
    ch.finalize()
    comm.close()


def test_chol_state_rules_side_effects_and_device_output():
    import torch
    N, v = 1024, 128
    rng = np.random.default_rng(1)
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.inverse()                                                 # no factorisation yet
    S = hp_ref.random_spd(N, 1e2, rng)
    ch.data[...] = S
    ch.parallelCholesky()
    L0 = ch.local_factor()
    B = rng.standard_normal((N, 3))
    x0 = ch.solve(B)
    n0 = _launches(cb.lib().cflx_chol_launch_count, ch._h)
    X1 = ch.inverse()
    out = np.full((N, N), 9.0)
    assert ch.inverse(out) is out and np.array_equal(out, X1)        # two calls, the same bits
    t = torch.full((N, N), float("nan"), dtype=torch.float64, device="cuda")
    assert ch.inverse(t) is t and np.array_equal(t.cpu().numpy(), X1)
    assert _launches(cb.lib().cflx_chol_launch_count, ch._h) == 0 and n0 > 0
    assert np.array_equal(ch.solve(B), x0) and np.array_equal(ch.local_factor(), L0)
    with pytest.raises(ValueError):
        ch.inverse(np.zeros((N, N - 1)))
    a = np.ascontiguousarray(ch.data)
    cb.check(cb.lib().cflx_chol_set_local(ch._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.inverse()                                                 # new input, not factored yet
    bad = S.copy()
    bad[N // 2, N // 2] = -1.0
    ch.data = bad
    with pytest.raises(cb.ConfluxError, match="positive definite"):
        ch.parallelCholesky()
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.inverse()                                                 # the factorisation failed
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- multi-GPU
@pytest.mark.parametrize("grid", [(1, 1, 2), (2, 2, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_lu_inverse(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1024, 64
    M = layout.dims(N, v, *grid)["M"]
    A = np.random.default_rng(P).standard_normal((M, M))
    locs = layout.scatter(A, v, *grid)

    def body(comm):
        gv = cb.lu_params(N, N, v, *grid, comm)
        gv.data[...] = locs[gv.rank]
        cb.LU_rep(gv)
        X, info = cb.lu_inverse(gv)
        gv.free_comms()
        return X, info

    rs = run_ranks(P, body)
    assert all(info == 0 for _, info in rs)
    for r, (X, _) in enumerate(rs):
        assert np.array_equal(X, rs[r - r % grid[2]][0])             # the layers agree bit for bit
    X = layout.assemble([x for x, _ in rs], N, v, *grid)
    X1 = _lu_run(A, v)
    assert np.abs(X - X1["inv"][0]).max() <= X_TOL * np.abs(X).max()
    assert _eta(A, X) <= ETA_TOL
    _close(X1)


@pytest.mark.parametrize("grid", [(1, 1, 2), (2, 2, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_chol_inverse(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1000, 48
    Np = chol_ref.dims(N, v, *grid)["N"]
    S = hp_ref.random_spd(Np, 1e2, np.random.default_rng(P))
    locs = chol_solve_ref.scatter(S, N, v, *grid)

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        res = ch.inverse(), ch.local_factor()
        ch.finalize()
        return res

    rs = run_ranks(P, body)
    for r, (X, _) in enumerate(rs):
        assert np.array_equal(X, rs[r - r % grid[2]][0])
    _chol_check(N, v, grid, [x for x, _ in rs], [l for _, l in rs], S)
