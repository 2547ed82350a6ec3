"""GPU: cflx_lu_solve_local and cflx_chol_solve_local (A X = B with B and X distributed like A, solved block by block on
the device).  Each block of columns equals, bit for bit, cflx_lu_solve / cflx_lu_solve_trans / cflx_chol_solve called on
those columns alone; the pack and scatter kernels match the restatement (oracle/solve_local_ref.py) at a grid position a
one-GPU run never reaches; host, device and in-place shares give the same bits and write nothing they must not; calls
repeat bit for bit and change nothing else; and the argument and state rules hold.

Tolerance: ||B - A X||_F / (||A||_F ||X||_F + ||B||_F) <= 1e-13, the solve tests' bound."""
import ctypes

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, hp_ref, layout, solve_local_ref, solve_ref
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
ETA_TOL = 1e-13
SENTINEL = -7777.0
ERR_ARG, ERR_STATE = -1, -5


def _ptr(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _blocks(M, v, nrhs):
    nc = solve_local_ref.block_cols(M, v)
    return [(c0, min(nc, nrhs - c0)) for c0 in range(0, nrhs, nc)]


def _launches(fn, h):
    n = ctypes.c_int64()
    cb.check(fn(h, ctypes.byref(n), 1), "launch_count")
    return n.value


# ----------------------------------------------------------------------------------------------- per-share kernels
def test_share_kernels_match_restatement():
    v, Px, Py, pos, M, nrhs = 8, 2, 3, (1, 2), 96, 150
    rng = np.random.default_rng(21)
    for kind, Kappa in (("lu", None), ("chol", 10)):                 # the Cholesky's real tiles stop short of the share
        Ml = M // v // Px * v
        ncl = cb.rhs_local_cols(nrhs, v, Py)
        B = rng.standard_normal((Ml, ncl + 3))
        for c0, w in [(0, 1), (0, 24), (13, 40), (56, 94), (149, 1)]:
            Xk = rng.standard_normal((M, -(-w // 8) * 8))
            X = np.full((Ml, ncl + 5), SENTINEL)                     # a sentinel in every entry the scatter must not write
            Bk, Xo = cb.dbg.solve_local_share(kind, v, (Px, Py), pos, M, nrhs, c0, w, Ml, Kappa=Kappa, B=B, Xk=Xk, X=X)
            assert np.array_equal(Bk, solve_local_ref.pack_share(kind, B, M, v, Px, Py, *pos, nrhs, c0, w, Kappa))
            want = solve_local_ref.scatter_share(kind, Xk, X.copy(), v, Px, Py, *pos, nrhs, c0, w, Kappa)
            assert np.array_equal(Xo, want)


# ----------------------------------------------------------------------------------------------- one GPU, bit equality
def _lu(N, v, seed):
    M = layout.dims(N, v, 1, 1, 1)["M"]
    A = np.random.default_rng(seed).standard_normal((M, M))
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    gv.data[...] = A
    cb.LU_rep(gv)
    return gv, comm, A


def _solve_alone(fn, h, G, c0, w):
    """fn (cflx_lu_solve, _solve_trans or cflx_chol_solve) on columns [c0, c0 + w) of G alone"""
    b = np.ascontiguousarray(G[:, c0:c0 + w])
    x = np.empty_like(b)
    cb.check(fn(h, w, _ptr(b), w, _ptr(x), w), "solve")
    return x


LU_SIZES = [(16, 4), (96, 16), (100, 16), (512, 64), (1024, 128), (4096, 256), (5120, 256)]


@pytest.mark.parametrize("trans", [False, True], ids=["N", "T"])
@pytest.mark.parametrize("N,v", LU_SIZES)
def test_lu_blocks_equal_solve_bits(N, v, trans):
    gv, comm, A = _lu(N, v, N + v)
    M = gv.M
    nrhs = M if (N, v) == (5120, 256) else M + 5                       # two or three blocks, the last one narrower
    blocks = _blocks(M, v, nrhs)
    assert len(blocks) >= 2 and blocks[-1][1] < blocks[0][1]
    G = np.random.default_rng(v).standard_normal((M, nrhs))
    B = solve_local_ref.distribute("lu", G, v)[0]
    X = cb.lu_solve_local(gv, B, nrhs, trans=trans)
    fn = cb.lib().cflx_lu_solve_trans if trans else cb.lib().cflx_lu_solve
    for c0, w in blocks:
        assert np.array_equal(X[:, c0:c0 + w], _solve_alone(fn, gv._h, G, c0, w))
    assert solve_ref.backward_error(A.T if trans else A, X[:, :nrhs], G) <= ETA_TOL
    gv.free_comms()
    comm.close()


CHOL_SIZES = [(16, 4), (100, 16), (1024, 128), (5120, 512)]


@pytest.mark.parametrize("N,v", CHOL_SIZES)
def test_chol_blocks_equal_solve_bits(N, v):
    d = chol_ref.dims(N, v, 1, 1, 1)
    M = d["N"]
    S = hp_ref.random_spd(M, 1e3, np.random.default_rng(N + v))
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    ch.data[...] = S
    ch.parallelCholesky()
    nrhs = M if (N, v) == (5120, 512) else M + 5
    assert len(_blocks(M, v, nrhs)) >= 2
    G = np.random.default_rng(v).standard_normal((M, nrhs))
    B = solve_local_ref.distribute("chol", G, v, Kappa=d["Kappa"])[0]
    X = ch.solve_local(B, nrhs)
    for c0, w in _blocks(M, v, nrhs):
        assert np.array_equal(X[:, c0:c0 + w], _solve_alone(cb.lib().cflx_chol_solve, ch._h, G, c0, w))
    assert solve_ref.backward_error(S, X[:, :nrhs], G) <= ETA_TOL
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- memory kinds
def test_lu_memory_kinds_in_place_and_side_effects():
    import torch
    N, v = 1024, 128
    gv, comm, A = _lu(N, v, 3)
    nrhs = 2 * v + 3                                                   # padding columns in the last local tile
    ncl = cb.rhs_local_cols(nrhs, v, 1)
    G = np.random.default_rng(4).standard_normal((gv.M, nrhs))
    B = solve_local_ref.distribute("lu", G, v, pad=np.nan, ld_extra=5)[0]  # NaN in the padding and the ld padding
    B0 = B.copy()
    C0 = np.zeros((gv.Ml, gv.Nl))
    perm0 = np.empty(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C0.ctypes.data, perm0.ctypes.data), "get_factors")
    b1 = G[:, :7].copy()
    x0 = cb.lu_solve(gv, b1)
    _launches(cb.lib().cflx_lu_launch_count, gv._h)

    X1 = cb.lu_solve_local(gv, B, nrhs, out=np.full_like(B, SENTINEL))  # host in, host out
    assert np.array_equal(B, B0, equal_nan=True)                       # B unchanged
    assert np.all(X1[:, nrhs:] == SENTINEL) and np.all(np.isfinite(X1[:, :nrhs]))
    X2 = cb.lu_solve_local(gv, B, nrhs, out=np.full_like(B, SENTINEL))
    assert np.array_equal(X1, X2)                                      # two calls, the same bits
    for trans in (False, True):
        Xh = cb.lu_solve_local(gv, B, nrhs, trans=trans, out=np.full_like(B, SENTINEL))
        tb = torch.from_numpy(B).cuda()
        tx = torch.full(B.shape, SENTINEL, dtype=torch.float64, device="cuda")
        assert cb.lu_solve_local(gv, tb, nrhs, trans=trans, out=tx) is tx  # device in, device out
        assert np.array_equal(tx.cpu().numpy(), Xh)
        assert np.array_equal(tb.cpu().numpy(), B0, equal_nan=True)
        assert cb.lu_solve_local(gv, tb, nrhs, trans=trans, out=tb) is tb  # in place on the device
        assert np.array_equal(tb.cpu().numpy()[:, :nrhs], Xh[:, :nrhs])
        assert np.all(np.isnan(tb.cpu().numpy()[:, nrhs:]))
        Bi = B.copy()
        assert cb.lu_solve_local(gv, Bi, nrhs, trans=trans, out=Bi) is Bi  # in place on the host
        assert np.array_equal(Bi[:, :nrhs], Xh[:, :nrhs]) and np.all(np.isnan(Bi[:, nrhs:]))
        Xm = cb.lu_solve_local(gv, tb.new_tensor(B), nrhs, trans=trans, out=np.full_like(B, SENTINEL))  # device in, host out
        assert np.array_equal(Xm, Xh)
        tx.fill_(SENTINEL)
        cb.lu_solve_local(gv, B, nrhs, trans=trans, out=tx)           # host in, device out
        assert np.array_equal(tx.cpu().numpy(), Xh)
    tw = torch.full((gv.M, ncl + 16), SENTINEL, dtype=torch.float64, device="cuda")
    cb.lu_solve_local(gv, B, nrhs, out=tw[:, :ncl + 2])                # a strided device share: ld = ncl + 16
    assert np.array_equal(tw.cpu().numpy()[:, :nrhs], X1[:, :nrhs])
    assert np.all(tw.cpu().numpy()[:, nrhs:] == SENTINEL)

    assert _launches(cb.lib().cflx_lu_launch_count, gv._h) == 0
    assert np.array_equal(cb.lu_solve(gv, b1), x0)                    # a later solve: the same bits
    C1 = np.zeros_like(C0)
    perm1 = np.empty_like(perm0)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C1.ctypes.data, perm1.ctypes.data), "get_factors")
    assert np.array_equal(C1, C0) and np.array_equal(perm1, perm0)
    gv.free_comms()
    comm.close()


def test_chol_memory_kinds_in_place_and_side_effects():
    import torch
    N, v = 1000, 48                                                    # Kappa = 21 tiles
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    S = hp_ref.random_spd(ch.N, 1e2, np.random.default_rng(2))
    ch.data[...] = S
    ch.parallelCholesky()
    L0 = ch.local_factor()
    nrhs = 3 * v + 1
    G = np.random.default_rng(5).standard_normal((ch.N, nrhs))
    B = solve_local_ref.distribute("chol", G, v, Kappa=ch.Kappa, ld_extra=3)[0]
    b1 = G[:, :3].copy()
    x0 = ch.solve(b1)
    n0 = _launches(cb.lib().cflx_chol_launch_count, ch._h)
    Xh = ch.solve_local(B, nrhs, out=np.full_like(B, SENTINEL))
    assert np.all(Xh[:, nrhs:] == SENTINEL) and np.all(np.isfinite(Xh[:, :nrhs]))
    Xn = ch.solve_local(B, nrhs)                                       # a new array: two calls, the same bits
    assert Xn.shape == (ch.Ml, cb.rhs_local_cols(nrhs, v, 1)) and np.array_equal(Xn[:, :nrhs], Xh[:, :nrhs])
    tb = torch.from_numpy(B).cuda()
    tx = torch.full(B.shape, SENTINEL, dtype=torch.float64, device="cuda")
    assert ch.solve_local(tb, nrhs, out=tx) is tx and np.array_equal(tx.cpu().numpy(), Xh)
    assert ch.solve_local(tb, nrhs, out=tb) is tb
    assert np.array_equal(tb.cpu().numpy()[:, :nrhs], Xh[:, :nrhs]) and np.all(np.isnan(tb.cpu().numpy()[:, nrhs:]))
    Bi = B.copy()
    ch.solve_local(Bi, nrhs, out=Bi)
    assert np.array_equal(Bi[:, :nrhs], Xh[:, :nrhs])
    assert _launches(cb.lib().cflx_chol_launch_count, ch._h) == 0 and n0 > 0
    assert np.array_equal(ch.solve(b1), x0) and np.array_equal(ch.local_factor(), L0)
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- rules
def test_argument_and_state_rules():
    import torch
    n, v = 64, 16
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    nrhs = 20
    ncl = cb.rhs_local_cols(nrhs, v, 1)
    B = np.ones((n, ncl))
    X = np.zeros((n, ncl))
    f = cb.lib().cflx_lu_solve_local
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_solve_local(gv, B, nrhs)                                 # no factorisation yet
    gv.data[...] = np.random.default_rng(1).standard_normal((n, n))
    cb.LU_rep(gv)
    assert f(gv._h, 2, nrhs, _ptr(B), ncl, _ptr(X), ncl) == ERR_ARG    # trans not 0 / 1
    assert f(gv._h, -1, nrhs, _ptr(B), ncl, _ptr(X), ncl) == ERR_ARG
    assert f(gv._h, 0, 0, _ptr(B), ncl, _ptr(X), ncl) == ERR_ARG       # nrhs < 1
    assert f(gv._h, 0, nrhs, _ptr(B), ncl - 1, _ptr(X), ncl) == ERR_ARG  # ldb below the local column count
    assert f(gv._h, 0, nrhs, _ptr(B), ncl, _ptr(X), ncl - 1) == ERR_ARG  # ldx below it
    assert f(gv._h, 0, nrhs, None, ncl, _ptr(X), ncl) == ERR_ARG      # NULL B on layer 0
    Bw = np.ones((n, ncl + 8))
    assert f(gv._h, 0, nrhs, _ptr(Bw), ncl + 8, _ptr(Bw), ncl) == ERR_ARG  # in place with ldx != ldb
    assert f(gv._h, 1, nrhs, _ptr(B), ncl, None, ncl) == 0            # X may be NULL
    with pytest.raises(ValueError):
        cb.lu_solve_local(gv, np.ones((n, ncl - 1)), nrhs)
    with pytest.raises(ValueError):
        cb.lu_solve_local(gv, B.astype(np.float32), nrhs)
    with pytest.raises(ValueError):
        cb.lu_solve_local(gv, np.ones((n, 2 * ncl))[:, ::2], nrhs)
    if n_gpus() >= 2:                                                  # device memory on another device
        t1 = torch.ones((n, ncl), dtype=torch.float64, device="cuda:1")
        assert f(gv._h, 0, nrhs, ctypes.c_void_p(t1.data_ptr()), ncl, _ptr(X), ncl) == ERR_ARG
        assert f(gv._h, 0, nrhs, _ptr(B), ncl, ctypes.c_void_p(t1.data_ptr()), ncl) == ERR_ARG
    a = np.ascontiguousarray(gv.data)
    cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_solve_local(gv, B, nrhs)                                 # new input, not factored yet
    gv.free_comms()

    N, v = 256, 32
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    ncl = cb.rhs_local_cols(nrhs, v, 1)
    B, X = np.ones((N, ncl)), np.zeros((N, ncl))
    g = cb.lib().cflx_chol_solve_local
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.solve_local(B, nrhs)                                        # no factorisation yet
    S = hp_ref.random_spd(N, 1e2, np.random.default_rng(3))
    ch.data[...] = S
    ch.parallelCholesky()
    assert g(ch._h, 0, _ptr(B), ncl, _ptr(X), ncl) == ERR_ARG
    assert g(ch._h, nrhs, _ptr(B), ncl - 1, _ptr(X), ncl) == ERR_ARG
    assert g(ch._h, nrhs, _ptr(B), ncl, _ptr(X), ncl - 1) == ERR_ARG
    assert g(ch._h, nrhs, None, ncl, _ptr(X), ncl) == ERR_ARG
    assert g(ch._h, nrhs, _ptr(B), ncl, _ptr(X), ncl) == 0
    a = np.ascontiguousarray(ch.data)
    cb.check(cb.lib().cflx_chol_set_local(ch._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.solve_local(B, nrhs)                                        # new input, not factored yet
    bad = S.copy()
    bad[N // 2, N // 2] = -1.0
    ch.data = bad
    with pytest.raises(cb.ConfluxError, match="positive definite"):
        ch.parallelCholesky()
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.solve_local(B, nrhs)                                        # the factorisation failed
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- multi-GPU
@pytest.mark.parametrize("grid", [(1, 1, 2), (2, 2, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_lu_solve_local(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1024, 64
    M = layout.dims(N, v, *grid)["M"]
    A = np.random.default_rng(P).standard_normal((M, M))
    locs = layout.scatter(A, v, *grid)
    nrhs = M + 70
    G = np.random.default_rng(P + 1).standard_normal((M, nrhs))
    Bs = solve_local_ref.distribute("lu", G, v, *grid)
    blocks = _blocks(M, v, nrhs)

    def body(comm):
        gv = cb.lu_params(N, N, v, *grid, comm)
        gv.data[...] = locs[gv.rank]
        cb.LU_rep(gv)
        out = {}
        for trans in (False, True):
            B = Bs[gv.rank] if gv.pk == 0 else None                    # not read off layer 0
            X = cb.lu_solve_local(gv, B, nrhs, trans=trans, out=np.full_like(Bs[gv.rank], SENTINEL))
            fn = cb.lib().cflx_lu_solve_trans if trans else cb.lib().cflx_lu_solve
            out[trans] = X, [_solve_alone(fn, gv._h, G, c0, w) for c0, w in blocks]
        gv.free_comms()
        return out

    rs = run_ranks(P, body)
    for trans in (False, True):
        for r in range(P):
            assert np.array_equal(rs[r][trans][0], rs[r - r % grid[2]][trans][0])  # the layers agree bit for bit
        X = solve_local_ref.collect("lu", [x[trans][0] for x in rs], M, nrhs, v, *grid)
        for (c0, w), xb in zip(blocks, rs[0][trans][1]):
            assert np.array_equal(X[:, c0:c0 + w], xb)
        assert solve_ref.backward_error(A.T if trans else A, X, G) <= ETA_TOL


@pytest.mark.parametrize("grid", [(2, 1, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_chol_solve_local(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1000, 48
    d = chol_ref.dims(N, v, *grid)
    S = hp_ref.random_spd(d["N"], 1e2, np.random.default_rng(P))
    locs = chol_solve_ref.scatter(S, N, v, *grid)
    nrhs = d["N"] + 9
    G = np.random.default_rng(P + 1).standard_normal((d["N"], nrhs))
    Bs = solve_local_ref.distribute("chol", G, v, *grid, Kappa=d["Kappa"])
    blocks = _blocks(d["N"], v, nrhs)

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        X = ch.solve_local(Bs[ch.rank], nrhs, out=np.full_like(Bs[ch.rank], SENTINEL))
        alone = [_solve_alone(cb.lib().cflx_chol_solve, ch._h, G, c0, w) for c0, w in blocks]
        ch.finalize()
        return X, alone

    rs = run_ranks(P, body)
    for r in range(P):
        assert np.array_equal(rs[r][0], rs[r - r % grid[2]][0])
    X = solve_local_ref.collect("chol", [x for x, _ in rs], d["N"], nrhs, v, *grid, Kappa=d["Kappa"])
    for (c0, w), xb in zip(blocks, rs[0][1]):
        assert np.array_equal(X[:, c0:c0 + w], xb)
    assert solve_ref.backward_error(S, X, G) <= ETA_TOL
