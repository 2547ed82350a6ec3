"""GPU: cflx_lu_solve (A X = B with the factors left on the device) and its narrow GEMM, against numpy, the host
triangular solves on the gathered factors and the schedule restatement (oracle/solve_ref.py); its state rules; and that
it leaves the factorisation untouched; and that X is bit for bit the one pinned in tests/golden/solve_bits.json."""
import json
import os

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import layout, solve_ref
from tests._harness import n_gpus, run_ranks
from tests.golden import make_solve_golden

pytestmark = pytest.mark.gpu
ETA_TOL = 1e-13           # normwise backward error ||B - A X||_F / (||A||_F ||X||_F + ||B||_F)
X_TOL = 1e-10             # against the host solve / the restatement, relative to max|X|
GRIDS = [(64, 8, 2, 2, 1), (128, 16, 1, 1, 2), (128, 8, 2, 2, 2), (512, 32, 2, 2, 1), (512, 64, 2, 2, 2),
         (1024, 128, 1, 1, 2)]


@pytest.mark.parametrize("M,N,K", [(1, 1, 4), (37, 3, 8), (1000, 1, 256), (4097, 64, 256), (513, 65, 128),
                                   (16128, 200, 512)])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-1.0, 1.0)])
def test_gemm_narrow_matches_numpy(M, N, K, alpha, beta):
    rng = np.random.default_rng(M + N + K)
    A = rng.standard_normal((M, K))
    B = rng.standard_normal((K, N))
    C = rng.standard_normal((M, N))
    want = beta * C + alpha * (A @ B)
    tol = 1e-13 * K * np.abs(A).max() * np.abs(B).max()
    D, ms = cb.dbg.gemm_narrow(A, B, C, alpha, beta)
    assert ms > 0 and np.abs(D - want).max() <= tol
    Ca = C.copy()
    D2, _ = cb.dbg.gemm_narrow(A, B, Ca, alpha, beta, out=Ca)           # D aliasing C on the device
    assert D2 is Ca and np.abs(Ca - want).max() <= tol


def test_gemm_narrow_refuses_k_not_multiple_of_4():
    with pytest.raises(cb.ConfluxError):
        cb.dbg.gemm_narrow(np.ones((8, 6)), np.ones((6, 8)))


def _solve_on_grid(N, v, Px, Py, Pz, Bs, A_locals=None, want_C=True):
    """Factor once, then solve every B in Bs (M x nrhs or (M,)); returns per-rank A, C, perm and the X of every B."""
    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        if A_locals is not None:
            gv.data[...] = np.asarray(A_locals[gv.rank]).reshape(gv.Ml, gv.Nl)
        C = np.zeros((gv.Ml, gv.Nl)) if want_C else None
        perm = np.zeros(gv.M, dtype=np.int32)
        cb.LU_rep(gv, C, perm)
        Xs = [cb.lu_solve(gv, B) for B in Bs]
        res = dict(A=gv.data.copy() if want_C else None, C=C, perm=perm, X=Xs)
        gv.free_comms()
        return res

    rs = run_ranks(Px * Py * Pz, body)
    return dict(A=[r["A"] for r in rs], C=[r["C"] for r in rs], perm=rs[0]["perm"], X=[r["X"] for r in rs])


def _check(g, N, v, Px, Py, Pz, Bs, restated=True):
    A = layout.assemble(g["A"], N, v, Px, Py, Pz)
    LU = layout.assemble(g["C"], N, v, Px, Py, Pz)
    for i, B in enumerate(Bs):
        X = g["X"][0][i]
        for Xr in g["X"]:
            assert np.array_equal(Xr[i], X)                              # bit-identical on every rank
        assert X.shape == B.shape
        X2, B2 = X.reshape(len(B), -1), B.reshape(len(B), -1)
        assert solve_ref.backward_error(A, X2, B2) <= ETA_TOL
        scale = np.abs(X).max()
        assert np.abs(X2 - solve_ref.host_solve(LU, g["perm"], B2)).max() <= X_TOL * scale
        if restated:
            Xo = solve_ref.solve(g["C"], g["perm"], B, N, v, Px, Py, Pz)
            assert np.abs(X - Xo).max() <= X_TOL * scale


@pytest.mark.parametrize("N,v", [(16, 4), (96, 16), (512, 64), (1024, 128), (4096, 256), (100, 16)])
def test_single_gpu_solve(N, v):
    M = layout.dims(N, v, 1, 1, 1)["M"]
    rng = np.random.default_rng(N)
    Bs = [rng.standard_normal((M, nrhs)) for nrhs in (1, 3, 64, 130)] + [rng.standard_normal(M)]
    g = _solve_on_grid(N, v, 1, 1, 1, Bs)
    _check(g, N, v, 1, 1, 1, Bs)


def test_single_gpu_solve_standard_normal_matrix():
    N, v = 1024, 128
    A = np.random.default_rng(3).standard_normal((N, N))
    Bs = [np.random.default_rng(4).standard_normal((N, 5))]
    g = _solve_on_grid(N, v, 1, 1, 1, Bs, A_locals=[A])
    _check(g, N, v, 1, 1, 1, Bs)


def test_state_rules():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(256, 256, 32, 1, 1, 1, comm)
    B = np.random.default_rng(1).standard_normal((gv.M, 2))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_solve(gv, B)                                              # no factorisation yet
    cb.LU_rep(gv)
    X = cb.lu_solve(gv, B)
    assert solve_ref.backward_error(gv.data, X, B) <= ETA_TOL
    with pytest.raises(cb.ConfluxError, match="status -1"):
        cb.lu_solve(gv, np.zeros((gv.M, 0)))                            # nrhs < 1
    B2 = np.random.default_rng(2).standard_normal(gv.M)
    x2 = cb.lu_solve(gv, B2)                                            # a second B after the same factorisation
    assert solve_ref.backward_error(gv.data, x2[:, None], B2[:, None]) <= ETA_TOL
    a = np.ascontiguousarray(gv.data)
    cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_solve(gv, B)                                              # new input, not factored yet
    gv.data = np.random.default_rng(9).standard_normal((gv.Ml, gv.Nl))
    cb.LU_rep(gv)                                                       # a different matrix: the cache must follow
    X3 = cb.lu_solve(gv, B)
    assert solve_ref.backward_error(gv.data, X3, B) <= ETA_TOL
    assert not np.allclose(X3, X)
    gv.free_comms()
    comm.close()


def test_streamed_run_can_be_solved():
    """A run whose input buffer was handed to the next matrix (next_data) still has its factors: it can be solved."""
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(512, 512, 64, 1, 1, 1, comm)
    rng = np.random.default_rng(21)
    mats = [cb.pinned_empty((gv.Ml, gv.Nl)) for _ in range(2)]
    for m in mats:
        m[...] = rng.standard_normal((gv.Ml, gv.Nl))
    B = rng.standard_normal((gv.M, 3))
    gv.data = mats[0]
    cb.LU_rep(gv, next_data=mats[1])
    with pytest.raises(cb.ConfluxError):
        cb.residual(gv)
    X0 = cb.lu_solve(gv, B)
    assert solve_ref.backward_error(mats[0], X0, B) <= ETA_TOL
    cb.LU_rep(gv, upload=False)                                         # factors the streamed matrix
    X1 = cb.lu_solve(gv, B)
    assert solve_ref.backward_error(mats[1], X1, B) <= ETA_TOL
    for m in mats:
        cb.pinned_free(m)
    gv.free_comms()
    comm.close()


def test_no_side_effects_on_factors_and_validation():
    N, v = 1024, 128

    def run(solve):
        comm = cb.Comm(1, 0, None, 0)
        gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
        cb.LU_rep(gv)
        if solve:
            cb.lu_solve(gv, np.random.default_rng(0).standard_normal((gv.M, 7)))
        C, perm = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
        cb.check(cb.lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "get_factors")
        resid = cb.validate(gv)
        C2, perm2 = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
        cb.LU_rep(gv, C2, perm2)                                        # a second factorisation after the solve
        gv.free_comms()
        comm.close()
        return C, perm, resid, C2, perm2

    C0, p0, r0, _, _ = run(False)
    C1, p1, r1, C2, p2 = run(True)
    assert np.array_equal(C0, C1) and np.array_equal(p0, p1) and r0 == r1
    assert np.array_equal(C2, C1) and np.array_equal(p2, p1)


def test_solve_is_deterministic():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(1024, 1024, 128, 1, 1, 1, comm)
    cb.LU_rep(gv)
    B = np.random.default_rng(8).standard_normal((gv.M, 9))
    assert np.array_equal(cb.lu_solve(gv, B), cb.lu_solve(gv, B))
    gv.free_comms()
    comm.close()


def test_solve_bits_are_pinned(golden_dir):
    """X of integer right-hand sides is the one recorded by tests/golden/make_solve_golden.py"""
    with open(os.path.join(golden_dir, "solve_bits.json")) as f:
        want = json.load(f)
    for N, v in make_solve_golden.LU_CASES:
        assert make_solve_golden.lu_solve_bits(N, v) == want[f"lu_{N}_{v}"], (N, v)


@pytest.mark.parametrize("N,v,Px,Py,Pz", GRIDS)
def test_multi_gpu_solve(N, v, Px, Py, Pz):
    if n_gpus() < Px * Py * Pz:
        pytest.skip(f"needs {Px * Py * Pz} GPUs")
    M = layout.dims(N, v, Px, Py, Pz)["M"]
    rng = np.random.default_rng(N + v)
    Bs = [rng.standard_normal((M, 3)), rng.standard_normal((M, 70))]
    g = _solve_on_grid(N, v, Px, Py, Pz, Bs)
    _check(g, N, v, Px, Py, Pz, Bs)
    # the same solve twice on the grid is bit-identical
    g2 = _solve_on_grid(N, v, Px, Py, Pz, Bs[:1])
    assert np.array_equal(g2["X"][0][0], g["X"][0][0])


def test_bench_size_backward_error():
    """BASELINE config C2 (N=16384, v=256, one GPU) with 4 right-hand sides."""
    N, v = 16384, 256
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    cb.LU_rep(gv)
    B = np.random.default_rng(16).standard_normal((gv.M, 4))
    X = cb.lu_solve(gv, B)
    assert solve_ref.backward_error(gv.data, X, B) <= ETA_TOL
    gv.free_comms()
    comm.close()
