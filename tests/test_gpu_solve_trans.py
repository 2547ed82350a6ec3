"""GPU: cflx_lu_solve_trans (A^T X = B with the factors left on the device) against the host triangular solves on the
device's own factors and the schedule restatement (oracle/solve_trans_ref.py); its state rules; and that it leaves the
factorisation, the validation and the plain solve (bit for bit, tests/golden/solve_bits.json) untouched.

Tolerances: the backward error ||B - A^T X||_F / (||A||_F ||X||_F + ||B||_F) <= 1e-13, and X within 1e-10 max|X| of the
host solve and of the restatement on the same factors (the same operations, in other summation orders)."""
import json
import os

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import layout, solve_ref, solve_trans_ref
from tests._harness import n_gpus, run_ranks
from tests.golden import make_solve_golden
from tests.test_gpu_solve import GRIDS

pytestmark = pytest.mark.gpu
ETA_TOL = 1e-13
X_TOL = 1e-10


def _solve_on_grid(N, v, Px, Py, Pz, Bs, A_locals=None):
    """Factor once, then solve A^T X = B for every B in Bs; returns per-rank A, C, perm and the X of every B."""
    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        if A_locals is not None:
            gv.data[...] = np.asarray(A_locals[gv.rank]).reshape(gv.Ml, gv.Nl)
        C = np.zeros((gv.Ml, gv.Nl))
        perm = np.zeros(gv.M, dtype=np.int32)
        cb.LU_rep(gv, C, perm)
        Xs = [cb.lu_solve(gv, B, trans=True) for B in Bs]
        res = dict(A=gv.data.copy(), C=C, perm=perm, X=Xs)
        gv.free_comms()
        return res

    rs = run_ranks(Px * Py * Pz, body)
    return dict(A=[r["A"] for r in rs], C=[r["C"] for r in rs], perm=rs[0]["perm"], X=[r["X"] for r in rs])


def _check(g, N, v, Px, Py, Pz, Bs):
    A = layout.assemble(g["A"], N, v, Px, Py, Pz)
    LU = layout.assemble(g["C"], N, v, Px, Py, Pz)
    for i, B in enumerate(Bs):
        X = g["X"][0][i]
        for Xr in g["X"]:
            assert np.array_equal(Xr[i], X)                              # bit-identical on every rank
        assert X.shape == B.shape
        X2, B2 = X.reshape(len(B), -1), B.reshape(len(B), -1)
        assert solve_ref.backward_error(A.T, X2, B2) <= ETA_TOL
        scale = np.abs(X).max()
        assert np.abs(X2 - solve_trans_ref.host_solve(LU, g["perm"], B2)).max() <= X_TOL * scale
        Xo = solve_trans_ref.solve(g["C"], g["perm"], B, N, v, Px, Py, Pz)
        assert np.abs(X - Xo).max() <= X_TOL * scale


@pytest.mark.parametrize("N,v", [(16, 4), (96, 16), (512, 64), (1024, 128), (4096, 256), (100, 16)])
def test_single_gpu_transposed_solve(N, v):
    M = layout.dims(N, v, 1, 1, 1)["M"]
    rng = np.random.default_rng(N + 1)
    Bs = [rng.standard_normal((M, nrhs)) for nrhs in (1, 3, 64, 130)] + [rng.standard_normal(M)]
    g = _solve_on_grid(N, v, 1, 1, 1, Bs)
    _check(g, N, v, 1, 1, 1, Bs)


def test_single_gpu_transposed_solve_standard_normal_matrix():
    N, v = 1024, 128
    A = np.random.default_rng(3).standard_normal((N, N))
    Bs = [np.random.default_rng(4).standard_normal((N, 5))]
    g = _solve_on_grid(N, v, 1, 1, 1, Bs, A_locals=[A])
    _check(g, N, v, 1, 1, 1, Bs)


def test_state_rules_and_queued_input():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(256, 256, 32, 1, 1, 1, comm)
    B = np.random.default_rng(1).standard_normal((gv.M, 2))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_solve(gv, B, trans=True)                                  # no factorisation yet
    cb.LU_rep(gv)
    X = cb.lu_solve(gv, B, trans=True)
    assert solve_ref.backward_error(gv.data.T, X, B) <= ETA_TOL
    with pytest.raises(cb.ConfluxError, match="status -1"):
        cb.lu_solve(gv, np.zeros((gv.M, 0)), trans=True)                # nrhs < 1
    a = np.ascontiguousarray(gv.data)
    cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_solve(gv, B, trans=True)                                  # new input, not factored yet
    gv.free_comms()
    comm.close()

    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(512, 512, 64, 1, 1, 1, comm)
    rng = np.random.default_rng(21)
    mats = [cb.pinned_empty((gv.Ml, gv.Nl)) for _ in range(2)]
    for m in mats:
        m[...] = rng.standard_normal((gv.Ml, gv.Nl))
    gv.data = mats[0]
    cb.LU_rep(gv, next_data=mats[1])
    B0 = rng.standard_normal((gv.M, 2))
    X0 = cb.lu_solve(gv, B0, trans=True)                                # the run whose input buffer was handed on
    assert solve_ref.backward_error(mats[0].T, X0, B0) <= ETA_TOL
    cb.LU_rep(gv, upload=False)                                         # factors the queued matrix
    B1 = rng.standard_normal((gv.M, 3))
    X1 = cb.lu_solve(gv, B1, trans=True)                                # a second solve after queue_next_local
    assert solve_ref.backward_error(mats[1].T, X1, B1) <= ETA_TOL
    for m in mats:
        cb.pinned_free(m)
    gv.free_comms()
    comm.close()


def test_no_side_effects_and_interleaving(golden_dir):
    """Two transposed solves give the same bits; the factors, permutation and residual are untouched; and plain solves
    interleaved with transposed ones after one factorisation still give the pinned bits."""
    N, v = 1024, 128

    def run(trans):
        comm = cb.Comm(1, 0, None, 0)
        gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
        cb.LU_rep(gv)
        B = np.random.default_rng(0).standard_normal((gv.M, 7))
        Xt = [cb.lu_solve(gv, B, trans=True) for _ in range(2)] if trans else None
        C, perm = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
        cb.check(cb.lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "get_factors")
        resid = cb.validate(gv)
        X = cb.lu_solve(gv, B)
        gv.free_comms()
        comm.close()
        return C, perm, resid, X, Xt

    C0, p0, r0, X0, _ = run(False)
    C1, p1, r1, X1, Xt = run(True)
    assert np.array_equal(Xt[0], Xt[1])
    assert np.array_equal(C0, C1) and np.array_equal(p0, p1) and r0 == r1 and np.array_equal(X0, X1)

    with open(os.path.join(golden_dir, "solve_bits.json")) as f:
        want = json.load(f)
    for Nn, vv in make_solve_golden.LU_CASES:                           # plain solves between transposed ones
        comm = cb.Comm(1, 0, None, 0)
        gv = cb.lu_params(Nn, Nn, vv, 1, 1, 1, comm)
        cb.LU_rep(gv)
        got = {}
        for n in make_solve_golden.NRHS:
            cb.lu_solve(gv, make_solve_golden.rhs(gv.M, n), trans=True)
            got[str(n)] = make_solve_golden.digest(cb.lu_solve(gv, make_solve_golden.rhs(gv.M, n)))
        gv.free_comms()
        comm.close()
        assert got == want[f"lu_{Nn}_{vv}"], (Nn, vv)


def test_interleaved_plain_solve_keeps_pinned_bits():
    """plain and transposed solves after one factorisation: the plain X is the one a fresh object gives"""
    N, v = 1024, 128
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    cb.LU_rep(gv)
    B = np.random.default_rng(5).integers(-4, 5, (gv.M, 64)).astype(np.float64)
    X0 = cb.lu_solve(gv, B)
    cb.lu_solve(gv, B[:, :3], trans=True)
    X1 = cb.lu_solve(gv, B)
    cb.lu_solve(gv, B, trans=True)
    X2 = cb.lu_solve(gv, B)
    assert np.array_equal(X0, X1) and np.array_equal(X0, X2)
    gv.free_comms()
    comm.close()


@pytest.mark.parametrize("N,v,Px,Py,Pz", GRIDS)
def test_multi_gpu_transposed_solve(N, v, Px, Py, Pz):
    if n_gpus() < Px * Py * Pz:
        pytest.skip(f"needs {Px * Py * Pz} GPUs")
    M = layout.dims(N, v, Px, Py, Pz)["M"]
    rng = np.random.default_rng(N + v + 1)
    Bs = [rng.standard_normal((M, 3)), rng.standard_normal((M, 70))]
    g = _solve_on_grid(N, v, Px, Py, Pz, Bs)
    _check(g, N, v, Px, Py, Pz, Bs)
    g2 = _solve_on_grid(N, v, Px, Py, Pz, Bs[:1])
    assert np.array_equal(g2["X"][0][0], g["X"][0][0])
