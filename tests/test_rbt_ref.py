"""CPU: the random butterfly transforms' restatement (oracle/rbt_ref.py): the library's host multipliers bit for bit,
their argument rules, the per-share operations reassembled against the global transform, the solve identity, and the new
device entry points' refusal without a GPU."""
import ctypes
import math

import numpy as np
import pytest

import conflux_b200 as cb
from conflux_b200 import _lib
from oracle import layout, rbt_ref


@pytest.mark.parametrize("M,depth,seed", [(2, 1, 0), (64, 2, 1), (96, 3, 12345), (256, 4, 2**64 - 1), (1024, 2, 99)])
def test_multipliers_bit_equal_and_in_range(M, depth, seed):
    u, v = cb.rbt_multipliers(M, depth, seed)
    ru, rv = rbt_ref.multipliers(M, depth, seed)
    assert np.array_equal(u, ru) and np.array_equal(v, rv)
    lo, hi = math.exp(-0.05), math.exp(0.05)
    assert ((u >= lo) & (u <= hi)).all() and ((v >= lo) & (v <= hi)).all()
    assert not np.array_equal(u, v)


def test_multiplier_argument_rules():
    L = _lib.lib()
    out = np.empty(64)
    seed = ctypes.c_uint64(0)
    for M, depth in [(16, 0), (16, 5), (0, 1), (-4, 1), (12, 3), (6, 2)]:
        assert L.cflx_rbt_multipliers(M, depth, seed, out.ctypes.data, out.ctypes.data) == -1
    assert L.cflx_rbt_multipliers(16, 2, seed, None, None) == -1
    assert L.cflx_rbt_multipliers(16, 2, seed, out.ctypes.data, None) == 0
    assert L.cflx_rbt_multipliers(16, 2, seed, None, out.ctypes.data) == 0


@pytest.mark.parametrize("depth", [1, 2, 3])
@pytest.mark.parametrize("Pz", [1, 2])
@pytest.mark.parametrize("P", [1, 2, 3])
def test_per_share_transform_is_the_global_one(P, Pz, depth):
    v = 4
    M = 2 * ((v * P) << depth)
    assert rbt_ref.fits(M, v, P, depth) and layout.dims(M, v, P, P, Pz)["M"] == M
    rng = np.random.default_rng(100 * P + 10 * Pz + depth)
    A = rng.standard_normal((M, M))
    u, vv = rbt_ref.multipliers(M, depth, 7 * depth)
    W = rbt_ref.global_w(A, u, vv)
    shares = layout.scatter(A, v, P, P, Pz)
    out = list(shares)
    for pi in range(P):
        for pj in range(P):
            r = layout.rank_of(pi, pj, 0, P, P, Pz)
            out[r] = rbt_ref.share_op(4, shares[r], v, depth, u, vv, (P, P), (pi, pj))
    assert np.array_equal(layout.assemble(out, M, v, P, P, Pz), W)
    U, V = rbt_ref.matrices(u, vv)
    assert np.linalg.norm(U.T @ A @ V - W) <= 1e-14 * np.linalg.norm(W)
    # the right-hand-side operations: a share of an M x n matrix by local rows is the global operation's rows
    B = rng.standard_normal((M, 5))
    su, sv = rbt_ref.scales(u), rbt_ref.scales(vv)
    for op, Mat in ((0, U.T), (1, V), (2, V.T), (3, U)):
        g = rbt_ref.apply_rows(op, B, su, sv, np.arange(M))
        assert np.abs(g - Mat @ B).max() <= 1e-14 * np.abs(g).max()
        for pi in range(P):
            rows = rbt_ref.global_index(M // P, v, P, pi)
            assert np.array_equal(rbt_ref.share_op(op, B[rows], v, depth, u, vv, (P, P), (pi, 0)), g[rows])


def test_forward_operation_is_the_explicit_butterfly():
    """the forward operation is the explicit U: U applied to inv(U) B gives B back within rounding"""
    M, depth = 64, 3
    u, vv = rbt_ref.multipliers(M, depth, 5)
    U, V = rbt_ref.matrices(u, vv)
    B = np.random.default_rng(0).standard_normal((M, 3))
    su, sv = rbt_ref.scales(u), rbt_ref.scales(vv)
    X = rbt_ref.apply_rows(3, np.linalg.solve(U, B), su, sv, np.arange(M))
    assert np.abs(X - B).max() <= 1e-14


@pytest.mark.parametrize("trans", [False, True])
@pytest.mark.parametrize("depth", [1, 2, 4])
def test_solve_through_the_transform(depth, trans):
    M = 128
    rng = np.random.default_rng(depth)
    A = rng.standard_normal((M, M)) + M * np.eye(M)
    B = rng.standard_normal((M, 4))
    u, vv = rbt_ref.multipliers(M, depth, 3)
    X = rbt_ref.solve(A, B, u, vv, trans)
    want = np.linalg.solve(A.T if trans else A, B)
    assert np.abs(X - want).max() <= 1e-12 * np.abs(want).max()


def test_divisibility_rule():
    assert rbt_ref.fits(1024, 256, 1, 2) and not rbt_ref.fits(1024, 256, 1, 3)
    assert rbt_ref.smallest_order(1000, 64, 2, 2) == 1024 and rbt_ref.smallest_order(512, 64, 2, 2) == 512
    assert rbt_ref.smallest_order(16384, 512, 1, 2) == 16384


def test_new_entry_points_refuse_without_gpu():
    n = ctypes.c_int(-1)
    assert _lib.lib().cflx_device_count(ctypes.byref(n)) == 0
    if n.value > 0:
        pytest.skip("GPU present")
    u, vv = cb.rbt_multipliers(64, 2, 0)
    with pytest.raises(cb.ConfluxError, match="no CPU fallback"):
        cb.dbg.rbt_share(4, np.eye(32), 8, 2, u=u, vv=vv, M=64)
    L = _lib.lib()
    assert L.cflx_lu_rbt(None, 2, ctypes.c_uint64(0), None, None) == -1
    assert L.cflx_lu_rbt_solve(None, 0, 1, None, 1, None, 1, 1, None, None) == -1
    assert L.cflx_lu_rbt_apply_local(None, 0, 1, None, 1) == -1
