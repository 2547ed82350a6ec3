"""CPU: the restatement of the LU in a prescribed row order (oracle/fixed_ref.py) against the pivoted restatement and
exact integer cases, the fixed schedule's per-grid-row pivot counts, and the new entry points' refusal without a GPU."""
import ctypes

import numpy as np
import pytest

import conflux_b200 as cb
from conflux_b200 import _lib
from oracle import fixed_ref, layout, restate

FACTOR_TOL = 1e-10        # as tests/test_gpu_lu.py: L\U element-wise, relative to ||A||_max


@pytest.mark.parametrize("N,v", [(16, 4), (64, 8), (96, 16), (256, 32), (512, 64), (1024, 128), (768, 256), (100, 16)])
def test_last_permutation_reproduces_the_pivoted_factors(N, v):
    A_loc = restate.init_matrix(N, v)
    o = restate.lu(A_loc, N, v)
    A = layout.assemble(A_loc, N, v, 1, 1, 1)
    want = layout.assemble(o["C"], N, v, 1, 1, 1)
    r = fixed_ref.lu(A, o["perm"], v)
    assert (r["nrepl"], r["info"]) == (0, 0)
    assert np.abs(r["LU"] - want).max() <= FACTOR_TOL * np.abs(A).max()


def integer_case(M, zero_cols, rng, small=()):
    """A = L U from integer factors, exact in floating point: unit L with entries in {-1, 0, 1}, U with pivots +-1 / +-2,
    U(j, j) = 0 at zero_cols and -0.25 at `small`; L's column is zero below those pivots, so no later step depends on
    them.  Returns (A, L\\U)."""
    L = np.tril(rng.integers(-1, 2, (M, M)).astype(float), -1)
    U = np.triu(rng.integers(-2, 3, (M, M)).astype(float), 1)
    d = rng.choice([-2.0, -1.0, 1.0, 2.0], M)
    for j in zero_cols:
        d[j] = 0.0
    for j in small:
        d[j] = -0.25
    for j in list(zero_cols) + list(small):
        L[j + 1:, j] = 0.0
    U += np.diag(d)
    A = (L + np.eye(M)) @ U
    return A, L + U


@pytest.mark.parametrize("M,v,zero", [(64, 16, 0), (64, 16, 5), (64, 16, 16), (64, 16, 15), (64, 16, 63), (128, 64, 32),
                                      (128, 64, 96)],
                         ids=["first", "inside-tile", "tile-boundary", "tile-end", "last", "block32-boundary",
                              "second-tile-block"])
def test_zero_pivot_info_and_tiny_replacement(M, v, zero):
    rng = np.random.default_rng(M + zero)
    A, LU = integer_case(M, [zero], rng)
    r = fixed_ref.lu(A, np.arange(M), v)
    assert (r["info"], r["nrepl"]) == (zero + 1, 0)
    assert np.array_equal(np.triu(r["LU"])[:zero + 1, :zero + 1], np.triu(LU)[:zero + 1, :zero + 1])
    r = fixed_ref.lu(A, np.arange(M), v, tiny=0.5)
    want = LU.copy()
    want[zero, zero] = 0.5
    assert (r["info"], r["nrepl"]) == (0, 1)
    assert np.array_equal(r["LU"], want)


def test_tiny_rule_keeps_the_sign_and_counts_every_replacement():
    M, v = 96, 32
    rng = np.random.default_rng(7)
    A, LU = integer_case(M, [3, 40], rng, small=[70])
    perm = rng.permutation(M)
    r = fixed_ref.lu(A[np.argsort(perm)], perm, v, tiny=0.5)    # rows scattered by perm^-1: A[perm] is the case again
    want = LU.copy()
    want[3, 3] = want[40, 40] = 0.5
    want[70, 70] = -0.5
    assert (r["info"], r["nrepl"]) == (0, 3)
    assert np.array_equal(r["LU"], want)
    assert fixed_ref.lu(A, np.arange(M), v, tiny=0.0)["info"] == 4


GRIDS = [(1, 1, 1), (1, 1, 2), (2, 2, 1), (2, 2, 2), (3, 3, 1), (3, 3, 2)]


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "x".join(map(str, g)))
@pytest.mark.parametrize("order", ["identity", "reversed", "random"])
def test_step_counts_sum_to_v_and_fit_the_active_rows(grid, order):
    v = 8
    d = layout.dims(150, v, *grid)
    M, Px = d["M"], grid[0]
    perm = {"identity": np.arange(M), "reversed": np.arange(M)[::-1],
            "random": np.random.default_rng(M).permutation(M)}[order]
    cnt = fixed_ref.step_counts(perm, v, Px)
    assert cnt.shape == (M // v, Px)
    assert (cnt.sum(axis=1) == v).all()
    held = np.array([sum(1 for g in range(M) if (g // v) % Px == p) for p in range(Px)])
    assert (held == d["Ml"]).all()
    active = held - np.vstack([np.zeros((1, Px), dtype=np.int64), np.cumsum(cnt, axis=0)[:-1]])
    assert (cnt <= active).all() and (active >= 0).all()
    assert (np.cumsum(cnt, axis=0)[-1] == held).all()            # every row is promoted exactly once


def test_new_entry_points_refuse_without_gpu():
    n = ctypes.c_int(-1)
    assert _lib.lib().cflx_device_count(ctypes.byref(n)) == 0
    if n.value > 0:
        pytest.skip("GPU present")
    with pytest.raises(cb.ConfluxError, match="no CPU fallback"):
        cb.dbg.getrf_nopiv_tile(np.eye(8))
    with pytest.raises(cb.ConfluxError, match="no CPU fallback"):   # LU_rep_fixed needs a handle, which needs a device
        cb.lu_params(64, 64, 16, 1, 1, 1, cb.Comm(1, 0, None, 0))
    info = ctypes.c_int()
    assert _lib.lib().cflx_lu_factor_fixed(None, None, 0.0, None, ctypes.byref(info), None) == -1
