"""CPU checks of oracle/ldlt_ref.py, the restatement cflx_chol_factor_ldlt and cflx_chol_rbt are tested against."""
import numpy as np
import pytest

from oracle import hp_ref, ldlt_ref, rbt_ref


@pytest.mark.parametrize("n,m,c_zero", [(40, 24, False), (48, 16, True), (7, 5, False)])
def test_kkt_factor_within_bounds(n, m, c_zero):
    K = ldlt_ref.kkt(n, m, seed=n + m, c_zero=c_zero)
    f = ldlt_ref.factor(K)
    assert f["info"] == 0 and f["nrepl"] == 0
    assert f["inertia"] == (n, m, 0) == ldlt_ref.inertia(K)
    assert np.all(np.diag(f["R"]) > 0)
    assert ldlt_ref.componentwise_ok(K, f["R"], f["s"])
    assert ldlt_ref.normwise_ok(K, f["R"], f["s"], hp_ref.diag_block_kappa(f["R"], 8))


@pytest.mark.parametrize("npos,nneg", [(32, 32), (60, 4), (1, 63)])
def test_rbt_transformed_inertia_and_bounds(npos, nneg):
    A = ldlt_ref.with_inertia(64, npos, nneg, seed=npos)
    A[0, 0] = 0.0  # a zero leading pivot: the factorisation without pivoting needs the transform
    assert ldlt_ref.factor(A)["info"] == 1
    u, _ = rbt_ref.multipliers(64, 2, 7)
    W = rbt_ref.global_w(ldlt_ref.mirror(A), u, u)
    f = ldlt_ref.factor(W)
    assert f["info"] == 0
    assert f["inertia"] == ldlt_ref.inertia(A) == ldlt_ref.inertia(W)
    assert ldlt_ref.componentwise_ok(W, f["R"], f["s"])


def test_spd_signs_are_plus_and_match_cholesky():
    A = hp_ref.random_spd(48, 1e3, np.random.default_rng(3))
    f = ldlt_ref.factor(A)
    assert np.all(f["s"] == 1.0) and f["inertia"] == (48, 0, 0)
    L = np.linalg.cholesky(A)
    assert np.abs(f["R"] - L).max() <= 1e-12 * np.abs(L).max()


def test_tiny_rule_and_zero_pivot():
    A = np.array([[0.0, 0.0], [1.0, 0.0]])
    f = ldlt_ref.factor(A)
    assert f["info"] == 1 and f["inertia"][2] >= 1
    g = ldlt_ref.factor(A, tiny=1e-8)
    assert g["nrepl"] >= 1 and g["info"] == 0 and g["s"][0] == 1.0
    h = ldlt_ref.factor(np.array([[-1e-12]]), tiny=1e-8)
    assert h["s"][0] == -1.0 and h["R"][0, 0] == pytest.approx(1e-4)


def test_residual_rejects_a_defect():
    K = ldlt_ref.kkt(20, 12, seed=1)
    f = ldlt_ref.factor(K)
    R = f["R"].copy()
    R[15, 3] *= 1 + 1e-9
    assert not ldlt_ref.componentwise_ok(K, R, f["s"])
    s = f["s"].copy()
    s[25] = -s[25]
    assert not ldlt_ref.componentwise_ok(K, f["R"], s)


def test_mirror():
    A = np.tril(np.arange(16.0).reshape(4, 4)) + np.triu(np.full((4, 4), np.nan), 1)
    M = ldlt_ref.mirror(A)
    assert np.array_equal(M, M.T) and np.array_equal(np.tril(M), np.tril(A))


@pytest.mark.parametrize("v,Px,Py,depth", [(32, 2, 1, 2), (32, 1, 2, 2), (16, 2, 3, 1), (64, 4, 2, 3), (8, 3, 3, 2)])
def test_fits_and_smallest_order_px_ne_py(v, Px, Py, depth):
    q = (v * np.lcm(Px, Py)) << depth
    for N in (v, q - v, q, q + v, 3 * q, 3 * q + 8):
        assert ldlt_ref.fits(N, v, Px, Py, depth) == (N % q == 0)
        m = ldlt_ref.smallest_order(N, v, Px, Py, depth)
        assert m >= N and m % q == 0 and m - N < q
        # both conditions of the rule: rows pair within a rank, and columns do
        assert ldlt_ref.fits(m, v, Px, Py, depth)
        assert rbt_ref.fits(m, v, Px, depth) and rbt_ref.fits(m, v, Py, depth)
    if Px != Py:
        # the LU's rule on Px alone is not enough when Py has another factor
        N = (v * Px) << depth
        assert rbt_ref.fits(N, v, Px, depth)
        assert ldlt_ref.fits(N, v, Px, Py, depth) == (N % ((v * np.lcm(Px, Py)) << depth) == 0)


def test_header_declares_the_new_entry_points():
    import os
    from conflux_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = open(os.path.join(root, "include", "conflux_b200.h")).read()
    for name in ("cflx_chol_factor_ldlt", "cflx_chol_rbt", "cflx_chol_rbt_solve", "cflx_chol_rbt_apply_local",
                 "cflx_chol_get_signs", "cflx_chol_get_input", "cflx_dbg_ldlt_tile",
                 "cflx_dbg_solve_signs"):
        assert name + "(" in h and name in _lib.SYMBOLS
