"""CPU: the restatement of cflx_lu_det / cflx_chol_det (oracle/det_ref.py).  Its exact-range pair is the exact product to
within n rounding errors; with scipy's LU factors it gives numpy's slogdet; its permutation parity is det(P); its
rank-by-rank diagonal gather gives the dense diagonal on every LU and Cholesky grid shape without reading anything off
the diagonal; and the C++ facades compile."""
import math
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import scipy.linalg

from oracle import chol_ref, chol_solve_ref, det_ref, layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -53


def _exact(d, s=(), square=False):
    p = Fraction(1)
    for x in d:
        p *= Fraction(abs(float(x)))
    for v in s:
        for x in v:
            p /= Fraction(abs(float(x)))
    return p * p if square else p


def _pair(r):
    return Fraction(r["mant"]) * Fraction(2) ** r["exp"]


@pytest.mark.parametrize("n", [1, 7, 255, 256, 257, 1000])
def test_pair_is_the_exact_product(n):
    rng = np.random.default_rng(n)
    d = rng.standard_normal(n) * np.exp2(rng.integers(-300, 300, n))
    r = det_ref.product(d)
    assert 0.5 <= r["mant"] < 1.0 and r["first_zero"] == 0 and r["nonfinite"] == 0
    assert r["neg"] == int(np.sum(d < 0)) % 2
    ex = _exact(d)
    assert abs(_pair(r) / ex - 1) <= (n + 16) * U
    s1, s2 = rng.uniform(0.5, 4.0, n), np.exp2(rng.integers(-60, 60, n).astype(float))
    r = det_ref.product(d, s1, s2, square=True)
    assert r["neg"] == 0
    assert abs(_pair(r) / _exact(d, (s1, s2), square=True) - 1) <= (6 * n + 16) * U


def test_extreme_and_special_entries():
    sub = np.array([5e-324, 2.5e-310, -1e-315, 2.0 ** -1000, 2.0 ** 1000, -2.0 ** 1023])
    r = det_ref.product(sub)
    assert abs(_pair(r) / _exact(sub) - 1) <= 16 * U and r["exp"] < -2000
    assert r["neg"] == 0                                              # two negatives
    pw = np.array([5e-324, 2.0 ** -1000, 2.0 ** 1000, -2.0 ** 1023, 0.75])
    assert _pair(det_ref.product(pw)) == _exact(pw)                   # one significant bit each but 0.75: no rounding
    n = 300
    for pos in (0, n // 2, n - 1):
        d = np.full(n, 3.0)
        d[pos] = 0.0
        r = det_ref.product(d)
        assert (r["first_zero"], r["mant"], r["exp"], r["nonfinite"]) == (pos + 1, 0.0, 0, 0)
    d = np.full(n, 3.0)
    d[10], d[20] = np.inf, 0.0
    r = det_ref.product(d)
    assert r["nonfinite"] == 1 and math.isnan(r["mant"]) and r["first_zero"] == 21
    d[10], d[5] = np.nan, 0.0
    r = det_ref.product(d)
    assert r["nonfinite"] == 0 and r["mant"] == 0.0 and r["first_zero"] == 6
    r = det_ref.product(np.full(n, 3.0), np.r_[np.ones(n - 1), 0.0])    # a zero divisor
    assert r["nonfinite"] == 1 and r["first_zero"] == 0


def _perm_of(P):
    """perm with row q of P^T A = row perm[q] of A, for scipy's A = P L U"""
    return np.argmax(P, axis=0)


@pytest.mark.parametrize("n", [1, 2, 5, 40, 200])
def test_parity_is_det_of_P(n):
    rng = np.random.default_rng(n)
    for _ in range(5):
        perm = rng.permutation(n)
        P = np.eye(n)[perm]
        assert (-1) ** det_ref.perm_parity(perm) == round(np.linalg.det(P))


def _graded(n, rng):
    return np.diag(np.exp2(rng.integers(-200, 200, n).astype(float))) @ rng.standard_normal((n, n)) @ np.diag(
        np.exp2(rng.integers(-200, 200, n).astype(float)))


def _hilbert(n):
    i = np.arange(n)
    return 1.0 / (i[:, None] + i[None, :] + 1.0)


@pytest.mark.parametrize("kind", ["random", "graded", "hilbert", "big"])
def test_lu_restatement_matches_slogdet(kind):
    rng = np.random.default_rng(len(kind))
    n = {"random": 150, "graded": 120, "hilbert": 10, "big": 600}[kind]
    A = {"random": lambda: rng.standard_normal((n, n)), "graded": lambda: _graded(n, rng),
         "hilbert": lambda: _hilbert(n), "big": lambda: 5.0 + rng.random((n, n))}[kind]()
    P, L, Uf = scipy.linalg.lu(A)
    perm = _perm_of(P)
    assert np.array_equal(A[perm], P.T @ A)
    r = det_ref.product(np.diag(Uf))
    sign = (-1.0) ** (r["neg"] ^ det_ref.perm_parity(perm))
    lad = det_ref.logabs(r["mant"], r["exp"])
    s_np, l_np = np.linalg.slogdet(A)
    assert sign == s_np
    assert abs(lad - l_np) <= 1e-13 * abs(l_np) + np.linalg.cond(A, 1) * n * U     # kappa n u: two LU codes
    if kind == "big":
        with np.errstate(over="ignore"):
            assert not np.isfinite(np.prod(np.diag(Uf)))             # the plain product overflows
        assert r["exp"] > 1024


def _nan_off_diag(shares, v, Px, Py, Pz, Nt):
    """copies of the shares with NaN everywhere but the diagonal entries of the real diagonal tiles of layer 0"""
    out = []
    for r, A in enumerate(shares):
        pi, pj, pk = r // (Py * Pz), (r // Pz) % Py, r % Pz
        B = np.full_like(A, np.nan)
        if pk == 0:
            for t in range(Nt):
                lr, lc = (t // Px) * v, (t // Py) * v
                if t % Px == pi and t % Py == pj and lr < A.shape[0] and lc < A.shape[1]:
                    for e in range(v):
                        B[lr + e, lc + e] = A[lr + e, lc + e]
        out.append(B)
    return out


LU_GRIDS = [((1, 1, 1), 96, 8), ((1, 1, 2), 96, 8), ((2, 2, 1), 96, 8), ((2, 2, 2), 96, 8), ((3, 3, 1), 96, 8),
            ((1, 1, 1), 100, 16), ((2, 2, 1), 100, 16)]


@pytest.mark.parametrize("grid,N,v", LU_GRIDS, ids=lambda x: "x".join(map(str, x)) if isinstance(x, tuple) else str(x))
def test_lu_gather_is_the_dense_diagonal(grid, N, v):
    d = layout.dims(N, v, *grid)
    A = np.random.default_rng(N + sum(grid)).standard_normal((d["M"], d["M"]))
    shares = _nan_off_diag(layout.scatter(A, v, *grid), v, *grid, d["Nt"])
    g = det_ref.gather_diag(shares, v, *grid, d["Nt"], d["M"])
    assert np.array_equal(g, np.diag(A))
    perm = np.random.default_rng(1).permutation(d["M"])
    want = det_ref.product(np.diag(A))
    o = det_ref.lu_det(shares, perm, N, v, *grid)
    assert (o["mantissa"], o["exponent"], o["info"]) == (want["mant"], want["exp"], 0)


CHOL_GRIDS = [((1, 1, 1), 100, 16), ((2, 2, 1), 96, 8), ((2, 2, 2), 96, 8), ((4, 2, 1), 100, 8), ((3, 2, 1), 100, 8),
              ((1, 3, 2), 100, 8), ((1, 1, 2), 64, 8)]


@pytest.mark.parametrize("grid,N,v", CHOL_GRIDS, ids=lambda x: "x".join(map(str, x)) if isinstance(x, tuple) else str(x))
def test_chol_gather_is_the_dense_diagonal(grid, N, v):
    d = chol_ref.dims(N, v, *grid)
    L = np.tril(np.random.default_rng(N + sum(grid)).uniform(0.5, 2.0, (d["N"], d["N"])))
    shares = chol_solve_ref.scatter(L, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)
    shares = _nan_off_diag(shares, v, *grid, d["Kappa"])
    assert np.array_equal(det_ref.gather_diag(shares, v, *grid, d["Kappa"], d["N"]), np.diag(L))
    o = det_ref.chol_det(shares, N, v, *grid)
    assert abs(o["logabsdet"] - 2 * np.sum(np.log(np.diag(L)))) <= 1e-12 * d["N"]


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")
def test_cpp_facades_compile(tmp_path):
    src = tmp_path / "use_det.cpp"
    src.write_text('#include "conflux/lu/conflux_b200.hpp"\n'
                   '#include "conflux/cholesky/conflux_b200_cholesky.hpp"\n'
                   "double f(conflux::lu_params<double>& g) { double s, m; int64_t e; int k;\n"
                   "  return conflux::LU_det(g, true, &s, &m, &e, &k) + conflux::choleskyLogdet(false, &m, &e); }\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)], check=True)
