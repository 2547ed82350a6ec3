"""CPU: oracle/cond_ref.py restates LAPACK's condition estimators (dgecon with NORM = '1' on dgetrf factors, dpocon with
UPLO = 'L' on a Cholesky factor) and the 1-norm of an input in the conflux layout, read as the device kernel reads it."""
import numpy as np
import pytest
import scipy.linalg as sl
from scipy.linalg import lapack

from oracle import chol_ref, chol_solve_ref, cond_ref, layout

SIZES = [1, 2, 7, 64, 200, 512]


def _graded(n, rng):
    d = 2.0 ** np.linspace(-10, 10, n)
    return d[:, None] * rng.standard_normal((n, n)) * d[None, :]


def _kappa(n, rng, kappa=1e8):
    U, _ = np.linalg.qr(rng.standard_normal((n, n)))
    V, _ = np.linalg.qr(rng.standard_normal((n, n)))
    return (U * np.logspace(0, -np.log10(kappa), n)) @ V.T


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["random", "graded", "kappa"])
def test_gecon_matches_lapack(n, kind):
    rng = np.random.default_rng(n)
    A = {"random": rng.standard_normal((n, n)), "graded": _graded(n, rng), "kappa": _kappa(n, rng)}[kind]
    lu, piv, info = lapack.dgetrf(A)
    assert info == 0
    anorm = np.abs(A).sum(0).max()
    want, info = lapack.dgecon(lu, anorm, norm="1")
    assert info == 0
    got, _ = cond_ref.gecon(lu, anorm)
    assert abs(got - want) <= 1e-12 * want


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["random", "graded", "kappa"])
def test_pocon_matches_lapack(n, kind):
    rng = np.random.default_rng(n + 1)
    G = {"random": rng.standard_normal((n, n)), "graded": _graded(n, rng), "kappa": _kappa(n, rng, 1e4)}[kind]
    A = G @ G.T + (n if kind == "random" else 0) * np.eye(n)
    A = (A + A.T) / 2
    L = np.linalg.cholesky(A)
    anorm = np.abs(A).sum(0).max()
    want, info = lapack.dpocon(L, anorm, uplo="L")
    assert info == 0
    got, _ = cond_ref.pocon(L, anorm)
    assert abs(got - want) <= 1e-12 * want


def test_singular_estimate_is_zero():
    assert cond_ref.rcond(1.0, np.inf) == 0.0 and cond_ref.rcond(1.0, np.nan) == 0.0 and cond_ref.rcond(0.0, 1.0) == 0.0


GRIDS = [(64, 8, 1, 1, 1), (128, 16, 1, 1, 2), (64, 8, 2, 2, 1), (128, 8, 2, 2, 2), (96, 8, 3, 3, 1), (100, 16, 1, 1, 1)]


@pytest.mark.parametrize("N,v,Px,Py,Pz", GRIDS)
def test_norm1_of_lu_layout(N, v, Px, Py, Pz):
    M = layout.dims(N, v, Px, Py, Pz)["M"]
    A = np.random.default_rng(N + Px).standard_normal((M, M))
    locs = layout.scatter(A, v, Px, Py, Pz)
    for r in range(len(locs)):
        if r % Pz:
            locs[r][...] = np.nan                                        # the layers pk != 0 are not read
    assert cond_ref.norm1_lu(locs, N, v, Px, Py, Pz) == np.abs(A).sum(0).max() or np.isclose(
        cond_ref.norm1_lu(locs, N, v, Px, Py, Pz), np.abs(A).sum(0).max(), rtol=1e-15, atol=0)


@pytest.mark.parametrize("N,v,Px,Py,Pz", GRIDS + [(100, 16, 2, 1, 1), (112, 16, 3, 2, 1), (80, 16, 1, 3, 2)])
def test_norm1_of_cholesky_layout(N, v, Px, Py, Pz):
    d = chol_ref.dims(N, v, Px, Py, Pz)
    A = np.random.default_rng(N + Py).standard_normal((d["N"], d["N"]))
    locs = chol_solve_ref.scatter(A, N, v, Px, Py, Pz, upper=np.nan, pad=np.nan, layers=np.nan)
    for r in range(len(locs)):                                           # the diagonal tiles' upper triangles
        if r % Pz:
            continue
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        for lti in range(d["Ml"] // v):
            for ltj in range(d["Nl"] // v):
                if lti * Px + pi == ltj * Py + pj < d["Kappa"]:
                    blk = locs[r][lti * v:(lti + 1) * v, ltj * v:(ltj + 1) * v]
                    blk[np.triu_indices(v, 1)] = np.nan
    got = cond_ref.norm1_chol(locs, N, v, Px, Py, Pz)
    want = np.abs(chol_ref.lower_sym(A)).sum(0).max()
    assert np.isfinite(got) and abs(got - want) <= 1e-15 * want
