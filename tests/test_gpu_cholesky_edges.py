"""GPU: the Cholesky path kernel by kernel and end to end, against the extended-precision references and the error
bounds of oracle/hp_ref.py, on awkward inputs (ill-conditioned, graded, exact, NaN in entries that must not be read),
tile sizes that are not a multiple of 32, the 128-block tile driver, the int8 update, and matrices that are not
positive definite (the error must name LAPACK's column).

Constants: every tolerance is one of the hp_ref bounds (gamma_n = n u / (1 - n u), u = 2^-53):
  * diag_inverse_kernel (substitution):   |T X^ - I| <= gamma_nb |T| |X^|
  * potrf_tile_kernel / potrf128_kernel:  |A - L^ L^T| <= gamma_{v+1} |L^| |L^T|
  * the 128-block tile driver and the whole factorisation (panels solved with inverted diagonal blocks):
        ||A - L^ L^T||_F <= gamma_{n+1} (1 + 4 kappa_max) || |L^| |L^T| ||_F,
    kappa_max = the largest condition number of an inverted diagonal block (128 for the tile driver, nb of the panel
    TRSM), and the forward error against the longdouble factor ||L^ - L||_F / ||L||_2 <= kappa(A) eps / (1 - kappa(A) eps)
    with eps that bound over ||A||_2."""
import re

import numpy as np
import pytest
import scipy.linalg

import conflux_b200 as cb
from oracle import chol_ref, hp_ref as hp
from tests._harness import n_gpus, run_ranks
from tests.golden import make_chol_golden

pytestmark = pytest.mark.gpu

NBS = [4, 8, 16, 32, 64, 128]


def _chol_nb(v):
    return next(nb for nb in (128, 64, 32, 16, 8, 4) if v % nb == 0)


def _kappa_max(L, v):
    """largest condition number among the diagonal blocks the factorisation inverts"""
    k = hp.diag_block_kappa(L, _chol_nb(v))
    if v % 128 == 0 and v >= 256:
        k = max(k, hp.diag_block_kappa(L, 128))
    return k


def _spd(kind, n, rng):
    if kind == "k1e2":
        return hp.random_spd(n, 1e2, rng)
    if kind == "k1e8":
        return hp.random_spd(n, 1e8, rng)
    if kind == "graded":
        d = np.logspace(-3, 3, n)
        return d[:, None] * hp.random_spd(n, 1e2, rng) * d[None, :]
    if kind == "exact":
        return hp.exact_spd(n, rng)[0]
    if kind == "exact_wellcond":       # entries in {-1, 0, 1}, diagonal 8 .. 32: kappa(L) ~ 10 at n = 512
        return hp.exact_spd(n, rng, lmax=1, dmin=3, dmax=6)[0]
    raise ValueError(kind)


# ----------------------------------------------------------------------------------------------- diag_inverse_kernel
def _triangles(v, kind, rng, nb):
    """A00 = L\\U packed: U upper with its diagonal, L unit lower below it"""
    if kind == "well":
        U = np.triu(rng.uniform(-1, 1, (v, v))) * (2.0 / np.sqrt(v)) + np.diag(1.0 + rng.random(v))
        Lo = np.tril(rng.uniform(-1, 1, (v, v)), -1) * (2.0 / np.sqrt(v))
    elif kind == "graded":
        g = np.logspace(-6, 6, v)
        U = g[:, None] * (np.triu(rng.uniform(-1, 1, (v, v))) * (2.0 / np.sqrt(v)) + np.eye(v))
        Lo = np.tril(rng.uniform(-1, 1, (v, v)), -1) * (2.0 / np.sqrt(v))
    else:   # ill-conditioned, kappa_2 = 1e10 per block: U = R of a QR of a matrix with singular values 1 .. 1e-10, and a
            # unit lower I + t N with t set by bisection on log10 kappa
        U = np.zeros((v, v))
        Lo = np.zeros((v, v))
        for b in range(0, v, nb):
            n = min(nb, v - b)
            Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
            Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
            U[b:b + n, b:b + n] = np.linalg.qr((Q1 * np.logspace(0, -10, n)) @ Q2)[1]
            N = np.tril(rng.uniform(-1, 1, (n, n)), -1)
            lo, hi = 0.0, 1e6
            for _ in range(60):
                t = np.sqrt(lo * hi) if lo > 0 else hi / 1e6
                lo, hi = (t, hi) if np.linalg.cond(np.eye(n) + t * N) < 1e10 else (lo, t)
            Lo[b:b + n, b:b + n] = hi * N
    return np.triu(U) + np.tril(Lo, -1)


@pytest.mark.parametrize("nb", NBS)
@pytest.mark.parametrize("kind", ["well", "graded", "ill"])
def test_diag_inverse_componentwise_bound(nb, kind):
    rng = np.random.default_rng(nb * 7 + len(kind))
    for nblk in (1, 2, 3, 4):
        v = nb * nblk
        A00 = _triangles(v, kind, rng, nb)
        Uinv, LinvT = cb.dbg.diag_inverse(A00, nb)
        assert Uinv.shape == (nblk, nb, nb)
        for j in range(nblk):
            blk = A00[j * nb:(j + 1) * nb, j * nb:(j + 1) * nb]
            U, L = np.triu(blk), np.tril(blk, -1) + np.eye(nb)
            assert hp.inverse_componentwise_ok(U, Uinv[j]), (v, j)
            assert hp.inverse_componentwise_ok(L, LinvT[j].T), (v, j)
            assert nb == 4 or not hp.inverse_componentwise_ok(U, Uinv[j].T)   # the check sees the kernel's output


@pytest.mark.parametrize("nb", NBS)
def test_diag_inverse_reads_only_its_blocks_and_not_the_unit_diagonal(nb):
    rng = np.random.default_rng(100 + nb)
    v = 3 * nb
    A00 = _triangles(v, "well", rng, nb)
    Uinv, LinvT = cb.dbg.diag_inverse(A00, nb)
    outside = np.ones((v, v), dtype=bool)
    for j in range(3):
        outside[j * nb:(j + 1) * nb, j * nb:(j + 1) * nb] = False
    An = A00.copy()
    An[outside] = np.nan
    Un, Ln = cb.dbg.diag_inverse(An, nb)
    assert np.array_equal(Un, Uinv) and np.array_equal(Ln, LinvT)
    Ad = A00.copy()
    Ad[np.diag_indices(v)] *= 3.0
    _, Ld = cb.dbg.diag_inverse(Ad, nb)
    assert np.array_equal(Ld, LinvT)


# ----------------------------------------------------------------------------------------------- one diagonal tile
TILE_V = [4, 12, 16, 36, 48, 100, 160, 224, 480]


def _tile_cases(v):
    return [(v, 0)] + ([(v, 1)] if v == 128 else [])


@pytest.mark.parametrize("v,variant", [c for v in TILE_V + [128] for c in _tile_cases(v)])
@pytest.mark.parametrize("kind", ["k1e2", "k1e8", "graded"])
def test_potrf_kernels_componentwise_bound(v, variant, kind):
    rng = np.random.default_rng(v * 3 + variant)
    A = _spd(kind, v, rng)
    L, LT, info = cb.dbg.potrf_tile(A, variant)
    assert info == 0
    assert np.array_equal(LT, L.T) and not np.triu(L, 1).any()
    res = hp.chol_residual(A, L)
    assert hp.chol_componentwise_ok(A, L, res)
    assert v == 4 or not hp.chol_componentwise_ok(A, L.T)        # the check sees the kernel's output


@pytest.mark.parametrize("v,variant", [c for v in TILE_V + [128] for c in _tile_cases(v)])
def test_potrf_kernels_exact_input_and_unread_upper_triangle(v, variant):
    rng = np.random.default_rng(1000 + v)
    A, L0 = hp.exact_spd(v, rng)
    L, _, info = cb.dbg.potrf_tile(A, variant)
    assert info == 0 and np.array_equal(L, L0)                  # every operation is exact: L bit for bit
    S = _spd("k1e2", v, rng)
    Az, An = np.tril(S), np.tril(S)
    An[np.triu_indices(v, 1)] = np.nan                          # LAPACK uplo='L': the upper triangle is not read
    Lz, LTz, _ = cb.dbg.potrf_tile(Az, variant)
    Ln, LTn, _ = cb.dbg.potrf_tile(An, variant)
    assert np.array_equal(Ln, Lz) and np.array_equal(LTn, LTz)


@pytest.mark.parametrize("v", [256, 384, 512])
@pytest.mark.parametrize("kind", ["k1e2", "k1e8", "graded", "exact_wellcond"])
def test_blocked_tile_path_kappa_bound(v, kind):
    rng = np.random.default_rng(v + len(kind))
    A = _spd(kind, v, rng)
    L, LT, info = cb.dbg.potrf_tile(A, 2)
    assert info == 0 and np.array_equal(LT, L.T) and not np.triu(L, 1).any()
    kmax = hp.diag_block_kappa(L, 128)
    res = hp.chol_residual(A, L)
    assert hp.chol_normwise_ok(A, L, kmax, res)
    assert not hp.chol_normwise_ok(A, L.T, kmax)
    if kind in ("k1e2", "k1e8"):
        Lref, _ = hp.cholesky(A)
        assert hp.chol_forward_ok(A, L, Lref, kmax, res)
    An = np.tril(A)
    An[np.triu_indices(v, 1)] = np.nan
    assert np.array_equal(cb.dbg.potrf_tile(An, 2)[0], cb.dbg.potrf_tile(np.tril(A), 2)[0])


@pytest.mark.parametrize("v,variant,k0", [(48, 0, 0), (48, 0, 40), (100, 0, 77), (128, 1, 5), (128, 1, 127), (256, 2, 3),
                                          (256, 2, 200), (384, 2, 131), (512, 2, 511)])
def test_potrf_tile_reports_the_first_failing_column(v, variant, k0):
    rng = np.random.default_rng(v + k0)
    L0 = np.linalg.cholesky(hp.random_spd(v, 1e2, rng))
    A = L0 @ L0.T
    A[k0, k0] -= L0[k0, k0] ** 2 + 0.25                       # pivot k0 becomes -0.25
    assert scipy.linalg.lapack.dpotrf(A, lower=1)[1] == k0 + 1
    assert cb.dbg.potrf_tile(A, variant)[2] == k0 + 1


# ----------------------------------------------------------------------------------------------- whole factorisation
def _factor(A, v, want_resid=False, n_runs=1):
    N = A.shape[0]
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    assert (ch.Ml, ch.Nl) == (N, N)
    ch.data[...] = A
    out = []
    for _ in range(n_runs):
        ch.parallelCholesky()
        out.append(np.tril(ch.local_factor()))
    resid = [ch.validate(), ch.validate()] if want_resid else None
    ch.finalize()
    comm.close()
    return out, resid


E2E = [(1152, 384), (480, 48), (800, 100), (1120, 160), (2048, 256)]


@pytest.mark.parametrize("N,v", E2E)
def test_factor_against_longdouble(N, v):
    rng = np.random.default_rng(N + v)
    for kind in ("k1e2", "k1e8"):
        A = _spd(kind, N, rng)
        (L, L2), resid = _factor(A, v, want_resid=True, n_runs=2)
        assert np.array_equal(L, L2), "two factorisations differ"
        assert resid[0] == resid[1], "two validations of the same factor differ"
        kmax = _kappa_max(L, v)
        res = hp.chol_residual(A, L)
        assert hp.chol_normwise_ok(A, L, kmax, res), kind
        Lref, info = hp.cholesky(A)
        assert info == 0 and hp.chol_forward_ok(A, L, Lref, kmax, res), kind
        R = res[0]
        host = float(np.sqrt(np.sum(R * R))) / float(np.linalg.norm(np.tril(A)))
        assert host / 10 <= resid[0][1] <= host * 10, (resid[0], host)
        if kind == "k1e2":                                     # the upper triangle is never read
            An = A.copy()
            An[np.triu_indices(N, 1)] = np.nan
            assert np.array_equal(_factor(An, v)[0][0], L)


@pytest.mark.parametrize("N,v", E2E)
def test_factor_graded_matrix_rowwise(N, v):
    """A = D S D with D = diag(2^-10 .. 2^10): L(A) = D L(S).  Scaling by powers of two commutes with every rounding
    (sqrt(d^2 x) = d sqrt(x) for d = 2^k, and every sum the algorithm forms adds terms of one common scale), so the
    default path must return D times the factor of S bit for bit, row by row.  The graded factor also meets the normwise
    bound on its own."""
    rng = np.random.default_rng(7 * N + v)
    d = 2.0 ** np.round(np.linspace(-10, 10, N))
    S = hp.random_spd(N, 1e2, rng)
    A = d[:, None] * S * d[None, :]
    (L,), _ = _factor(A, v)
    (LS,), _ = _factor(S, v)
    assert np.array_equal(L, d[:, None] * LS)
    assert hp.chol_normwise_ok(A, L, _kappa_max(L, v))


@pytest.mark.parametrize("update,kind,N,v",
                         [(u,) + c for u in make_chol_golden.UPDATES for c in make_chol_golden.update_cases(u)])
def test_default_path_factor_bits_are_pinned(update, kind, N, v, golden_dir):
    """the factor and the launch count of one factorisation of each trailing-update kind are those recorded in
    tests/golden/chol_factor_bits.json (the default FP64 update) and update_factor_bits.json (int8, TF32, TF32x3), by
    tests/golden/make_chol_golden.py"""
    want = make_chol_golden.golden(update, golden_dir)[f"{kind}_{N}_{v}"]
    assert make_chol_golden.factor_bits(kind, N, v, update) == want


@pytest.mark.parametrize("v", [128, 256, 512])
def test_factor_ozaki_update(v, monkeypatch):
    N = 4 * v
    rng = np.random.default_rng(v)
    A = _spd("k1e2", N, rng)
    (Ld,), _ = _factor(A, v)
    monkeypatch.setenv("CFLX_GEMM", "ozaki")                   # read when the object is created
    (L, L2), resid = _factor(A, v, want_resid=True, n_runs=2)
    assert np.array_equal(L, L2) and resid[0] == resid[1]
    assert not np.array_equal(L, Ld), "CFLX_GEMM=ozaki did not change the update path"
    kmax = _kappa_max(L, v)
    res = hp.chol_residual(A, L)
    Lref, _ = hp.cholesky(A)
    assert hp.chol_normwise_ok(A, L, kmax, res) and hp.chol_forward_ok(A, L, Lref, kmax, res)
    assert hp.chol_forward_ok(A, Ld, Lref, kmax)


# ----------------------------------------------------------------------------------------------- not positive definite
def _not_pd(N, k0, rng):
    L0 = np.linalg.cholesky(hp.random_spd(N, 1e2, rng))
    A = L0 @ L0.T
    A[k0, k0] -= L0[k0, k0] ** 2 + 0.25
    return A


@pytest.mark.parametrize("N,v,k0", [(480, 48, 7), (480, 48, 250), (480, 48, 470), (768, 256, 10), (768, 256, 300),
                                    (768, 256, 700), (768, 256, 140), (1152, 384, 384 + 130)])
def test_not_positive_definite_names_lapacks_column(N, v, k0):
    rng = np.random.default_rng(N + k0)
    A = _not_pd(N, k0, rng)
    assert scipy.linalg.lapack.dpotrf(A, lower=1)[1] == k0 + 1
    S = _spd("k1e2", N, rng)
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    ch.data[...] = A
    with pytest.raises(cb.ConfluxError, match="positive definite") as e:
        ch.parallelCholesky()
    assert int(re.search(r"column (\d+)", str(e.value)).group(1)) == k0 + 1
    ch.data[...] = S                                          # the object is usable again, with nothing left over
    ch.parallelCholesky()
    L = np.tril(ch.local_factor())
    ch.finalize()
    comm.close()
    assert np.array_equal(L, _factor(S, v)[0][0])


@pytest.mark.parametrize("grid,k0", [((2, 1, 1), 200), ((2, 2, 1), 130), ((1, 1, 2), 40)])
def test_not_positive_definite_same_error_on_every_rank(grid, k0):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 512, 64
    A = _not_pd(N, k0, np.random.default_rng(k0))

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = 0.0
        if ch.pz == 0:
            for lti in range(ch.Ml // v):
                for ltj in range(ch.Nl // v):
                    gi, gj = lti * ch.PX + ch.px, ltj * ch.PY + ch.py
                    if gi < ch.Kappa and gj < ch.Kappa:
                        ch.data[lti * v:(lti + 1) * v, ltj * v:(ltj + 1) * v] = A[gi * v:(gi + 1) * v, gj * v:(gj + 1) * v]
        try:
            ch.parallelCholesky()
            msg = None
        except cb.ConfluxError as e:
            msg = str(e)
        ch.finalize()
        return msg

    msgs = run_ranks(P, body)
    assert all(m is not None and m == msgs[0] for m in msgs), msgs
    assert int(re.search(r"column (\d+)", msgs[0]).group(1)) == k0 + 1
