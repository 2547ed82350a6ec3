"""CPU: the restatement of the mixed-precision drivers (oracle/mixed_ref.py) -- the TF32 split, its rounding and
exponent range, the product bound, and dsgesv's control flow on hand-built cases (scipy has no dsgesv / dsposv)."""
import numpy as np
import pytest

from oracle import mixed_ref


def test_rna_ties_round_away_from_zero():
    one = np.float32(1.0)
    ulp = np.float32(2.0 ** -10)          # TF32 spacing at 1
    half = np.float32(2.0 ** -11)
    x = np.array([one + half, one + ulp + half, -(one + half), -(one + ulp + half), one + half * np.float32(0.999)],
                 np.float32)
    r = mixed_ref.rna_tf32(x)
    assert r[0] == one + ulp and r[1] == one + 2 * ulp          # ties: away from zero, whatever the last bit
    assert r[2] == -(one + ulp) and r[3] == -(one + 2 * ulp)
    assert r[4] == one                                           # below the tie: nearest
    assert np.all(mixed_ref.rna_tf32(r) == r)                    # idempotent
    assert np.all((r.view(np.uint32) & 0x1FFF) == 0)             # 10 explicit mantissa bits


@pytest.mark.parametrize("K", [1, 4, 12, 64, 200])
def test_hi_lo_reconstruct_to_2_pow_minus_22(K):
    rng = np.random.default_rng(K)
    S = rng.standard_normal((K, 50)) * np.exp2(rng.integers(-20, 20, (K, 50)))
    hi, lo, e = mixed_ref.split(S, 3)
    KP = -(-K // 8) * 8
    assert hi.shape == (50, KP) and np.all(hi[:, K:] == 0) and np.all(lo[:, K:] == 0)
    s = np.ldexp(S.T, -e[:, None].astype(np.int64))
    assert np.all(np.abs(s) < 1.0) and np.all(np.abs(s).max(axis=1) >= 0.5)
    tiny = np.abs(s) < 2.0 ** -100                                # FP32 subnormal range of the scaled entries
    rec = hi[:, :K].astype(np.float64) + lo[:, :K].astype(np.float64)
    assert np.all(np.abs(rec - s)[~tiny] <= 2.0 ** -22 * np.abs(s)[~tiny])
    h1, l1, e1 = mixed_ref.split(S, 1)
    assert l1 is None and np.array_equal(h1, hi) and np.array_equal(e1, e)
    assert np.all(np.abs(hi[:, :K] - s)[~tiny] <= 2.0 ** -11 * np.abs(s)[~tiny])


def test_exponent_extremes_and_zero_rows():
    rng = np.random.default_rng(1)
    S = rng.uniform(0.5, 1.0, (16, 5)) * np.array([2.0 ** 1000, 2.0 ** -1000, 0.0, 2.0 ** -1060, 1.0])
    hi, lo, e = mixed_ref.split(S, 3)
    assert e.tolist()[:3] == [1000, -1000, 0] and e[4] == 0
    assert e[3] == np.frexp(np.abs(S[:, 3]).max())[1]            # a subnormal row gets its own exponent
    assert np.all(hi[2] == 0) and np.all(lo[2] == 0)
    back = np.ldexp(hi[:, :16].astype(np.float64) + lo[:, :16].astype(np.float64), e[:, None].astype(np.int64)).T
    nz = S != 0
    assert np.all(np.abs(back - S)[nz] <= 2.0 ** -22 * np.abs(S)[nz])


def test_product_bound_accepts_float64_and_separates_terms():
    rng = np.random.default_rng(2)
    K, M, N = 256, 40, 30
    AT, B, C = rng.standard_normal((K, M)), rng.standard_normal((K, N)), rng.standard_normal((M, N))
    exact = C - AT.T @ B
    err = {}
    for t in (1, 3):
        D, bound, _ = mixed_ref.gemm(AT, B, C, t)
        # the split products in float32 accumulation stay inside the bound
        hA, lA, ea, hB, lB, eb = mixed_ref.split(AT, t) + mixed_ref.split(B, t)
        P = hA.astype(np.float32) @ hB.astype(np.float32).T
        if t == 3:
            P = P + (hA.astype(np.float32) @ lB.astype(np.float32).T + lA.astype(np.float32) @ hB.astype(np.float32).T)
        D32 = C - P.astype(np.float64) * np.ldexp(1.0, (ea[:, None] + eb[None, :]).astype(np.int64))
        assert np.all(np.abs(D32 - D) <= bound)
        err[t] = np.abs(D - exact).max() / np.abs(AT).max() / np.abs(B).max() / K
    assert err[3] < err[1] / 500


def _lu_low(A, rel):
    """a low-precision factorisation stand-in: the LU of A perturbed by `rel` relative, as numpy's solve"""
    rng = np.random.default_rng(7)
    F = A * (1 + rel * rng.uniform(-1, 1, A.shape))
    return F


def _solve(F, R):
    return np.linalg.solve(F, R)


def test_loop_converges_on_a_dominant_matrix():
    rng = np.random.default_rng(3)
    n = 120
    A = rng.standard_normal((n, n)) + n * np.eye(n)
    B = rng.standard_normal((n, 3))
    X, it, berr = mixed_ref.sv_mixed(A, B, lambda A: _lu_low(A, 2.0 ** -11), _solve)
    assert 1 <= it <= 5
    assert np.all(berr <= np.sqrt(n) * 2.0 ** -53)
    X0, it0, _ = mixed_ref.sv_mixed(A, B, lambda A: A, _solve)     # an exact factorisation converges at once
    assert it0 in (0, 1)


def test_loop_gives_up_on_an_ill_conditioned_matrix():
    rng = np.random.default_rng(4)
    n = 80
    Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
    Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = Q1 @ np.diag(np.logspace(0, -12, n)) @ Q2.T               # kappa = 1e12
    B = rng.standard_normal((n, 2))
    calls = []
    X, it, berr = mixed_ref.sv_mixed(A, B, lambda A: _lu_low(A, 2.0 ** -11), _solve,
                                     solve64=lambda A, B: calls.append(1) or np.linalg.solve(A, B), itmax=10)
    assert it == mixed_ref.NO_CONVERGENCE and calls == [1]
    assert np.array_equal(X, np.linalg.solve(A, B))


def test_loop_falls_back_on_a_failed_factorisation():
    rng = np.random.default_rng(5)
    A = rng.standard_normal((30, 30)) + 30 * np.eye(30)
    B = rng.standard_normal(30)
    X, it, berr = mixed_ref.sv_mixed(A, B, lambda A: None, _solve)
    assert it == mixed_ref.LOW_PREC_FAILED
    assert np.array_equal(X, np.linalg.solve(A, B.reshape(30, 1)))


def test_loop_stops_on_non_finite_norms():
    A = np.eye(4) * 2.0
    B = np.ones(4)
    X, it, _ = mixed_ref.sv_mixed(A, B, lambda A: A, lambda F, R: np.full_like(R, np.nan))
    assert it == mixed_ref.NO_CONVERGENCE and np.all(X == 0.5)
