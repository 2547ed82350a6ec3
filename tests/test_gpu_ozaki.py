"""GPU: the int8 wgmma trailing update (conflux_b200/csrc/ozaki.cu) in isolation, through the C ABI.
  * the digit planes and exponents equal the numpy restatement exactly;
  * the result equals the restatement BIT FOR BIT (all plane products are exact integers and the FP64 recombination is
    reproduced in the kernel's order) -- this pins the TMA / wgmma descriptor / accumulator layout logic;
  * the result agrees with a plain FP64 product to rounding level (what cblas_dgemm gives the reference)."""
import numpy as np
import pytest

import conflux_b200 as cb
from oracle import ozaki_ref

pytestmark = pytest.mark.gpu


def _case(M, N, K, seed, kind="lu"):
    rng = np.random.default_rng(seed)
    if kind == "lu":            # what the trailing update sees: |l| <= 1 multipliers, U rows of mixed magnitude
        AT = rng.uniform(-1, 1, (K, M)) * rng.choice([1.0, 1e-3, 1e-7], size=(K, M))
        B = rng.standard_normal((K, N)) * 6.0
    elif kind == "ints":        # small integers: every plane but the first two is zero, sums are exact in FP64 too
        AT = rng.integers(-8, 9, (K, M)).astype(np.float64)
        B = rng.integers(-8, 9, (K, N)).astype(np.float64)
    else:                       # wide dynamic range + zero rows / columns
        AT = rng.standard_normal((K, M)) * np.exp2(rng.integers(-30, 30, (1, M)).astype(np.float64))
        B = rng.standard_normal((K, N)) * np.exp2(rng.integers(-30, 30, (1, N)).astype(np.float64))
        AT[:, ::7] = 0.0
        B[:, 1::5] = 0.0
    C = rng.standard_normal((M, N))
    return AT, B, C


@pytest.mark.parametrize("M,N,K,kind", [(128, 64, 128, "ints"), (128, 64, 128, "lu"), (256, 128, 256, "lu"),
                                        (200, 130, 128, "lu"), (129, 66, 384, "wide"), (1000, 514, 512, "lu"),
                                        (37, 2, 128, "wide"), (1536, 1024, 256, "lu")])
def test_ozaki_gemm_bit_exact_vs_restatement(M, N, K, kind):
    AT, B, C = _case(M, N, K, M + 3 * N + K, kind)
    r = cb.dbg.ozaki_gemm(AT, B, C, want_planes=True)
    ref, (pa, pb, ea, eb) = ozaki_ref.gemm(AT, B, C)
    assert np.array_equal(r["ea"], ea) and np.array_equal(r["eb"], eb)
    assert np.array_equal(r["pa"], pa) and np.array_equal(r["pb"], pb)
    assert np.array_equal(r["D"], ref), (np.abs(r["D"] - ref).max(), np.argwhere(r["D"] != ref)[:5])
    if kind == "ints":
        assert np.array_equal(r["D"], C - AT.T @ B)            # exact in both arithmetics
    # against plain FP64: error below K * 2^-52 of |row max| * |column max| (the scheme's bound, see ozaki.cu)
    plain = C - AT.T @ B
    bound = K * 2.0 ** -50 * np.abs(AT).max(axis=0)[:, None] * np.abs(B).max(axis=0)[None, :] + 1e-300
    assert np.all(np.abs(r["D"] - plain) <= bound + 4 * np.finfo(float).eps * np.abs(plain))


def test_ozaki_gemm_speed_probe():
    """Not a correctness test: prints the kernel time at the first-step shape of BASELINE config C2."""
    M = N = 16128
    K = 256
    rng = np.random.default_rng(1)
    AT = rng.uniform(-1, 1, (K, M))
    B = rng.standard_normal((K, N))
    r = cb.dbg.ozaki_gemm(AT, B, None, reps=3)
    tf = 2.0 * M * N * K / (r["ms"] * 1e-3) / 1e12
    print(f"ozaki int8 wgmma trailing update {M}x{N}x{K}: {r['ms']:.3f} ms = {tf:.1f} TFLOP/s FP64-equivalent, "
          f"digit planes {r['split_ms']:.3f} ms")
    _, dm = cb.dbg.gemm_tn(AT, B, None, -1.0, 0.0, reps=3)
    print(f"DMMA kernel same shape: {dm:.3f} ms = {2.0 * M * N * K / (dm * 1e-3) / 1e12:.1f} TFLOP/s")
    assert r["ms"] > 0
