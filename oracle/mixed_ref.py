"""oracle/mixed_ref.py -- TEST INFRASTRUCTURE: CPU restatement of the mixed-precision drivers (cflx_lu_sv_mixed /
cflx_chol_sv_mixed, conflux_b200/csrc/tf32.cu and refine.cu mixed_run).
  * split(): the per-row power-of-two scale and the TF32 terms, bit for bit: s = x 2^-e with e from frexp of the row's
    largest magnitude, hi = rna(fp32(s)), lo = rna(fp32(s - hi)), where rna is cvt.rna.tf32.f32's rounding on the FP32
    bits (10 explicit mantissa bits, ties away from zero); the K tail zero up to KP = K rounded up to 8;
  * gemm(): D_ref = C - the kept products of the split terms (each TF32 x TF32 product is exact in float64), and the
    bound the kernel's FP32 accumulation must meet: |D - D_ref| <= (K + 2) 2^-23 |A_s| |B_s|, scaled by 2^(ea + eb),
    plus FP32 underflow and the rounding of the final FP64 subtraction.  The order of the FP32 additions is not restated;
  * sv_mixed(): LAPACK dsgesv's control flow with an injectable low-precision factorisation and solve."""
import numpy as np

ITMAX = 30
NO_CONVERGENCE = -31
LOW_PREC_FAILED = -3


def rna_tf32(f):
    """cvt.rna.tf32.f32 on float32 values (finite): round to 10 explicit mantissa bits, ties away from zero"""
    u = np.ascontiguousarray(f, dtype=np.float32).view(np.uint32)
    mag = ((u & np.uint32(0x7FFFFFFF)) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return ((u & np.uint32(0x80000000)) | mag).astype(np.uint32).view(np.float32)


def split(S, terms):
    """S: (K, n) K-major operand as the kernel reads it (S[k, o]).  Returns (hi, lo, e): hi, lo float32 (n, KP) (lo None
    for one term), e int32 (n,) with every row's largest magnitude times 2^-e in [0.5, 1) (0 for a zero row)."""
    S = np.asarray(S, dtype=np.float64)
    K, n = S.shape
    KP = -(-K // 8) * 8
    mx = np.abs(S).max(axis=0) if K else np.zeros(n)
    e = np.where(mx > 0, np.frexp(mx)[1], 0).astype(np.int32)
    s = np.ldexp(S.T, -e[:, None].astype(np.int64))
    h = rna_tf32(s.astype(np.float32))
    hi = np.zeros((n, KP), np.float32)
    hi[:, :K] = h
    lo = None
    if terms == 3:
        lo = np.zeros((n, KP), np.float32)
        lo[:, :K] = rna_tf32((s - h.astype(np.float64)).astype(np.float32))
    return hi, lo, e


def gemm(AT, B, C, terms, row0=0, col0=0):
    """D = C - A B on the split terms of AT (K, row0 + M) and B (K, col0 + N), rows row0.. / columns col0.. of the
    window.  Returns (D_ref, bound, parts) with parts = (hiA, loA, ea, hiB, loB, eb) as split() gives them."""
    hA, lA, ea = split(AT, terms)
    hB, lB, eb = split(B, terms)
    a, b = slice(row0, None), slice(col0, None)
    Ah, Bh = hA[a].astype(np.float64), hB[b].astype(np.float64)
    P = Ah @ Bh.T
    mag = np.abs(Ah) @ np.abs(Bh).T
    if terms == 3:
        Al, Bl = lA[a].astype(np.float64), lB[b].astype(np.float64)
        P = P + Ah @ Bl.T + Al @ Bh.T
        mag = mag + np.abs(Ah) @ np.abs(Bl).T + np.abs(Al) @ np.abs(Bh).T
    scale = np.ldexp(1.0, (ea[a][:, None] + eb[b][None, :]).astype(np.int64))
    K = AT.shape[0]
    prod = P * scale
    C = np.zeros_like(prod) if C is None else np.asarray(C, dtype=np.float64)
    D = C - prod
    # every term is below 1 in magnitude: products the tensor cores flush below FP32's normal range add K 2^-125
    bound = ((K + 2) * 2.0 ** -23 * mag + K * 2.0 ** -125) * scale + 4 * 2.0 ** -53 * (np.abs(C) + np.abs(prod)) + 1e-300
    return D, bound, (hA, lA, ea, hB, lB, eb)


def sv_mixed(A, B, factor_low, solve_low, solve64=None, itmax=0, eps=2.0 ** -53):
    """dsgesv's loop: F = factor_low(A) (None: a zero or non-positive pivot), x = solve_low(F, b), then while some
    column has ||r||_inf > ||x||_inf ||A||_inf eps sqrt(n): x += solve_low(F, r), at most itmax (<= 0: 30) times.
    Returns (X, iter, berr): iter the corrections taken, -3 (factor failed) or -31 (not converged, or a norm not
    finite), in which case X = solve64(A, B) (default numpy.linalg.solve); berr = ||r|| / (||A|| ||x||) per column."""
    A = np.asarray(A, dtype=np.float64)
    B2 = np.asarray(B, dtype=np.float64).reshape(A.shape[0], -1)
    n = A.shape[0]
    itmax = itmax if itmax > 0 else ITMAX
    solve64 = solve64 or np.linalg.solve
    anrm = np.abs(A).sum(axis=1).max()
    cte = anrm * eps * np.sqrt(n)

    def norms(X):
        R = B2 - A @ X
        xn, rn = np.abs(X).max(axis=0), np.abs(R).max(axis=0)
        return R, xn, rn

    F = factor_low(A)
    it = LOW_PREC_FAILED
    if F is not None:
        X = solve_low(F, B2)
        R, xn, rn = norms(X)
        k = 0
        while True:
            if np.all(rn <= xn * cte):
                it = k
                break
            if not (np.all(np.isfinite(xn)) and np.all(np.isfinite(rn))) or k == itmax:
                it = NO_CONVERGENCE
                break
            X = X + solve_low(F, R)
            k += 1
            R, xn, rn = norms(X)
    if it < 0:
        X = solve64(A, B2)
        R, xn, rn = norms(X)
    return X, it, rn / (anrm * xn)
