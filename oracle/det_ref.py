"""oracle/det_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_det and cflx_chol_det
(conflux_b200/csrc/det.cu, with the diagonal gather of equil.cu).

The specification of the determinant, checkable without GPUs:
  * product(): the device's exact-range product, bit for bit.  A value x is the pair (m, e) = frexp(|x|); a (x) b takes
    (f, k) = frexp(m_a m_b) and gives (f, e_a + e_b + k); a (/) b the same with m_a / m_b.  Thread t of DET_THREADS folds
    its chunk [t c, min(n, (t + 1) c)), c = ceil(n / DET_THREADS), left to right from (0.5, 1), skipping zero and
    non-finite entries; then slot t (x)= slot t + w for w = DET_THREADS / 2 .. 1.  The divisors are reduced alike;
    square squares every product; the result is D (/) S1 (/) S2.  With the first zero and the first bad entry (not finite
    in d; not finite or zero in a divisor) the result is (NaN, 0) when the bad entry comes first, else (0, 0).
  * perm_parity(): det(P) of the permutation with row q of P A = row perm[q] of A, by cycle decomposition.
  * gather_diag(): the diagonal of the layer-0 shares, rank by rank as the device gathers it (only the diagonal entries
    of the real diagonal tiles a share holds are read; the world sum has one contributor per element).
  * lu_det() / chol_det(): what cflx_lu_det / cflx_chol_det return for those shares."""
import math

import numpy as np

from . import chol_ref, layout

DET_THREADS = 256
LN2 = 0.69314718055994530942


def _norm(p, e):
    f, k = math.frexp(p)
    return (f, e + k)


def mul(a, b):
    return _norm(a[0] * b[0], a[1] + b[1])


def div(a, b):
    return _norm(a[0] / b[0], a[1] - b[1])


def product(d, s1=None, s2=None, square=False, threads=DET_THREADS):
    """dict(mant, exp, neg, first_zero, nonfinite) of the device's product kernel (cflx_dbg_det)"""
    vs = [[float(x) for x in np.asarray(v, dtype=np.float64)] if v is not None else None for v in (d, s1, s2)]
    n = len(vs[0])
    c = -(-n // threads)
    slots = []
    for t in range(threads):
        p = [(0.5, 1)] * 3
        neg, zero, bad = 0, n, n
        for i in range(t * c, min(n, (t + 1) * c)):
            for q in range(3):
                if vs[q] is None:
                    continue
                x = vs[q][i]
                neg += x < 0.0
                if q == 0 and x == 0.0:
                    zero = min(zero, i)
                elif not math.isfinite(x) or x == 0.0:
                    bad = min(bad, i)
                else:
                    p[q] = mul(p[q], math.frexp(abs(x)))
        slots.append([p, neg, zero, bad])
    w = threads // 2
    while w:
        for t in range(w):
            x, y = slots[t], slots[t + w]
            x[0] = [mul(x[0][q], y[0][q]) for q in range(3)]
            x[1] += y[1]
            x[2] = min(x[2], y[2])
            x[3] = min(x[3], y[3])
        w //= 2
    p, neg, zero, bad = slots[0]
    if square:
        p = [mul(a, a) for a in p]
    r = p[0]
    if s1 is not None:
        r = div(r, p[1])
    if s2 is not None:
        r = div(r, p[2])
    nonfinite = bad < zero
    if nonfinite:
        r = (math.nan, 0)
    elif zero < n:
        r = (0.0, 0)
    return dict(mant=r[0], exp=r[1], neg=0 if square else neg & 1, first_zero=zero + 1 if zero < n else 0,
                nonfinite=int(nonfinite))


def logabs(mant, exp):
    """log |det| of the pair, as the library forms it on the host"""
    if math.isnan(mant):
        return math.nan
    if mant == 0.0:
        return -math.inf
    return math.log(mant) + exp * LN2


def perm_parity(perm):
    """0 when the permutation is even, 1 when odd: M minus its number of cycles, mod 2"""
    perm = [int(x) for x in perm]
    seen = [False] * len(perm)
    odd = 0
    for i in range(len(perm)):
        j = i
        while not seen[j]:
            seen[j] = True
            odd ^= j != i
            j = perm[j]
    return odd


def gather_diag(shares, v, Px, Py, Pz, Nt, M):
    """the world sum of every rank's M-vector: a_gg where the rank (layer 0) holds the diagonal tile g // v < Nt, zeros
    elsewhere.  shares: every rank's Ml x Nl array, in rank order; only those diagonal entries are read."""
    d = np.zeros(M)
    for r, A in enumerate(shares):
        pi, pj, pk = r // (Py * Pz), (r // Pz) % Py, r % Pz
        part = np.zeros(M)
        if pk == 0:
            Ml, Nl = A.shape
            for t in range(min(Nt, M // v)):
                lr, lc = (t // Px) * v, (t // Py) * v
                if t % Px == pi and t % Py == pj and lr < Ml and lc < Nl:
                    for e in range(v):
                        part[t * v + e] = A[lr + e, lc + e]
        d += part
    return d


def _out(p, sign=None):
    o = dict(mantissa=p["mant"], exponent=p["exp"], logabsdet=logabs(p["mant"], p["exp"]))
    if sign is not None:
        o["sign"] = sign
    return o


def lu_det(C_shares, perm, N, v, Px=1, Py=1, Pz=1, r=None, c=None):
    """cflx_lu_det on every rank's share of L\\U (cflx_lu_get_factors) and the permutation: dict(sign, logabsdet,
    mantissa, exponent, info).  r / c: the scales to divide by (unscaled = 1), or None."""
    dm = layout.dims(N, v, Px, Py, Pz)
    d = gather_diag(C_shares, v, Px, Py, Pz, dm["Nt"], dm["M"])
    p = product(d, r, c)
    if p["nonfinite"]:
        sign = math.nan
    elif p["first_zero"]:
        sign = 0.0
    else:
        sign = -1.0 if (p["neg"] ^ perm_parity(perm)) else 1.0
    o = _out(p, sign)
    o["info"] = p["first_zero"]
    return o


def chol_det(L_shares, N, v, Px=1, Py=1, Pz=1, s=None):
    """cflx_chol_det on every rank's share of L (cflx_chol_get_local): dict(logabsdet, mantissa, exponent).  s: the scale
    to divide by squared (unscaled = 1), or None."""
    dm = chol_ref.dims(N, v, Px, Py, Pz)
    d = gather_diag(L_shares, v, Px, Py, Pz, dm["Kappa"], dm["N"])
    return _out(product(d, s, None, square=True))
