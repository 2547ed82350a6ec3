"""tools/ozaki_study.py -- CPU feasibility study for the round-2 item "FP64 trailing update on the int8 tensor cores".

Emulates, in numpy with exact integer arithmetic, an Ozaki-style error-free-slicing DGEMM
    C -= L * U,   L = sum_p 2^(eL_i - 7p) Lp,  U = sum_q 2^(eU_j - 7q) Uq,   Lp, Uq int8 slices (7 magnitude bits),
where row i of L and column j of U share one exponent each, every slice product Lp*Uq is an exact int8 x int8 -> int32
GEMM (what an int8 tensor-core MMA computes), and only the products with p + q <= s + 1 are formed.  It then runs the
blocked right-looking LU (partial pivoting inside each panel, exactly the P = 1 data flow of this repo) with that GEMM as
the trailing update and reports ||PA - LU||_F / ||A||_F against the number of slices s, on the bench's generator.

    python tools/ozaki_study.py [N] [v]
"""
import sys
import numpy as np


def slices(X, axis, s):
    """Split X into s int8 slices sharing one exponent per row (axis=1) / column (axis=0). Returns (slices, exp)."""
    mx = np.max(np.abs(X), axis=axis, keepdims=True)
    e = np.where(mx > 0, np.ceil(np.log2(np.where(mx > 0, mx, 1.0))) + 1, 0.0)   # |X| * 2^-e < 1/2... < 1
    R = X * np.exp2(-e)                                                          # |R| < 1
    out = []
    for _ in range(s):
        R = R * 128.0                      # next 7 bits
        S = np.rint(R)                     # in [-128, 128]; clip to int8 range keeps it exact enough (|S| <= 127 after rint of <128)
        S = np.clip(S, -127, 127)
        R = R - S
        out.append(S)                  # integers held in float64: products and k-sums (<= 127^2 k) stay exact
    return out, e


def ozaki_gemm(L, U, s):
    Ls, eL = slices(L, 1, s)
    Us, eU = slices(U, 0, s)
    acc = np.zeros((L.shape[0], U.shape[1]))
    nprod = 0
    for p in range(s):
        for q in range(s):
            if p + q <= s - 1:             # 0-based: keep the s(s+1)/2 leading products
                acc += (Ls[p] @ Us[q]).astype(np.float64) * 2.0 ** (-7.0 * (p + q + 2))
                nprod += 1
    return acc * np.exp2(eL) * np.exp2(eU), nprod


def blocked_lu(A, v, gemm):
    A = A.copy()
    n = A.shape[0]
    perm = np.arange(n)
    for k in range(0, n, v):
        for j in range(k, k + v):          # panel: partial pivoting
            p = j + int(np.argmax(np.abs(A[j:, j])))
            if p != j:
                A[[j, p]] = A[[p, j]]
                perm[[j, p]] = perm[[p, j]]
            A[j + 1:, j] /= A[j, j]
            A[j + 1:, j + 1:k + v] -= np.outer(A[j + 1:, j], A[j, j + 1:k + v])
        if k + v < n:
            L00 = np.tril(A[k:k + v, k:k + v], -1) + np.eye(v)
            A[k:k + v, k + v:] = np.linalg.solve(L00, A[k:k + v, k + v:])
            A[k + v:, k + v:] -= gemm(A[k + v:, k:k + v], A[k:k + v, k + v:])
    return A, perm


def residual(A, LU, perm):
    L = np.tril(LU, -1) + np.eye(A.shape[0])
    return np.linalg.norm(A[perm] - L @ np.triu(LU)) / np.linalg.norm(A)


if __name__ == "__main__":
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    v = int(sys.argv[2]) if len(sys.argv) > 2 else 128
    sys.path.insert(0, __file__.rsplit("/", 2)[0])
    from oracle import restate
    A = restate.init_matrix(N, v)[0]
    LU, perm = blocked_lu(A, v, lambda L, U: L @ U)
    print(f"N={N} v={v}: native FP64 update        residual {residual(A, LU, perm):.2e}")
    for s in (5, 6, 7, 8, 9):
        cnt = [0]

        def g(L, U, s=s):
            C, n = ozaki_gemm(L, U, s)
            cnt[0] = n
            return C
        LU, perm2 = blocked_lu(A, v, g)
        same = bool(np.array_equal(perm, perm2))
        print(f"N={N} v={v}: {s} int8 slices ({cnt[0]:2d} int8 GEMMs) residual {residual(A, LU, perm2):.2e}  pivots == native: {same}"
              f"   int8-peak-equivalent {4500 / cnt[0]:.0f} TFLOP/s")
