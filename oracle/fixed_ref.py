"""oracle/fixed_ref.py -- numpy restatement of cflx_lu_factor_fixed: the LU of A[perm] without a pivot search, blocked
in the order the GPU runs it (steps of v columns; inside the v x v diagonal block, 32-column blocks), with the tiny-pivot
rule and the first zero pivot.  Also the host bookkeeping of the fixed schedule: each grid row's pivot count per step.
Test infrastructure: only tests/ and tools/ import this."""
import numpy as np

TILE_NB = 32   # the column block of the one-CTA tile kernel (fixed.cu)


def _replace(d, tiny):
    """the tiny rule: |d| < tiny -> copysign(tiny, d), +tiny for +-0; (value, replaced)"""
    if abs(d) < tiny:
        return (tiny if d == 0.0 else float(np.copysign(tiny, d))), True
    return d, False


def tile_lu(B, tiny=0.0, col0=0, nb=TILE_NB):
    """Unpivoted LU of the square block B (right-looking over nb-column blocks, as the tile kernel): (L\\U, nrepl,
    first) with first = col0 + 1 + the column of the first exactly zero pivot, 0 when there is none."""
    A = np.array(B, dtype=np.float64)
    v = A.shape[0]
    nrepl, first = 0, 0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for jb in range(0, v, nb):
            e = min(v, jb + nb)
            for c in range(jb, e):                                  # the diagonal block
                d, r = _replace(A[c, c], tiny)
                nrepl += r
                if d == 0.0 and first == 0:
                    first = col0 + c + 1
                A[c, c] = d
                A[c + 1:e, c] /= d
                A[c + 1:e, c + 1:e] -= np.outer(A[c + 1:e, c], A[c, c + 1:e])
            U11 = np.triu(A[jb:e, jb:e])
            L11 = np.tril(A[jb:e, jb:e], -1) + np.eye(e - jb)
            if e < v:
                A[e:, jb:e] = _solve_right_upper(A[e:, jb:e], U11)  # L21 = A21 inv(U11)
                A[jb:e, e:] = _solve_left_unit(L11, A[jb:e, e:])    # U12 = inv(L11) A12
                A[e:, e:] -= A[e:, jb:e] @ A[jb:e, e:]
    return A, nrepl, first


def _solve_right_upper(X, U):
    out = np.array(X, dtype=np.float64)
    for c in range(U.shape[0]):
        out[:, c] = (out[:, c] - out[:, :c] @ U[:c, c]) / U[c, c]
    return out


def _solve_left_unit(L, X):
    out = np.array(X, dtype=np.float64)
    for r in range(L.shape[0]):
        out[r] -= L[r, :r] @ out[:r]
    return out


def lu(A, perm, v, tiny=0.0):
    """The factorisation of A[perm] in steps of v columns: per step the tile LU of the diagonal block (tile_lu), the
    TRSMs of the L panel and the U row, the rank-v trailing update.  Returns dict(LU = L\\U of P A, nrepl, info)."""
    perm = np.asarray(perm)
    M = A.shape[0]
    assert sorted(perm.tolist()) == list(range(M)), "perm is not a permutation"
    F = np.array(A, dtype=np.float64)[perm]
    nrepl, info = 0, 0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for k0 in range(0, M, v):
            k1 = min(M, k0 + v)
            D, r, f = tile_lu(F[k0:k1, k0:k1], tiny, col0=k0)
            F[k0:k1, k0:k1] = D
            nrepl += r
            if f and not info:
                info = f
            if k1 < M:
                U = np.triu(D)
                L = np.tril(D, -1) + np.eye(k1 - k0)
                F[k1:, k0:k1] = _solve_right_upper(F[k1:, k0:k1], U)
                F[k0:k1, k1:] = _solve_left_unit(L, F[k0:k1, k1:])
                F[k1:, k1:] -= F[k1:, k0:k1] @ F[k0:k1, k1:]
    return dict(LU=F, nrepl=nrepl, info=info)


def step_counts(perm, v, Px):
    """counts[k][p]: the rows of step k (perm[k v .. k v + v)) that grid row p owns, (g / v) % Px == p: the pivot count
    each rank computes on the host"""
    perm = np.asarray(perm)
    Nt = len(perm) // v
    out = np.zeros((Nt, Px), dtype=np.int64)
    for k in range(Nt):
        for g in perm[k * v:(k + 1) * v]:
            out[k, (int(g) // v) % Px] += 1
    return out

