"""oracle/rbt_ref.py -- numpy restatement of the random butterfly transforms (cflx_rbt_multipliers, cflx_lu_rbt,
cflx_lu_rbt_apply_local, cflx_dbg_rbt_share): the multipliers, the per-share operations, the dense global W = U^T A V
(elementwise in the library's order, and from explicit butterfly matrices) and the divisibility rule.
Test infrastructure: only tests/ and tools/ import this."""
import math

import numpy as np

MASK = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15
SQRT1_2 = math.sqrt(0.5)   # fl(1/sqrt 2), correctly rounded


def _splitmix_final(z):
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & MASK
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def multipliers(M, depth, seed):
    """(u, v): the r values of U (side 0) and V (side 1), (depth, M) each, with Python's math.exp (the C library's)"""
    out = []
    for side in (0, 1):
        r = np.empty((depth, M))
        for l in range(depth):
            for i in range(M):
                k = (seed + GOLDEN * ((((2 * l + side) << 32) + i + 1) & MASK)) & MASK
                w = (_splitmix_final(k) >> 11) * 2.0 ** -53
                r[l, i] = math.exp((w - 0.5) / 10.0)
        out.append(r)
    return tuple(out)


def scales(r):
    """the device multipliers s = fl(r fl(1/sqrt 2))"""
    return np.asarray(r, dtype=np.float64) * SQRT1_2


def fits(M, v, Px, depth):
    """the transform is local to every rank's share exactly when M is a multiple of 2^depth v Px"""
    return M % ((v * Px) << depth) == 0


def smallest_order(M, v, Px, depth):
    """the smallest M' >= M that fits: pad A with the identity to that order"""
    q = (v * Px) << depth
    return -(-M // q) * q


def global_index(n, v, P, p):
    """the global index of every local index of an n-long local dimension at position p of P (Layout::row / col)"""
    l = np.arange(n)
    return ((l // v) * P + p) * v + l % v


def _rows_level(X, s, idx, l, fwd):
    """one level on the rows of X (the rows' global indices idx, s the level's multipliers by global index)"""
    n = X.shape[0]
    h = n >> (l + 1)
    Y = X.reshape(-1, 2, h, X.shape[1])
    S = s[idx].reshape(-1, 2, h, 1)
    a, b = Y[:, 0].copy(), Y[:, 1].copy()
    if fwd:
        ta, tb = S[:, 0] * a, S[:, 1] * b
        Y[:, 0], Y[:, 1] = ta + tb, ta - tb
    else:
        Y[:, 0], Y[:, 1] = S[:, 0] * (a + b), S[:, 1] * (a - b)


def apply_rows(op, X, su, sv, rows):
    """op 0 U^T, 1 V, 2 V^T, 3 U on the rows of X (a copy is returned); su / sv the device multipliers (depth, M), rows the
    global index of every local row"""
    X = np.array(X, dtype=np.float64)
    s = su if op in (0, 3) else sv
    d = s.shape[0]
    fwd = op in (1, 3)
    for l in (range(d) if fwd else reversed(range(d))):
        _rows_level(X, s[l], rows, l, fwd)
    return X


def apply_w(X, su, sv, rows, cols):
    """W = U^T X V on a matrix share: for l = d-1 .. 0, U's level l on the rows, then V's level l on the columns (the
    transposed operation along each row)"""
    X = np.array(X, dtype=np.float64)
    XT = X.T   # a view: the column operations write X
    for l in reversed(range(su.shape[0])):
        _rows_level(X, su[l], rows, l, False)
        T = np.ascontiguousarray(XT)
        _rows_level(T, sv[l], cols, l, False)
        X[...] = T.T
    return X


def share_op(op, X, v, depth, u, vv, grid=(1, 1), pos=(0, 0)):
    """cflx_dbg_rbt_share restated: u / vv the r values"""
    Px, Py = grid
    su = scales(u) if u is not None else None
    sv = scales(vv) if vv is not None else None
    rows = global_index(X.shape[0], v, Px, pos[0])
    if op == 4:
        return apply_w(X, su, sv, rows, global_index(X.shape[1], v, Py, pos[1]))
    return apply_rows(op, X, su, sv, rows)


def global_w(A, u, vv):
    """the dense U^T A V elementwise, in the library's order"""
    M = A.shape[0]
    return apply_w(A, scales(u), scales(vv), np.arange(M), np.arange(M))


def butterfly(s, l):
    """the explicit M x M matrix of level l with multipliers s (by global index): diag over the blocks of
    (1/sqrt 2) [R0 R1; R0 -R1], its 1/sqrt 2 folded into s"""
    M = s.shape[0]
    B = np.zeros((M, M))
    n = M >> l
    h = n // 2
    for b0 in range(0, M, n):
        p = np.arange(b0, b0 + h)
        q = p + h
        B[p, p], B[p, q] = s[p], s[q]
        B[q, p], B[q, q] = s[p], -s[q]
    return B


def matrices(u, vv):
    """(U, V) = (B_{d-1} .. B_0) of each side, from the device multipliers"""
    out = []
    for r in (u, vv):
        s = scales(r)
        M = s.shape[1]
        X = np.eye(M)
        for l in range(s.shape[0]):
            X = butterfly(s[l], l) @ X
        out.append(X)
    return tuple(out)


def solve(A, B, u, vv, trans=False):
    """X = V inv(W) U^T B, or U inv(W)^T V^T B, with W = U^T A V from the explicit matrices"""
    U, V = matrices(u, vv)
    W = U.T @ A @ V
    if trans:
        return U @ np.linalg.solve(W.T, V.T @ B)
    return V @ np.linalg.solve(W, U.T @ B)
