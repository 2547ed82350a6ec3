"""oracle/solve_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_solve (conflux_b200/csrc/lu.cu, solve.cu).

The specification of the solve's communication schedule, checkable without GPUs.  It takes every rank's factors in the
conflux block-cyclic layout (what cflx_lu_get_factors / restate.lu return: tile (I, J) of L\\U on rank (I % Px, J % Py, 0))
and the permutation, and simulates, rank by rank:
  * W: each rank's partial right-hand side (Ml x ldn).  Ranks (pi, 0, 0) start with the rows of P*B of their tile rows,
    all others with zeros, so the sum of W over a grid row is the right-hand side of that grid row's tiles;
  * per tile t of the forward sweep: the reduce of tile t's rows over the grid row (every layer contributes) onto the
    diagonal owner (t % Px, t % Py, 0), the nb-block sweep Y_j = inv(L_jj) R_j, R_i -= L_ij Y_j (i > j), the broadcast
    over the grid column, the owner keeping Y_t as its W rows (the other ranks of the grid row zeroing theirs), and the
    update W[tiles I > t] -= L[I, t] Y_t on every layer-0 rank of the grid column;
  * the backward sweep likewise with U (X_j = inv(U_jj) R_j, R_i -= U_ij X_j for i < j; update of the tiles I < t);
  * the final all-reduce of the per-rank X buffers, to which only the diagonal owners contribute.
"""
import numpy as np

from . import layout


def pick_nb(v):
    """Block size of the diagonal inverses (lu.cu pick_nb with its default cap of 128, and chol.cu chol_pick_nb)."""
    for nb in (128, 64, 32, 16, 8, 4):
        if v % nb == 0:
            return nb
    raise ValueError(f"v={v}: no supported block size")


def solve(C_locals, perm, B, N, v, Px=1, Py=1, Pz=1):
    """X (M x nrhs, or (M,) for a vector B) with A X = B, from the per-rank factors C_locals and perm."""
    d = layout.dims(N, v, Px, Py, Pz)
    M, Ml, Nl, Nt, P = d["M"], d["Ml"], d["Nl"], d["Nt"], d["P"]
    B = np.asarray(B, dtype=np.float64)
    vec = B.ndim == 1
    B = B.reshape(M, -1)
    nrhs = B.shape[1]
    ldn = -(-nrhs // 8) * 8
    Bp = np.zeros((M, ldn))
    Bp[:, :nrhs] = B
    perm = np.asarray(perm)
    C = [np.asarray(c, dtype=np.float64).reshape(Ml, Nl) for c in C_locals]
    assert len(C) == P
    nb = pick_nb(v)
    nblk = v // nb
    rank = lambda pi, pj, pk: layout.rank_of(pi, pj, pk, Px, Py, Pz)  # noqa: E731
    first_local_tile = lambda t, pi: min(Ml // v, (t - pi + Px - 1) // Px)  # noqa: E731  (first local tile >= t)

    W = [np.zeros((Ml, ldn)) for _ in range(P)]
    for pi in range(Px):
        for q in range(M):
            k, i = divmod(q, v)
            if k % Px == pi:
                W[rank(pi, 0, 0)][(k // Px) * v + i] = Bp[perm[q]]

    def reduced(t):
        lr = (t // Px) * v
        return sum(W[rank(t % Px, pj, pk)][lr:lr + v] for pj in range(Py) for pk in range(Pz))

    def diag_tile(t):
        lr, lc = (t // Px) * v, (t // Py) * v
        return C[rank(t % Px, t % Py, 0)][lr:lr + v, lc:lc + v]

    for t in range(Nt):                                           # forward sweep: L Y = P B
        pr, pc = t % Px, t % Py
        Ctt, R = diag_tile(t), reduced(t).copy()
        Y = np.zeros((v, ldn))
        for j in range(nblk):
            s = slice(j * nb, (j + 1) * nb)
            Linv = np.linalg.inv(np.tril(Ctt[s, s], -1) + np.eye(nb))
            Y[s] = Linv @ R[s]
            R[(j + 1) * nb:] -= Ctt[(j + 1) * nb:, s] @ Y[s]
        lr, lc = (t // Px) * v, (t // Py) * v
        for pj in range(Py):
            W[rank(pr, pj, 0)][lr:lr + v] = Y if pj == pc else 0.0
        for pi in range(Px):
            r = rank(pi, pc, 0)
            lo = first_local_tile(t + 1, pi) * v
            W[r][lo:] -= C[r][lo:, lc:lc + v] @ Y

    Xr = [np.zeros((M, ldn)) for _ in range(P)]
    for t in reversed(range(Nt)):                                 # backward sweep: U X = Y
        pr, pc = t % Px, t % Py
        Ctt, R = diag_tile(t), reduced(t).copy()
        Xt = np.zeros((v, ldn))
        for j in reversed(range(nblk)):
            s = slice(j * nb, (j + 1) * nb)
            Uinv = np.linalg.inv(np.triu(Ctt[s, s]))
            Xt[s] = Uinv @ R[s]
            R[:j * nb] -= Ctt[:j * nb, s] @ Xt[s]
        Xr[rank(pr, pc, 0)][t * v:(t + 1) * v] = Xt
        lc = (t // Py) * v
        for pi in range(Px):
            r = rank(pi, pc, 0)
            hi = first_local_tile(t, pi) * v
            W[r][:hi] -= C[r][:hi, lc:lc + v] @ Xt
    X = sum(Xr)[:, :nrhs]                                         # the all-reduce: one contributor per element
    return X.reshape(M) if vec else X


def host_solve(LU, perm, B):
    """Reference answer: triangular solves with the assembled factors, X = U^-1 L^-1 B[perm]."""
    from scipy.linalg import solve_triangular
    B = np.asarray(B, dtype=np.float64)
    Y = solve_triangular(LU, B[np.asarray(perm)], lower=True, unit_diagonal=True)
    return solve_triangular(LU, Y, lower=False)


def backward_error(A, X, B):
    """Normwise backward error ||B - A X||_F / (||A||_F ||X||_F + ||B||_F); X and B may be vectors."""
    X, B = np.asarray(X).reshape(len(B), -1), np.asarray(B).reshape(len(B), -1)
    return float(np.linalg.norm(B - A @ X) / (np.linalg.norm(A) * np.linalg.norm(X) + np.linalg.norm(B)))
