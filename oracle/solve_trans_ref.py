"""oracle/solve_trans_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_solve_trans (conflux_b200/csrc/lu.cu,
solve.cu): A^T X = B with the LU factors in the conflux layout (what cflx_lu_get_factors / restate.lu return).

With P A = L U (row q of P A is row perm[q] of A):  A^T X = B  <=>  U^T (L^T W) = B,  X[perm[q]] = W[q].
Simulated rank by rank:
  * Z: each rank's partial right-hand side by local tile column (Nl x ldn).  Ranks (0, pj, 0) start with the rows of B of
    their tile columns (local column (k / Py) v + i holds row k v + i), all others with zeros;
  * forward sweep U^T Y = B, t ascending: the reduce of Z's tile t / Py over the grid column (every layer contributes)
    onto the owner (t % Px, t % Py, 0); Y_j = inv(U_jj)^T R_j, R_i -= U_ji^T Y_j (i > j); the owner keeps Y_t in Z, the
    other layer-0 ranks of the grid column zero their copy; the broadcast over the grid row; Z[local columns gj > t] -=
    U[t, gj]^T Y_t on every layer-0 rank of that grid row;
  * backward sweep L^T W = Y, t descending: the same reduce; W_j = inv(L_jj)^T R_j (unit L), R_i -= L_ji^T W_j (i < j);
    the owner writes W_t into its X rows; the broadcast; Z[local columns gj < t] -= L[t, gj]^T W_t;
  * the all-reduce of the per-rank X buffers, then X[perm[q]] = W[q] on every rank.
Every collective is recorded per rank as (communicator, op, root, count); collectives over a communicator of one rank are
skipped, as on the device.  pa=True restates the condition estimate's products with P A: no final P^T."""
import numpy as np

from . import layout
from .solve_ref import backward_error, pick_nb  # noqa: F401  (backward_error: for the tests)


def solve(C_locals, perm, B, N, v, Px=1, Py=1, Pz=1, log=None, pa=False):
    """X (M x nrhs, or (M,) for a vector B) with A^T X = B ((P A)^T X = B with pa), from the per-rank factors C_locals."""
    d = layout.dims(N, v, Px, Py, Pz)
    M, Ml, Nl, Nt, P = d["M"], d["Ml"], d["Nl"], d["Nt"], d["P"]
    B = np.asarray(B, dtype=np.float64)
    vec = B.ndim == 1
    B = B.reshape(M, -1)
    nrhs = B.shape[1]
    ldn = -(-nrhs // 8) * 8
    Bp = np.zeros((M, ldn))
    Bp[:, :nrhs] = B
    C = [np.asarray(c, dtype=np.float64).reshape(Ml, Nl) for c in C_locals]
    assert len(C) == P
    nb = pick_nb(v)
    nblk = v // nb
    tile = v * ldn
    rank = lambda pi, pj, pk: layout.rank_of(pi, pj, pk, Px, Py, Pz)  # noqa: E731
    first_local_tile = lambda g, p, Pd: max(0, -(-(g - p) // Pd))    # noqa: E731  (first local tile with index >= g)
    calls = {r: [] for r in range(P)}

    def collective(members, comm, op, root, count):
        if len(members) > 1:
            for r in members:
                calls[r].append((comm, op, root, count))

    # the LU's communicators: the grid row (jk) and the grid column (ik) of every layer, layer 0 at rank p * Pz
    row_members = lambda pi: [rank(pi, pj, pk) for pj in range(Py) for pk in range(Pz)]  # noqa: E731
    col_members = lambda pj: [rank(pi, pj, pk) for pi in range(Px) for pk in range(Pz)]  # noqa: E731

    Z = {r: np.zeros((Nl, ldn)) for r in range(P)}
    for pj in range(Py):
        for q in range(M):
            k, i = divmod(q, v)
            if k % Py == pj:
                Z[rank(0, pj, 0)][(k // Py) * v + i] = Bp[q]

    def diag_tile(t):
        lr, lc = (t // Px) * v, (t // Py) * v
        return C[rank(t % Px, t % Py, 0)][lr:lr + v, lc:lc + v]

    for t in range(Nt):                                             # forward sweep: U^T Y = B
        pr, pc = t % Px, t % Py
        lr, lc = (t // Px) * v, (t // Py) * v
        collective(col_members(pc), ("col", pc), "reduce", pr * Pz, tile)
        R = sum(Z[r][lc:lc + v] for r in col_members(pc)).copy()
        Ctt = diag_tile(t)
        Y = np.zeros((v, ldn))
        for j in range(nblk):
            s = slice(j * nb, (j + 1) * nb)
            Uinv = np.linalg.inv(np.triu(Ctt[s, s]))
            Y[s] = Uinv.T @ R[s]
            R[(j + 1) * nb:] -= Ctt[s, (j + 1) * nb:].T @ Y[s]
        for pi in range(Px):
            Z[rank(pi, pc, 0)][lc:lc + v] = Y if pi == pr else 0.0
        collective(row_members(pr), ("row", pr), "broadcast", pc * Pz, tile)
        for pj in range(Py):
            r = rank(pr, pj, 0)
            lo = first_local_tile(t + 1, pj, Py) * v
            if lo < Nl:
                Z[r][lo:] -= C[r][lr:lr + v, lo:].T @ Y

    Xr = {r: np.zeros((M, ldn)) for r in range(P)}
    for t in reversed(range(Nt)):                                   # backward sweep: L^T W = Y
        pr, pc = t % Px, t % Py
        lr, lc = (t // Px) * v, (t // Py) * v
        collective(col_members(pc), ("col", pc), "reduce", pr * Pz, tile)
        R = sum(Z[r][lc:lc + v] for r in col_members(pc)).copy()
        Ctt = diag_tile(t)
        Wt = np.zeros((v, ldn))
        for j in reversed(range(nblk)):
            s = slice(j * nb, (j + 1) * nb)
            Linv = np.linalg.inv(np.tril(Ctt[s, s], -1) + np.eye(nb))
            Wt[s] = Linv.T @ R[s]
            R[:j * nb] -= Ctt[s, :j * nb].T @ Wt[s]
        Xr[rank(pr, pc, 0)][t * v:(t + 1) * v] = Wt
        collective(row_members(pr), ("row", pr), "broadcast", pc * Pz, tile)
        for pj in range(Py):
            r = rank(pr, pj, 0)
            m = first_local_tile(t, pj, Py) * v
            if m > 0:
                Z[r][:m] -= C[r][lr:lr + v, :m].T @ Wt
    collective(list(range(P)), ("world",), "allreduce", None, M * ldn)
    if log is not None:
        log.update(calls)
    W = sum(Xr.values())[:, :nrhs]                                  # one contributor per element
    X = W.copy()
    if not pa:
        X[np.asarray(perm)] = W
    return X.reshape(M) if vec else X


def host_solve(LU, perm, B):
    """Reference answer: X[perm] = L^-T U^-T B with the assembled factors."""
    from scipy.linalg import solve_triangular
    B = np.asarray(B, dtype=np.float64)
    Y = solve_triangular(LU, B, trans="T")
    W = solve_triangular(LU, Y, trans="T", lower=True, unit_diagonal=True)
    X = np.empty_like(W)
    X[np.asarray(perm)] = W
    return X
