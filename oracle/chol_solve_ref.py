"""oracle/chol_solve_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_chol_solve (conflux_b200/csrc/chol.cu,
solve.cu).

The specification of the Cholesky solve's schedule, checkable without GPUs.  It takes every rank's local share of the
factor in the CONFCHOX layout (what cflx_chol_get_local returns: tile (gi, gj), gi >= gj, of L on rank (gi % Px, gj % Py,
0) at local tile (gi / Px, gj / Py)) and simulates, rank by rank:
  * W: each layer-0 rank's partial right-hand side (Ml x ldn, by local tile row).  Ranks (pi, 0, 0) start with the rows
    of B of their real tile rows, all others with zeros;
  * forward sweep, per tile t: the reduce of W's tile t over the grid row onto the owner (t % Px, t % Py, 0), the nb-block
    sweep Y_j = inv(L_jj) R_j, R_i -= L_ij Y_j (i > j), the owner keeping Y_t in Z at its local column t / Py, the
    broadcast of Y_t over the grid column, and W[real tiles I > t] -= L[I, t] Y_t on every layer-0 rank of that column;
  * backward sweep, per tile t = Kappa - 1 .. 0: the reduce of Z's tile t over the grid column onto the owner, X_j =
    inv(L_jj)^T R_j, R_i -= L_ji^T X_j (i < j), the broadcast of X_t over the grid row, and Z[local columns gj < t] -=
    L[t, gj]^T X_t on every layer-0 rank of that row;
  * the final all-reduce of the per-rank X buffers, to which only the diagonal owners contribute.
Only the entries the device reads are read here: the tiles on and below the diagonal, the real tiles (global index <
Kappa) and layer 0.  Every collective is recorded per rank as (communicator, op, root, count); collectives over a
communicator of one rank are skipped, as on the device."""
import numpy as np

from . import chol_ref, layout
from .solve_ref import backward_error, pick_nb  # noqa: F401  (backward_error: for the tests)


def scatter(A, N, v, Px=1, Py=1, Pz=1, upper=None, pad=0.0, layers=0.0):
    """Global (padded) matrix -> the per-rank local arrays of the CONFCHOX layout, in rank order.  upper: value of every
    entry of the tiles above the diagonal (None: A's own); pad: value of the local tiles with a global index >= Kappa;
    layers: value of every entry on the layers pk != 0."""
    d = chol_ref.dims(N, v, Px, Py, Pz)
    K, Ml, Nl = d["Kappa"], d["Ml"], d["Nl"]
    out = []
    for r in range(d["P"]):
        pi, pj, pk = r // (Py * Pz), (r // Pz) % Py, r % Pz
        loc = np.full((Ml, Nl), float(layers if pk else pad))
        if pk == 0:
            for lti in range(Ml // v):
                for ltj in range(Nl // v):
                    gi, gj = lti * Px + pi, ltj * Py + pj
                    if gi >= K or gj >= K:
                        continue
                    blk = A[gi * v:(gi + 1) * v, gj * v:(gj + 1) * v]
                    loc[lti * v:(lti + 1) * v, ltj * v:(ltj + 1) * v] = upper if (gi < gj and upper is not None) else blk
        out.append(loc)
    return out


def solve(L_locals, B, N, v, Px=1, Py=1, Pz=1, log=None):
    """X (N x nrhs, or (N,) for a vector B; N the padded size) with L L^T X = B.  log: a dict that receives, per rank, the
    list of the collectives that rank issues, as (communicator, op, root, count)."""
    d = chol_ref.dims(N, v, Px, Py, Pz)
    Np, K, Ml, Nl, P = d["N"], d["Kappa"], d["Ml"], d["Nl"], d["P"]
    B = np.asarray(B, dtype=np.float64)
    vec = B.ndim == 1
    B = B.reshape(Np, -1)
    nrhs = B.shape[1]
    ldn = -(-nrhs // 8) * 8
    Bp = np.zeros((Np, ldn))
    Bp[:, :nrhs] = B
    L = [np.asarray(x, dtype=np.float64).reshape(Ml, Nl) for x in L_locals]
    assert len(L) == P
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

    row_members = lambda pi: [rank(pi, pj, 0) for pj in range(Py)]  # noqa: E731  (j_comm of layer 0, key pj)
    col_members = lambda pj: [rank(pi, pj, 0) for pi in range(Px)]  # noqa: E731  (i_comm of layer 0, key pi)

    W = {r: np.zeros((Ml, ldn)) for r in range(P)}
    Z = {r: np.zeros((Nl, ldn)) for r in range(P)}
    for pi in range(Px):
        for lti in range(first_local_tile(K, pi, Px)):
            gi = lti * Px + pi
            W[rank(pi, 0, 0)][lti * v:(lti + 1) * v] = Bp[gi * v:(gi + 1) * v]

    def diag_blocks(t):
        lr, lc = (t // Px) * v, (t // Py) * v
        Ltt = L[rank(t % Px, t % Py, 0)][lr:lr + v, lc:lc + v]
        return Ltt, [np.linalg.inv(np.tril(Ltt[j * nb:(j + 1) * nb, j * nb:(j + 1) * nb])) for j in range(nblk)]

    for t in range(K):                                              # forward sweep: L Y = B
        pr, pc = t % Px, t % Py
        lr, lc = (t // Px) * v, (t // Py) * v
        collective(row_members(pr), ("row", pr), "reduce", pc, tile)
        R = sum(W[r][lr:lr + v] for r in row_members(pr)).copy()
        Ltt, Linv = diag_blocks(t)
        Y = np.zeros((v, ldn))
        for j in range(nblk):
            s = slice(j * nb, (j + 1) * nb)
            Y[s] = Linv[j] @ R[s]
            R[(j + 1) * nb:] -= Ltt[(j + 1) * nb:, s] @ Y[s]
        Z[rank(pr, pc, 0)][lc:lc + v] = Y
        collective(col_members(pc), ("col", pc), "broadcast", pr, tile)
        for pi in range(Px):
            r = rank(pi, pc, 0)
            lo, hi = first_local_tile(t + 1, pi, Px) * v, first_local_tile(K, pi, Px) * v
            if lo < hi:
                W[r][lo:hi] -= L[r][lo:hi, lc:lc + v] @ Y

    Xr = {r: np.zeros((Np, ldn)) for r in range(P)}
    for t in reversed(range(K)):                                    # backward sweep: L^T X = Y
        pr, pc = t % Px, t % Py
        lr, lc = (t // Px) * v, (t // Py) * v
        collective(col_members(pc), ("col", pc), "reduce", pr, tile)
        R = sum(Z[r][lc:lc + v] for r in col_members(pc)).copy()
        Ltt, Linv = diag_blocks(t)
        Xt = np.zeros((v, ldn))
        for j in reversed(range(nblk)):
            s = slice(j * nb, (j + 1) * nb)
            Xt[s] = Linv[j].T @ R[s]
            R[:j * nb] -= Ltt[s, :j * nb].T @ Xt[s]
        Xr[rank(pr, pc, 0)][t * v:(t + 1) * v] = Xt
        collective(row_members(pr), ("row", pr), "broadcast", pc, tile)
        for pj in range(Py):
            r = rank(pr, pj, 0)
            m = first_local_tile(t, pj, Py) * v
            if m > 0:
                Z[r][:m] -= L[r][lr:lr + v, :m].T @ Xt
    collective(list(range(P)), ("world",), "allreduce", None, Np * ldn)
    if log is not None:
        log.update(calls)
    X = sum(Xr.values())[:, :nrhs]                                  # one contributor per element
    return X.reshape(Np) if vec else X

