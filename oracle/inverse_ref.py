"""oracle/inverse_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_inverse and cflx_chol_inverse
(conflux_b200/csrc/inverse.cu on the sweeps of solve.cu).

The specification of the inverse's schedule, checkable without GPUs.  It takes every rank's share of the factors (the LU:
L\\U in the conflux layout and the permutation, as restate.lu / cflx_lu_get_factors give them; the Cholesky: L in the
CONFCHOX layout, as cflx_chol_get_local gives it) and simulates, rank by rank, per block of nc columns [c0, c0 + nc):
  * the seed: X, W and Z zeroed on every rank, then W[r][j] = (global row of r == c0 + j) on the ranks (pi, 0, 0), for
    the LU's Ml rows (the identity row map: P A is solved) or the Cholesky's real rows;
  * the sweeps of the engine, tile by tile as solve.cu runs them (reduce onto the diagonal owner, nb-block solve with the
    inverted diagonal blocks, broadcast, update), over the tile ranges that skip the block's zero rows (T0 = c0 / v):
      LU:       L Y = E over tiles [T0, Nt) keeping Y_t as the owner's W rows; U Z = Y over every tile;
      Cholesky: L Y = E over [T0, Kappa) keeping Y_t in Z; L^T X = Y over [T0, Kappa), updating local columns
                T0 <= gj < t only;
  * the world all-reduce of the per-rank X, to which only the diagonal owners contribute;
  * the scatter of block column j into every rank's share: the LU to global column perm[c0 + j], every local row; the
    Cholesky to global column c0 + j, the real tiles on and below the diagonal only, and at the end zeros on the rest.
Every collective is recorded per rank as (communicator, op, root, count); collectives over a communicator of one rank are
skipped, as on the device.  Every update launch is recorded as (sweep, m, n, k) with n the block's nc columns, for the
flop count.  Each update's product is formed tile by tile, so that running the full tile range instead of the skipping
one changes no bit of what is kept.  Only the entries the device reads are read."""
import numpy as np

from . import chol_ref, layout
from .solve_ref import pick_nb


def flt(g, p, P):
    """first local tile (row or column) whose global tile index is >= g, on grid position p of P"""
    return 0 if g <= p else -(-(g - p) // P)


def seed_share(Ml, v, Px, pi, rows, c0, nc):
    """the seed kernel on one share: W (Ml x ldn) with W[r][j] = (global row of r == c0 + j) for r < rows, j < nc"""
    ldn = -(-nc // 8) * 8
    W = np.zeros((Ml, ldn))
    for r in range(rows):
        j = ((r // v) * Px + pi) * v + r % v - c0
        if 0 <= j < nc:
            W[r, j] = 1.0
    return W


def scatter_share(kind, X, c0, nc, perm, share, v, Px, Py, pi, pj, Kappa=None):
    """the scatter kernel on one share (in place, returned): column j < nc of X (by global row) to the local column of
    global column perm[c0 + j] ("lu", every local row) or c0 + j ("chol": real tiles, index < Kappa, on and below the
    diagonal)"""
    Ml, Nl = share.shape
    for j in range(nc):
        gc = int(perm[c0 + j]) if kind == "lu" else c0 + j
        tc = gc // v
        if tc % Py != pj or (tc // Py) * v >= Nl:
            continue
        lc = (tc // Py) * v + gc % v
        for r in range(Ml):
            gr = ((r // v) * Px + pi) * v + r % v
            if kind == "chol" and (gr // v >= Kappa or gr // v < tc):
                continue
            share[r, lc] = X[gr, j]
    return share


def zero_share(share, v, Px, Py, pi, pj, Kappa):
    """the Cholesky's zero pass (in place, returned): zero on tiles above the diagonal and tiles with index >= Kappa"""
    Ml, Nl = share.shape
    for lti in range(Ml // v):
        tr = lti * Px + pi
        for ltj in range(Nl // v):
            tc = ltj * Py + pj
            if tr >= Kappa or tc >= Kappa or tr < tc:
                share[lti * v:(lti + 1) * v, ltj * v:(ltj + 1) * v] = 0.0
    return share


def _run(kind, F_locals, perm, N, v, Px, Py, Pz, nc, skip, log, launches):
    if kind == "lu":
        d = layout.dims(N, v, Px, Py, Pz)
        M, Ml, Nl, Nt, P = d["M"], d["Ml"], d["Nl"], d["Nt"], d["P"]
    else:
        d = chol_ref.dims(N, v, Px, Py, Pz)
        M, Ml, Nl, Nt, P = d["N"], d["Ml"], d["Nl"], d["Kappa"], d["P"]
    assert nc % v == 0 and nc >= v
    F = [np.asarray(x, dtype=np.float64).reshape(Ml, Nl) for x in F_locals]
    assert len(F) == P
    nb = pick_nb(v)
    nblk = v // nb
    rank = lambda pi, pj, pk: layout.rank_of(pi, pj, pk, Px, Py, Pz)  # noqa: E731
    lu = kind == "lu"
    layers = range(Pz) if lu else range(1)                             # the LU's every layer joins the sweeps
    real_rows = lambda pi: Ml if lu else flt(Nt, pi, Px) * v           # noqa: E731  (f.rows)
    calls = {r: [] for r in range(P)}

    def collective(members, comm, op, root, count):
        if len(members) > 1:
            for r in members:
                calls[r].append((comm, op, root, count))

    # communicators: the LU's jk / ik (every layer, NCCL rank p * Pz + pk), the Cholesky's j / i of layer 0
    row_members = lambda pi: [rank(pi, pj, pk) for pj in range(Py) for pk in layers]  # noqa: E731
    col_members = lambda pj: [rank(pi, pj, pk) for pi in range(Px) for pk in layers]  # noqa: E731
    stride = Pz if lu else 1

    def diag_solve(t, tri, R):
        Ftt = F[rank(t % Px, t % Py, 0)][(t // Px) * v:(t // Px + 1) * v, (t // Py) * v:(t // Py + 1) * v]
        R = R.copy()
        Y = np.zeros_like(R)
        blocks = range(nblk) if tri in ("L", "Lunit") else reversed(range(nblk))
        for j in blocks:
            s = slice(j * nb, (j + 1) * nb)
            if tri == "Lunit":
                Y[s] = np.linalg.inv(np.tril(Ftt[s, s], -1) + np.eye(nb)) @ R[s]
                R[(j + 1) * nb:] -= Ftt[(j + 1) * nb:, s] @ Y[s]
            elif tri == "L":
                Y[s] = np.linalg.inv(np.tril(Ftt[s, s])) @ R[s]
                R[(j + 1) * nb:] -= Ftt[(j + 1) * nb:, s] @ Y[s]
            elif tri == "U":
                Y[s] = np.linalg.inv(np.triu(Ftt[s, s])) @ R[s]
                R[:j * nb] -= Ftt[:j * nb, s] @ Y[s]
            else:                                                      # "LT": L_tt^T with the Cholesky's L
                Y[s] = np.linalg.inv(np.tril(Ftt[s, s])).T @ R[s]
                R[:j * nb] -= Ftt[s, :j * nb].T @ Y[s]
        return Y

    def row_sweep(W, forward, tri, keep, keep_div, clear_row, t_lo, t_hi, nc_b, tag):
        tile = v * W[0].shape[1]
        for i in range(t_lo, t_hi):
            t = i if forward else t_lo + t_hi - 1 - i
            pr, pc = t % Px, t % Py
            lr = (t // Px) * v
            owner = rank(pr, pc, 0)
            members = row_members(pr)
            collective(members, ("row", pr), "reduce", pc * stride, tile)
            R = sum(W[m][lr:lr + v] for m in members)
            Y = diag_solve(t, tri, R)
            keep[owner][(t // keep_div) * v:(t // keep_div + 1) * v] = Y
            if clear_row:
                for pj in range(Py):
                    if pj != pc:
                        W[rank(pr, pj, 0)][lr:lr + v] = 0.0
            collective(col_members(pc), ("col", pc), "broadcast", pr * stride, tile)
            lc = (t // Py) * v
            for pi in range(Px):
                r = rank(pi, pc, 0)
                tiles = real_rows(pi) // v
                lo = min(tiles, flt(t + 1, pi, Px)) * v if forward else 0
                hi = real_rows(pi) if forward else min(tiles, flt(t, pi, Px)) * v
                if lo < hi:
                    launches.append((tag, hi - lo, nc_b, v))
                    for a in range(lo, hi, v):                         # tile by tile
                        W[r][a:a + v] -= F[r][a:a + v, lc:lc + v] @ Y

    def col_sweep_back(Z, Xr, t_lo, t_hi, nc_b):
        tile = v * Z[0].shape[1]
        for i in range(t_lo, t_hi):
            t = t_lo + t_hi - 1 - i
            pr, pc = t % Px, t % Py
            lc, lr = (t // Py) * v, (t // Px) * v
            owner = rank(pr, pc, 0)
            members = col_members(pc)
            collective(members, ("col", pc), "reduce", pr, tile)
            R = sum(Z[m][lc:lc + v] for m in members)
            Xt = diag_solve(t, "LT", R)
            Xr[owner][t * v:(t + 1) * v] = Xt
            collective(row_members(pr), ("row", pr), "broadcast", pc, tile)
            for pj in range(Py):
                r = rank(pr, pj, 0)
                m, c_lo = flt(t, pj, Py) * v, flt(t_lo, pj, Py) * v
                if m > c_lo:
                    launches.append(("back", m - c_lo, nc_b, v))
                    for a in range(c_lo, m, v):
                        Z[r][a:a + v] -= F[r][lr:lr + v, a:a + v].T @ Xt

    shares = [np.full((Ml, Nl), np.nan) for _ in range(P)]
    for c0 in range(0, M, nc):
        nc_b = min(nc, M - c0)
        ldn = -(-nc // 8) * 8                                          # every block runs nc's width
        T0 = c0 // v if skip else 0
        W = {r: np.zeros((Ml, ldn)) for r in range(P)}
        Z = {r: np.zeros((Nl, ldn)) for r in range(P)}
        Xr = {r: np.zeros((M, ldn)) for r in range(P)}
        for pi in range(Px):
            Wseed = seed_share(Ml, v, Px, pi, real_rows(pi), c0, nc_b)
            W[rank(pi, 0, 0)][:, :Wseed.shape[1]] = Wseed
        if lu:
            row_sweep(W, True, "Lunit", W, Px, True, T0, Nt, nc_b, "fwd")
            row_sweep(W, False, "U", Xr, 1, False, 0, Nt, nc_b, "back")
        else:
            row_sweep(W, True, "L", Z, Py, False, T0, Nt, nc_b, "fwd")
            col_sweep_back(Z, Xr, T0, Nt, nc_b)
        collective(list(range(P)), ("world",), "allreduce", None, M * ldn)
        X = sum(Xr.values())                                           # one contributor per element
        for r in range(P):
            pi, pj = r // (Py * Pz), (r // Pz) % Py
            scatter_share(kind, X, c0, nc_b, perm, shares[r], v, Px, Py, pi, pj, Nt)
    if not lu:
        for r in range(P):
            pi, pj = r // (Py * Pz), (r // Pz) % Py
            zero_share(shares[r], v, Px, Py, pi, pj, Nt)
    if log is not None:
        log.update(calls)
    return shares


def lu_inverse(C_locals, perm, N, v, Px=1, Py=1, Pz=1, nc=None, skip=True, log=None, launches=None):
    """Every rank's Ml x Nl share of inv(A) from the per-rank factors C_locals and perm (cflx_lu_inverse).  nc: columns per
    block (a multiple of v; default all of M).  skip=False runs every sweep over every tile.  log / launches: a dict / list
    that receive the collectives per rank and the update launches."""
    M = layout.dims(N, v, Px, Py, Pz)["M"]
    return _run("lu", C_locals, perm, N, v, Px, Py, Pz, nc or M, skip, log, [] if launches is None else launches)


def chol_inverse(L_locals, N, v, Px=1, Py=1, Pz=1, nc=None, skip=True, log=None, launches=None):
    """Every rank's Ml x Nl share of dpotri's lower triangle from the per-rank factor L_locals (cflx_chol_inverse)."""
    M = chol_ref.dims(N, v, Px, Py, Pz)["N"]
    return _run("chol", L_locals, None, N, v, Px, Py, Pz, nc or M, skip, log, [] if launches is None else launches)
