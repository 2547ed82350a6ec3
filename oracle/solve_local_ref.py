"""oracle/solve_local_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_solve_local and cflx_chol_solve_local
(conflux_b200/csrc/solve_local.cu on the solves of solve.cu).

B and X are M x nrhs matrices tiled v x v like A: global tile (I, J) on grid position (I % Px, J % Py) at local tile
(I / Px, J / Py) of a row-major share of Ml x rhs_local_cols(nrhs, v, Py).  The schedule, per block of w <= nc columns
[c0, c0 + w) (nc = block_cols(M, v), the inverse's width):
  * pack: every layer-0 share writes its entries of the block into a zeroed M x round_up(w, 8) buffer by global row
    (the LU: every local row; the Cholesky: the rows of real tiles, global tile index < Kappa); local columns with a
    global index >= nrhs are not read;
  * the world sum of the packed buffers, with exactly one contributor per element;
  * the solve of the assembled block (here densely, on the assembled factors);
  * scatter: the solved block into every rank's X share, the layers pk != 0 included, at the same entries.
Only the entries the device reads are read, and only those it writes are written."""
import numpy as np
from scipy.linalg import solve_triangular

from . import chol_ref, layout, solve_ref, solve_trans_ref


def rhs_local_cols(nrhs, v, Py):
    """v * ceil(ceil(nrhs / v) / Py): lu_params' padding rule applied to nrhs"""
    return v * -(-(-(-nrhs // v)) // Py)


def block_cols(M, v):
    """the inverse's block width: the whole number of tiles nearest 2048 columns, all of M when M is smaller"""
    return min(max(1, (2048 + v // 2) // v) * v, M)


def local_rows(kind, Ml, v, Px, pi, Kappa=None):
    """the local rows a distributed solve reads and writes: every row ("lu"), or those before the first local tile with a
    global index >= Kappa ("chol")"""
    if kind == "lu":
        return Ml
    first = 0 if Kappa <= pi else -(-(Kappa - pi) // Px)
    return min(Ml, first * v)


def block_entries(kind, Ml, v, Px, Py, pi, pj, nrhs, c0, w, Kappa=None):
    """(local rows, local columns, their global rows, their block columns) of the share's entries of block [c0, c0 + w)"""
    rows = np.arange(local_rows(kind, Ml, v, Px, pi, Kappa))
    lc = np.arange(rhs_local_cols(nrhs, v, Py))
    gc = ((lc // v) * Py + pj) * v + lc % v
    keep = (gc >= c0) & (gc < c0 + w)
    gr = ((rows // v) * Px + pi) * v + rows % v
    return rows, lc[keep], gr, gc[keep] - c0


def pack_share(kind, B, M, v, Px, Py, pi, pj, nrhs, c0, w, Kappa=None):
    """the pack kernel on one share B (Ml x n >= rhs_local_cols): the M x round_up(w, 8) buffer, zero where the share
    holds nothing"""
    rows, lc, gr, j = block_entries(kind, B.shape[0], v, Px, Py, pi, pj, nrhs, c0, w, Kappa)
    Bk = np.zeros((M, -(-w // 8) * 8))
    Bk[np.ix_(gr, j)] = B[np.ix_(rows, lc)]
    return Bk


def scatter_share(kind, Xk, X, v, Px, Py, pi, pj, nrhs, c0, w, Kappa=None):
    """the scatter kernel on one share X (in place, returned): block column j of Xk (by global row) into the share's local
    column of global column c0 + j, at the rows the pack reads"""
    rows, lc, gr, j = block_entries(kind, X.shape[0], v, Px, Py, pi, pj, nrhs, c0, w, Kappa)
    X[np.ix_(rows, lc)] = Xk[np.ix_(gr, j)]
    return X


def _dense_solve(kind, F, perm, B, trans):
    if kind == "lu":
        return (solve_trans_ref if trans else solve_ref).host_solve(F, perm, B)
    Y = solve_triangular(F, B, lower=True)
    return solve_triangular(F, Y, lower=True, trans="T")


def solve_local(kind, F_locals, perm, B_locals, X_locals, nrhs, N, v, Px=1, Py=1, Pz=1, trans=False, nc=None):
    """The schedule over all ranks.  F_locals: every rank's share of the factors (the LU: L\\U and perm as
    cflx_lu_get_factors gives them; the Cholesky: L as cflx_chol_get_local gives it); B_locals: every rank's B share
    (read on layer 0 only; may be None elsewhere); X_locals: every rank's X share, written in place (None: not
    written).  Returns X_locals.  Asserts that each element of every assembled block has exactly one contributor."""
    if kind == "lu":
        d = layout.dims(N, v, Px, Py, Pz)
        M, Ml, Kappa = d["M"], d["Ml"], None
        F = layout.assemble(F_locals, N, v, Px, Py, Pz)
    else:
        d = chol_ref.dims(N, v, Px, Py, Pz)
        M, Ml, Kappa = d["N"], d["Ml"], d["Kappa"]
        F = np.tril(chol_ref.assemble(F_locals, N, v, Px, Py, Pz))
    P = Px * Py * Pz
    nc = nc or block_cols(M, v)
    pos = lambda r: (r // (Py * Pz), (r // Pz) % Py)  # noqa: E731
    for c0 in range(0, nrhs, nc):
        w = min(nc, nrhs - c0)
        ldn = -(-w // 8) * 8
        Bk, count = np.zeros((M, ldn)), np.zeros((M, ldn), dtype=int)
        for r in range(0, P, Pz):                                      # layer 0; the other layers contribute zeros
            pi, pj = pos(r)
            Bk += pack_share(kind, B_locals[r], M, v, Px, Py, pi, pj, nrhs, c0, w, Kappa)
            _, _, gr, j = block_entries(kind, Ml, v, Px, Py, pi, pj, nrhs, c0, w, Kappa)
            count[np.ix_(gr, j)] += 1
        assert np.all(count[:, :w] == 1) and np.all(count[:, w:] == 0)
        Xk = np.zeros((M, ldn))
        Xk[:, :w] = _dense_solve(kind, F, perm, Bk[:, :w], trans)
        for r in range(P):
            if X_locals[r] is not None:
                scatter_share(kind, Xk, X_locals[r], v, Px, Py, *pos(r), nrhs, c0, w, Kappa)
    return X_locals


def distribute(kind, G, v, Px=1, Py=1, Pz=1, Kappa=None, pad=np.nan, ld_extra=0):
    """G (M x nrhs) -> every rank's share (Ml x rhs_local_cols + ld_extra, Ml = M / Px for "lu", ceil(Kappa / Px) v for
    "chol"): G's entries where a solve reads and writes them, on every layer, `pad` elsewhere"""
    M, nrhs = G.shape
    Ml = M // Px if kind == "lu" else -(-Kappa // Px) * v
    out = []
    for r in range(Px * Py * Pz):
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        s = np.full((Ml, rhs_local_cols(nrhs, v, Py) + ld_extra), pad)
        rows, lc, gr, j = block_entries(kind, Ml, v, Px, Py, pi, pj, nrhs, 0, nrhs, Kappa)
        s[np.ix_(rows, lc)] = G[np.ix_(gr, j)]
        out.append(s)
    return out


def collect(kind, X_locals, M, nrhs, v, Px=1, Py=1, Pz=1, Kappa=None):
    """the M x nrhs matrix whose layer-0 shares are X_locals"""
    G = np.zeros((M, nrhs))
    for r in range(0, Px * Py * Pz, Pz):
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        rows, lc, gr, j = block_entries(kind, X_locals[r].shape[0], v, Px, Py, pi, pj, nrhs, 0, nrhs, Kappa)
        G[np.ix_(gr, j)] = X_locals[r][np.ix_(rows, lc)]
    return G
