"""oracle/refine_local_ref.py -- TEST INFRASTRUCTURE: numpy restatement of the block rule of the distributed refinement
and expert drivers, cflx_lu_refine_local, _refine_x_local, _svx_local, _svxx_local and their Cholesky counterparts
(conflux_b200/csrc/solve_local.cu's block loop around the replicated cores of refine.cu and equil.cu).

B and X are distributed as in cflx_lu_solve_local (oracle/solve_local_ref.py).  The block rule:
  * the columns go in blocks [c0, c0 + w) of w <= block_cols(v): the whole number of tiles nearest REFINE_NC columns, at
    least one tile, whatever M and nrhs are; every block but the last is that wide;
  * each block of B (and, for refine and refine_x, of X) is packed and assembled as solve_local assembles it, then run
    through the replicated driver's core on those w columns alone, and X's block is scattered back;
  * the zero-pivot check, the pivot growth and the dgecon / dpocon rcond run once per call, before the blocks, so the
    matrix-level outputs are the replicated driver's;
  * info: a zero pivot k as the replicated driver (no block runs); svx's M + 1 as the replicated driver; refine_x's and
    svxx's M + j merge to the first global column j over all blocks.
The device workspace grows with w, not with nrhs (workspace_doubles)."""
import numpy as np

from . import solve_local_ref

REFINE_NC = 256   # CFLX_REFINE_NC (conflux_b200/csrc/lu_state.h)


def block_cols(v):
    """the block width: the whole number of tiles nearest REFINE_NC columns, at least one tile"""
    return max(1, (REFINE_NC + v // 2) // v) * v


def blocks(nrhs, v):
    """[(c0, w)] of a call on nrhs columns"""
    nc = block_cols(v)
    return [(c0, min(nc, nrhs - c0)) for c0 in range(0, nrhs, nc)]


def workspace_doubles(M, v, Ml, Nl, P, w):
    """the bound on the device workspace of one block of w columns (ldn = round_up(w, 8)), in doubles:
    ldn (15 M + 2 v + (2 P + 5)(Ml + Nl)) + 2 M.  Per M x ldn: the refinement's X, B, R, D, rhs, ratio, W and the tail T (8),
    the expert drivers' scaled B and X (2), the block loop's assembled B and X (2) and the solves' B, X and Xg (3); per
    (Ml + Nl) x ldn: the gathered heads and tails (2), the residual partials (2) and their all-gather over P ranks (2 P),
    and the solves' W and Z (1); the solves' R and Y (v x ldn each); and the pivot growth's column maxima of A and of the
    factor (M each), which do not depend on w."""
    ldn = -(-w // 8) * 8
    return ldn * (15 * M + 2 * v + (2 * P + 5) * (Ml + Nl)) + 2 * M


def merge_info(block_infos, M):
    """the call's info from each block's (in block order, c0 ascending; each M + j with j the block's first flagged
    column, 1-based, or 0): M + the first global column over all blocks, else 0"""
    for (c0, _), k in block_infos:
        if k > M:
            return k + c0
    return 0


def run(core, B, X, nrhs, v):
    """The block rule on the collected M x nrhs B and X (X None: output only): core(c0, Bk, Xk) -> (Xk refined or solved,
    dict of per-column outputs, info) on the w columns of one block alone.  Returns (X, per-column outputs concatenated
    by column, info merged as merge_info)."""
    M = B.shape[0]
    Xo = np.empty((M, nrhs))
    outs, infos = {}, []
    for c0, w in blocks(nrhs, v):
        xk, out, k = core(c0, B[:, c0:c0 + w].copy(), None if X is None else X[:, c0:c0 + w].copy())
        Xo[:, c0:c0 + w] = xk
        for name, val in out.items():
            if val is not None:
                outs.setdefault(name, []).append(val)
        infos.append(((c0, w), k))
    return Xo, {n: np.concatenate(v_) for n, v_ in outs.items()}, merge_info(infos, M)


def distribute(kind, G, v, Px=1, Py=1, Pz=1, Kappa=None, pad=np.nan, ld_extra=0):
    """every rank's share of G in the layout of cflx_lu_solve_local (solve_local_ref.distribute)"""
    return solve_local_ref.distribute(kind, G, v, Px, Py, Pz, Kappa=Kappa, pad=pad, ld_extra=ld_extra)


def collect(kind, X_locals, M, nrhs, v, Px=1, Py=1, Pz=1, Kappa=None):
    """the M x nrhs matrix whose layer-0 shares are X_locals (solve_local_ref.collect)"""
    return solve_local_ref.collect(kind, X_locals, M, nrhs, v, Px, Py, Pz, Kappa=Kappa)
