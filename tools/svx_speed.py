"""tools/svx_speed.py -- equilibration and the expert drivers at the C2 size (N=16384, v=256, one GPU).

Prints the card, its power limit and SM clocks; then the median (host clock around the synchronous call) of
lu_equilibrate(upload=False) and cholesky.equilibrate(upload=False) with the rate implied by the bytes their passes move
(LU: the row pass, the column pass and the apply pass each read the share once, the apply pass writes it once; Cholesky:
the apply pass reads and writes the lower triangle once; both on a matrix that forces scaling); then, after factoring the
equilibrated matrix, lu_svx and cholesky.svx at nrhs = 1, 16, 64 against solve + rcond + refine called separately on the
same factors."""
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import conflux_b200 as cb
from tools.cond_speed import card


def wall(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def main():
    torch.cuda.init()
    print(f"card: {card()}")
    N, v = 16384, 256
    comm = cb.Comm(1, 0, None, 0)
    rng = np.random.default_rng(0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    share = 8.0 * gv.Ml * gv.Nl
    rows = np.logspace(0, 8, N)
    rng.shuffle(rows)
    gv.data *= rows[:, None]                                       # rowcnd < 0.1: the apply pass runs ('R' or 'B')
    a = np.ascontiguousarray(gv.data)

    def lu_eq():
        cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
        t0 = time.perf_counter()
        e = cb.lu_equilibrate(gv, upload=False)
        return (time.perf_counter() - t0) * 1e3, e["equed"]
    ts = [lu_eq() for _ in range(5)]
    ms = statistics.median(t for t, _ in ts)
    print(f"lu_equilibrate C2 (equed {ts[0][1]}): {ms:.2f} ms, {4 * share / (ms * 1e-3) / 1e12:.2f} TB/s "
          f"(4 x {share / 2**30:.1f} GiB)")
    cb.LU_rep(gv, upload=False)                                    # the equilibrated row-scaled matrix: svx runs with 'R'
    for nrhs in (1, 16, 64):
        B = rng.standard_normal((gv.M, nrhs))
        cb.lu_svx(gv, B)
        sep = wall(lambda: (cb.lu_refine(gv, B, cb.lu_solve(gv, B)), cb.lu_rcond(gv)), 3)
        svx = wall(lambda: cb.lu_svx(gv, B), 3)
        print(f"lu nrhs={nrhs:3d}: svx {svx:8.2f} ms, solve + rcond + refine {sep:8.2f} ms")
    gv.free_comms()

    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    s = np.logspace(0, 3, ch.N)
    rng.shuffle(s)
    ch.data *= s[:, None] * s[None, :]                             # scond < 0.1: the apply pass runs
    c = np.ascontiguousarray(ch.data)

    def ch_eq():
        cb.check(cb.lib().cflx_chol_set_local(ch._h, c.ctypes.data), "set_local")
        t0 = time.perf_counter()
        e = ch.equilibrate(upload=False)
        return (time.perf_counter() - t0) * 1e3, e["equed"]
    ts = [ch_eq() for _ in range(5)]
    ms = statistics.median(t for t, _ in ts)
    low = 8.0 * ch.N * (ch.N + v) / 2
    print(f"cholesky.equilibrate C2 (equed {ts[0][1]}): {ms:.2f} ms, {2 * low / (ms * 1e-3) / 1e12:.2f} TB/s "
          f"(2 x {low / 2**30:.1f} GiB)")
    ch.parallelCholesky(upload=False)                              # the equilibrated matrix: svx runs with 'Y'
    for nrhs in (1, 16, 64):
        B = rng.standard_normal((ch.N, nrhs))
        ch.svx(B)
        sep = wall(lambda: (ch.refine(B, ch.solve(B)), ch.rcond()), 3)
        svx = wall(lambda: ch.svx(B), 3)
        print(f"chol nrhs={nrhs:3d}: svx {svx:8.2f} ms, solve + rcond + refine {sep:8.2f} ms")
    ch.finalize()
    comm.close()


if __name__ == "__main__":
    main()
