"""tools/refine_speed.py -- iterative refinement at the C2 size (N=16384, v=256, one GPU).

Prints the card, its power limit and SM clocks; then, after one LU factorisation, for nrhs = 1, 16, 64, 256 the median
(host clock around the synchronous call) of the plain solve and of lu_refine with and without the forward-error
estimator, started from the solve's X; then dbg.residual on the C2 share in each mode (NN, TN, and the symmetric-lower
mode on the Cholesky generator's share) with its read rate of A, against the 1-norm kernel's 2.99 TB/s and the 3.35 TB/s
data-sheet figure."""
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
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    print(f"LU factor C2: {cb.LU_rep(gv):.1f} ms")
    rng = np.random.default_rng(0)
    for nrhs in (1, 16, 64, 256):
        B = rng.standard_normal((gv.M, nrhs))
        X = cb.lu_solve(gv, B)
        cb.lu_refine(gv, B, X)
        s = wall(lambda: cb.lu_solve(gv, B), 5)
        r = wall(lambda: cb.lu_refine(gv, B, X, ferr=False), 5)
        f = wall(lambda: cb.lu_refine(gv, B, X), 3)
        _, fe, be = cb.lu_refine(gv, B, X)
        print(f"nrhs={nrhs:4d}: solve {s:8.2f} ms, refine {r:8.2f} ms, refine+ferr {f:8.2f} ms; "
              f"berr max {be.max():.1e}, ferr max {fe.max():.1e}")
    A = np.ascontiguousarray(gv.data)
    gv.free_comms()
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    S = np.ascontiguousarray(ch.data)
    ch.finalize()
    nbytes = 8.0 * A.size
    for nrhs in (1, 16, 64, 256):
        X = rng.standard_normal((N, nrhs))
        for mode, share, kw in (("nn", A, dict(Xc=X)), ("tn", A, dict(Xr=X)), ("sym", S, dict(Xc=X, Xr=X))):
            _, _, ms = cb.dbg.residual(share, mode, v, N // v, reps=10, **kw)
            read = nbytes / 2 if mode == "sym" else nbytes     # the symmetric mode reads the lower triangle, twice
            rate = (2 * read if mode == "sym" else read) / (ms * 1e-3) / 1e12
            print(f"residual {mode:3s} nrhs={nrhs:4d}: {ms:7.3f} ms, {rate:.2f} TB/s of A read "
                  f"({rate / 2.99:.2f}x the 1-norm kernel, {rate / 3.35:.2f}x 3.35 TB/s)")
    comm.close()


if __name__ == "__main__":
    main()
