"""tools/solve_local_speed.py -- the distributed-right-hand-side solves at the C2 size (N=16384, v=256, one GPU).

Prints the card, its power limit and SM clocks; then for the LU at nrhs in {64, 2048, 16384}: the median host-clock time of
lu_solve_local on torch CUDA shares (device in, device out) and of lu_solve on host B / X of the same columns, each with
the device memory the call adds to the solve cache (torch.cuda.mem_get_info before and after its first call, on a handle
whose solve data is already prepared by a one-column solve).  At nrhs = M the LU inverse (device output) is timed on the
same factors, and the Cholesky's solve_local at nrhs = M against its inverse.  The flop counts are 2 M^2 nrhs for a
solve, 4/3 M^3 for dgetri and 2/3 M^3 for dpotri."""
import argparse
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import conflux_b200 as cb
from tools.cond_speed import card


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def first_and_median(fn, reps):
    """(device memory the first call keeps, in MiB; median ms of `reps` further calls)"""
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    fn()
    torch.cuda.synchronize()
    grown = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 20
    return grown, statistics.median(timed(fn) for _ in range(reps))


def tf(flops, ms):
    return flops / (ms * 1e-3) / 1e12


def lu_case(N, v, nrhs, reps, comm):
    rng = np.random.default_rng(nrhs)
    res = {}
    for how in ("local", "host"):                                  # a fresh handle each: the solve cache starts small
        h = cb.lu_params(N, N, v, 1, 1, 1, comm)
        cb.LU_rep(h)
        M = h.M
        cb.lu_solve(h, np.ones(M))                                 # the solve data: factors redistributed, inverses
        if how == "local":
            ncl = cb.rhs_local_cols(nrhs, v, h.Py)
            B = torch.from_numpy(rng.standard_normal((h.Ml, ncl))).cuda()
            X = torch.empty_like(B)
            res[how] = first_and_median(lambda: cb.lu_solve_local(h, B, nrhs, out=X), reps)
            if nrhs == M:
                inv = torch.empty((h.Ml, h.Nl), dtype=torch.float64, device="cuda")
                cb.lu_inverse(h, inv)
                res["inverse"] = (0.0, statistics.median(timed(lambda: cb.lu_inverse(h, inv)) for _ in range(reps)))
                del inv
            del B, X
        else:
            Bh = rng.standard_normal((M, nrhs))
            res[how] = first_and_median(lambda: cb.lu_solve(h, Bh), reps)
        h.free_comms()
        torch.cuda.empty_cache()
    flops = 2.0 * M * M * nrhs
    line = (f"lu   N={M} v={v} nrhs={nrhs:6d}: solve_local device shares {res['local'][1]:9.1f} ms "
            f"({tf(flops, res['local'][1]):5.2f} TFLOP/s, cache +{res['local'][0]:7.0f} MiB) | lu_solve host B/X "
            f"{res['host'][1]:9.1f} ms ({tf(flops, res['host'][1]):5.2f} TFLOP/s, cache +{res['host'][0]:7.0f} MiB)")
    if "inverse" in res:
        t = res["inverse"][1]
        line += f" | lu_inverse device out {t:8.1f} ms ({tf(4.0 / 3.0 * M ** 3, t):5.2f} TFLOP/s), " \
                f"solve_local / inverse {res['local'][1] / t:4.2f}"
    print(line, flush=True)


def chol_case(N, v, reps, comm):
    h = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    h.parallelCholesky()
    M = h.N
    h.solve(np.ones(M))
    B = torch.from_numpy(np.random.default_rng(1).standard_normal((h.Ml, h.Nl))).cuda()
    X = torch.empty_like(B)
    grown, t = first_and_median(lambda: h.solve_local(B, M, out=X), reps)
    inv = torch.empty_like(B)
    h.inverse(inv)
    ti = statistics.median(timed(lambda: h.inverse(inv)) for _ in range(reps))
    print(f"chol N={M} v={v} nrhs={M:6d}: solve_local device shares {t:9.1f} ms ({tf(2.0 * M ** 3, t):5.2f} TFLOP/s, "
          f"cache +{grown:7.0f} MiB) | cholesky.inverse device out {ti:8.1f} ms ({tf(2.0 / 3.0 * M ** 3, ti):5.2f} "
          f"TFLOP/s), solve_local / inverse {t / ti:4.2f}", flush=True)
    h.finalize()
    del B, X, inv
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--v", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--nrhs", default="64,2048,16384")
    a = ap.parse_args()
    torch.cuda.init()
    print(f"card: {card()}", flush=True)
    comm = cb.Comm(1, 0, None, 0)
    for n in a.nrhs.split(","):
        lu_case(a.N, a.v, int(n), a.reps, comm)
    chol_case(a.N, a.v, a.reps, comm)
    comm.close()


if __name__ == "__main__":
    main()
