"""tools/det_speed.py -- the determinant at the C2 size (N=16384, v=256, one GPU).

Prints the card, its power limit and SM clocks; then for the LU and the Cholesky: the factorisation's time (host clock
around the synchronous call), the first lu_det / cholesky.det after it (cold: the LU's call also prepares the solve
cache, which redistributes the factors into the conflux layout) and the median of the following calls (warm), each
timed by the host clock around the synchronous call, over --reps factorisations.  For scale, the median time of one
lu_solve / cholesky.solve with one right-hand side on the warm cache."""
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


def run(kind, N, v, reps, warm, comm):
    if kind == "lu":
        h = cb.lu_params(N, N, v, 1, 1, 1, comm)
        factor = lambda: cb.LU_rep(h, upload=False)                 # noqa: E731
        det = lambda: cb.lu_det(h)                                  # noqa: E731
        solve = lambda b: cb.lu_solve(h, b)                         # noqa: E731
        cb.LU_rep(h)
    else:
        h = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
        factor = lambda: h.parallelCholesky(upload=False)           # noqa: E731
        det = lambda: h.det()                                       # noqa: E731
        solve = lambda b: h.solve(b)                                # noqa: E731
        h.parallelCholesky()
    b = np.random.default_rng(0).standard_normal(N)
    fac, cold, hot = [], [], []
    for _ in range(reps):
        fac.append(timed(factor))
        cold.append(timed(det))
        hot += [timed(det) for _ in range(warm)]
    t_solve = statistics.median(timed(lambda: solve(b)) for _ in range(warm))
    o = det()
    print(f"{kind:4s} N={N} v={v}: factor {statistics.median(fac):8.1f} ms | det cold {statistics.median(cold):7.2f} ms "
          f"(min {min(cold):.2f}, max {max(cold):.2f}) | warm {statistics.median(hot):6.3f} ms (min {min(hot):.3f}, max "
          f"{max(hot):.3f}) | solve nrhs=1 {t_solve:6.2f} ms | log|det| {o.get('logabsdet', o.get('logdet')):.6e}",
          flush=True)
    if kind == "lu":
        h.free_comms()
    else:
        h.finalize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--v", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warm", type=int, default=20)
    ap.add_argument("--only", default="lu,chol")
    a = ap.parse_args()
    torch.cuda.init()
    print(f"card: {card()}", flush=True)
    comm = cb.Comm(1, 0, None, 0)
    for kind in a.only.split(","):
        run(kind, a.N, a.v, a.reps, a.warm, comm)
    comm.close()


if __name__ == "__main__":
    main()
