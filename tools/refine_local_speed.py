"""tools/refine_local_speed.py -- the distributed refinement and expert drivers at the C2 size (N=16384, v=256, one GPU).

Prints the card, its power limit and SM clocks; then for the LU at nrhs in {1, 64, 1024}, B and X as torch CUDA shares:
  * refine_local: lu_refine_local on the device shares, against gathering B and X into replicated host arrays, lu_refine
    and copying X back into its share;
  * svx_local: lu_svx_local on the device shares, against the same gather, lu_svx and copy back.
Each variant runs on a handle of its own, so the device memory its first call leaves allocated (cudaMemGetInfo before and
after: the refinement, equilibration and solve caches, which the drivers keep) is the variant's own; the temporaries a
call frees on return are not in that figure, so the workspace bound of the header is printed beside it.  The timed calls
alternate the variants in each round and report the median host-clock time of `reps` rounds, each call ending in a device
synchronise.  X is reset to the same solution before every refine call."""
import argparse
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import conflux_b200 as cb
from oracle import refine_local_ref as rl
from tools.cond_speed import card


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def kept_mib(fn):
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    fn()
    torch.cuda.synchronize()
    return (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 20


def case(N, v, nrhs, reps, comm):
    rng = np.random.default_rng(nrhs)
    names = ("refine_local", "refine gather", "svx_local", "svx gather")
    hs = {}
    for n in names:
        h = cb.lu_params(N, N, v, 1, 1, 1, comm)
        h.data[...] = np.random.default_rng(0).standard_normal((h.Ml, h.Nl))
        cb.LU_rep(h)
        cb.lu_solve(h, np.ones(h.M))                              # the solve data: factors redistributed, inverses
        hs[n] = h
    h0 = hs[names[0]]
    M, ncl = h0.M, cb.rhs_local_cols(nrhs, v, h0.Py)
    B = torch.from_numpy(rng.standard_normal((h0.Ml, ncl))).cuda()
    X0 = torch.from_numpy(np.ascontiguousarray(np.pad(cb.lu_solve(h0, B.cpu().numpy()[:, :nrhs]),
                                                      ((0, 0), (0, ncl - nrhs))))).cuda()
    X = torch.empty_like(B)

    def gather(t):                                                  # the share of a 1 x 1 x 1 grid is the matrix
        return np.ascontiguousarray(t.cpu().numpy()[:, :nrhs])

    def run(n):
        h = hs[n]
        if n.startswith("refine"):
            X.copy_(X0)
        if n == "refine_local":
            return lambda: cb.lu_refine_local(h, B, X, nrhs)
        if n == "svx_local":
            return lambda: cb.lu_svx_local(h, B, nrhs, out=X)
        if n == "refine gather":
            return lambda: X[:, :nrhs].copy_(torch.from_numpy(cb.lu_refine(h, gather(B), gather(X))[0]))
        return lambda: X[:, :nrhs].copy_(torch.from_numpy(cb.lu_svx(h, gather(B))[0]))

    kept = {n: kept_mib(run(n)) for n in names}
    ts = {n: [] for n in names}
    for _ in range(reps):
        for n in names:                                             # the variants alternate in every round
            fn = run(n)
            ts[n].append(timed(fn))
    w = min(rl.block_cols(v), nrhs)
    bound = rl.workspace_doubles(M, v, h0.Ml, h0.Nl, 1, w) * 8 / 2 ** 20
    for n in names:
        print(f"lu N={M} v={v} nrhs={nrhs:5d} {n:14s}: {statistics.median(ts[n]):9.1f} ms (median of {reps}), "
              f"device memory kept +{kept[n]:7.0f} MiB" + (f" (block workspace bound {bound:.0f} MiB)" if "local" in n
                                                            else ""), flush=True)
    for h in hs.values():
        h.free_comms()
    del B, X, X0
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--v", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--nrhs", default="1,64,1024")
    a = ap.parse_args()
    torch.cuda.init()
    print(f"card: {card()}", flush=True)
    comm = cb.Comm(1, 0, None, 0)
    for n in a.nrhs.split(","):
        case(a.N, a.v, int(n), a.reps, comm)
    comm.close()


if __name__ == "__main__":
    main()
