"""tools/rbt_speed.py -- random butterfly transforms at N = 16384 with v = 256 (C2) and v = 512, one GPU.

Prints the card, its power limit and SM clocks, then per tile size:
- the transform kernels of cflx_lu_rbt (depth 2: one fused pass), from torch.profiler's kernel records, and their
  achieved bytes/s (one read and one write of the share per pass) against the H100 SXM's 3.35 TB/s;
- LU_rep_rbt (the transform's wall time plus the fixed factorisation's main loop) against LU_rep's main loop;
- end to end, upload excluded, host clock around calls that synchronise: rbt + fixed factor + lu_rbt_solve(refine=True)
  against LU_rep + lu_svx, at nrhs = 1 and 64;
- accuracy at nrhs = 1: the backward error max_i |b - A x|_i / (|A| |x| + |b|)_i of the RBT solution before and after
  refinement and of lu_svx's, the forward difference to lu_svx's solution, and the reciprocal pivot growth of the RBT
  factors (lu_svx's rpvgrw on them) and of the pivoted ones.
The compared variants alternate, `--reps` runs each, medians.  --json PATH also writes everything as JSON."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import conflux_b200 as cb
from conflux_b200._lib import lib
from tools.cond_speed import card

HBM_TBS = 3.35   # H100 SXM data sheet


def upload(gv):
    lib().cflx_lu_set_local(gv._h, np.ascontiguousarray(gv.data).ctypes.data)


def transform_kernels_ms(gv, depth, reps):
    """median over reps of the summed durations of the rbt kernels of one cflx_lu_rbt call, and their count per call;
    one profiling session around every call"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for r in range(reps):
            upload(gv)
            cb._lib.check(lib().cflx_lu_rbt(gv._h, depth, r, None, None), "lu_rbt")
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel" and "rbt_kernel" in e["name"]]
    if not ev or len(ev) % reps:
        raise RuntimeError(f"expected the transform kernels of {reps} calls in the trace, found {len(ev)}")
    n = len(ev) // reps
    ev.sort(key=lambda e: e["ts"])
    return statistics.median(sum(e["dur"] for e in ev[i * n:(i + 1) * n]) / 1e3 for i in range(reps)), n


def wall(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def berr(A, X, B):
    return float(np.max(np.abs(B - A @ X) / (np.abs(A) @ np.abs(X) + np.abs(B))))


def compare(comm, N, v, reps, depth=2):
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    out = {}
    kms, nk = transform_kernels_ms(gv, depth, reps)
    passes = (depth + 1) // 2
    gbytes = passes * 2 * 8 * gv.Ml * gv.Nl / 1e9
    out["transform"] = dict(kernel_ms=kms, kernels=nk, gbytes=gbytes, tbs=gbytes / kms, share_of_hbm=gbytes / kms / HBM_TBS)
    print(f"N={N} v={v}: transform kernels {kms:.3f} ms ({nk} launches), {gbytes:.2f} GB, {gbytes / kms:.2f} TB/s "
          f"= {100 * gbytes / kms / HBM_TBS:.0f}% of {HBM_TBS} TB/s")

    ident = np.arange(gv.M, dtype=np.int32)

    def rbt_factor():
        upload(gv)
        t = wall(lambda: cb._lib.check(lib().cflx_lu_rbt(gv._h, depth, 0, None, None), "lu_rbt"))
        ms, _, info = cb.LU_rep_fixed(gv, perm=ident, upload=False)
        assert info == 0
        return t + ms

    def piv_factor():
        upload(gv)
        return cb.LU_rep(gv, upload=False)

    rbt_factor(), piv_factor()                                   # warm-up
    rb, pv = [], []
    for _ in range(reps):
        rb.append(rbt_factor())
        pv.append(piv_factor())
    out["factor"] = dict(rbt_ms=rb, pivoted_ms=pv, rbt_median=statistics.median(rb), pivoted_median=statistics.median(pv))
    print(f"    LU_rep_rbt (transform wall + fixed main loop) median {statistics.median(rb):.2f} ms "
          f"{['%.2f' % x for x in rb]}; LU_rep median {statistics.median(pv):.2f} ms {['%.2f' % x for x in pv]}")

    rng = np.random.default_rng(v)
    for nrhs in (1, 64):
        B = rng.standard_normal((gv.M, nrhs))

        def e2e_rbt():
            upload(gv)
            return wall(lambda: (cb._lib.check(lib().cflx_lu_rbt(gv._h, depth, 0, None, None), "lu_rbt"),
                                 cb.LU_rep_fixed(gv, perm=ident, upload=False), cb.lu_rbt_solve(gv, B)))

        def e2e_piv():
            upload(gv)
            return wall(lambda: (cb.LU_rep(gv, upload=False), cb.lu_svx(gv, B)))

        e2e_rbt(), e2e_piv()
        er, ep = [], []
        for _ in range(reps):
            er.append(e2e_rbt())
            ep.append(e2e_piv())
        out[f"e2e_nrhs{nrhs}"] = dict(rbt_ms=er, pivoted_ms=ep, rbt_median=statistics.median(er),
                                      pivoted_median=statistics.median(ep))
        print(f"    end to end nrhs={nrhs}: rbt + fixed + lu_rbt_solve median {statistics.median(er):.2f} ms; "
              f"LU_rep + lu_svx median {statistics.median(ep):.2f} ms")

    A = gv.data
    B = rng.standard_normal((gv.M, 1))
    upload(gv)
    cb.LU_rep(gv, upload=False)
    Xp, sp = cb.lu_svx(gv, B)
    cb.LU_rep_rbt(gv, depth=depth)
    X0, _, _ = cb.lu_rbt_solve(gv, B, refine=False)
    X1, ferr, be1 = cb.lu_rbt_solve(gv, B, refine=True)
    _, sr = cb.lu_svx(gv, B)                                    # its rpvgrw: the RBT factors' growth on W
    acc = dict(berr_rbt_unrefined=berr(A, X0, B), berr_rbt_refined=berr(A, X1, B), berr_pivoted_svx=berr(A, Xp, B),
               berr_rbt_transformed_system=float(be1.max()), ferr_rbt_transformed_system=float(ferr.max()),
               fwd_vs_pivoted=float(np.abs(X1 - Xp).max() / np.abs(Xp).max()),
               fwd_vs_pivoted_unrefined=float(np.abs(X0 - Xp).max() / np.abs(Xp).max()),
               rpvgrw_rbt=sr["rpvgrw"], rpvgrw_pivoted=sp["rpvgrw"], rcond_pivoted=sp["rcond"])
    out["accuracy"] = acc
    print("    accuracy:", json.dumps({k: float("%.3g" % x) for k, x in acc.items()}))
    gv.free_comms()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    out = {"card": card(), "N": a.n}
    print("card:", out["card"])
    torch.cuda.init()
    comm = cb.Comm(1, 0, None, 0)
    for v in (256, 512):
        out[f"v{v}"] = compare(comm, a.n, v, a.reps)
    comm.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
