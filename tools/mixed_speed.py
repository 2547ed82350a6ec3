"""tools/mixed_speed.py -- the mixed-precision drivers (cflx_lu_sv_mixed / cflx_chol_sv_mixed) on one GPU.

Prints the card, its power limit and SM clocks, then:
(a) the trailing update alone at the C2 step-0 shape, 16128 x 16128 x 256: the TF32 kernel with one and three terms
    (cb.dbg.gemm_tf32, CUDA events over --reps launches, the split timed apart) against the FP64 kernel
    (cb.dbg.gemm_tn_window in place, C at the factorisation's leading dimension 16384), as FP64-equivalent TFLOP/s
    2 M N K / time;
(b) end to end at C2 (N = 16384, v = 256, 1x1x1), host clock around calls that synchronise, input already on the
    device: chol sv_mixed (tf32, tf32x3) against parallelCholesky + solve + refine(ferr=False) on the generator's input,
    and lu_sv_mixed against LU_rep + lu_solve + lu_refine(ferr=False) on the generator's input + N I; nrhs 1 and 64,
    the variants alternating, --reps runs each, medians; iterations and the normwise backward errors
    max_j ||b - A x||_inf / (||A||_inf ||x||_inf) printed.
--json PATH also writes everything as JSON."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import conflux_b200 as cb
from tools.cond_speed import card

N, V = 16384, 256


def wall(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def berr(A, X, B):
    X2, B2 = X.reshape(len(B), -1), B.reshape(len(B), -1)
    return float(np.max(np.abs(B2 - A @ X2).max(axis=0) / (np.abs(A).sum(axis=1).max() * np.abs(X2).max(axis=0))))


def part_a(reps):
    rng = np.random.default_rng(2024)
    M = N - V
    AT, B = rng.uniform(-1, 1, (V, M)), rng.uniform(-1, 1, (V, M))
    C = rng.uniform(-1, 1, (M, N))
    flop = 2.0 * M * M * V
    out = {}
    for terms in (1, 3):
        r = cb.dbg.gemm_tf32(terms, AT, B, C[:, :M], reps=reps)
        out[f"tf32x{terms}"] = dict(ms=r["ms"], split_ms=r["split_ms"], tflops=flop / (r["ms"] * 1e-3) / 1e12)
        del r
    _, _, ms = cb.dbg.gemm_tn_window(AT, B, C, M, M, V, -1.0, 1.0, at_off=(0, 0), b_off=(0, 0), c_off=(0, 0),
                                     in_place=True, reps=reps)
    out["fp64"] = dict(ms=ms, tflops=flop / (ms * 1e-3) / 1e12)
    return dict(M=M, N=M, K=V, **out)


def part_b(comm, kind, nrhs, reps):
    rng = np.random.default_rng(nrhs)
    if kind == "chol":
        h = cb.cholesky(N, V, (1, 1, 1), comm)
        A = np.tril(h.data) + np.tril(h.data, -1).T
        up = lambda: cb.check(cb.lib().cflx_chol_set_local(h._h, np.ascontiguousarray(h.data).ctypes.data), "set")  # noqa: E731

        def fp64(B):
            h.parallelCholesky(upload=False)
            X = h.solve(B)
            return h.refine(B, X, ferr=False)[0], None

        def mixed(B, prec):
            X, it, _ = h.sv_mixed(B, prec=prec, upload=False)
            return X, it
    else:
        h = cb.lu_params(N, N, V, 1, 1, 1, comm)
        h.data[np.diag_indices(N)] += N
        A = h.data
        up = lambda: cb.check(cb.lib().cflx_lu_set_local(h._h, np.ascontiguousarray(h.data).ctypes.data), "set")  # noqa: E731

        def fp64(B):
            cb.LU_rep(h, upload=False)
            X = cb.lu_solve(h, B)
            return cb.lu_refine(h, B, X, ferr=False)[0], None

        def mixed(B, prec):
            X, it, _ = cb.lu_sv_mixed(h, B, prec=prec, upload=False)
            return X, it
    up()
    B = rng.standard_normal((N, nrhs))
    variants = {"fp64": lambda: fp64(B), "tf32": lambda: mixed(B, "tf32"), "tf32x3": lambda: mixed(B, "tf32x3")}
    for f in variants.values():  # warm-up
        f()
    times = {k: [] for k in variants}
    last = {}
    for _ in range(reps):
        for k, f in variants.items():
            ms, last[k] = wall(f)
            times[k].append(ms)
    res = dict(kind=kind, nrhs=nrhs)
    for k in variants:
        X, it = last[k]
        res[k] = dict(ms=statistics.median(times[k]), all=[round(t, 2) for t in times[k]], iter=it, berr=berr(A, X, B))
    if kind == "chol":
        h.finalize()
    else:
        h.free_comms()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    rec = dict(tool="mixed_speed", card=card())
    print(json.dumps(rec["card"]), flush=True)
    rec["kernel"] = part_a(max(a.reps, 10))
    print(json.dumps(rec["kernel"]), flush=True)
    comm = cb.Comm(1, 0, None, 0)
    rec["e2e"] = []
    for kind in ("chol", "lu"):
        for nrhs in (1, 64):
            r = part_b(comm, kind, nrhs, a.reps)
            rec["e2e"].append(r)
            print(json.dumps(r), flush=True)
    comm.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
