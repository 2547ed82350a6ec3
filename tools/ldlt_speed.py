"""tools/ldlt_speed.py -- the signed Cholesky (cflx_chol_factor_ldlt) and the symmetric butterflies on one GPU.

Prints the card, its power limit and SM clocks, then:
(a) cflx_chol_factor against factor_ldlt on the generator's SPD input, N = 16384, v = 256 and 512: the factorisation
    loop's device ms, the two variants alternating, `--reps` runs each, medians;
(b) on the generator's matrix shifted by -sigma I (sigma = its diagonal value, so that about half the eigenvalues are
    negative), end to end with the upload excluded (host clock around calls that synchronise): rbt + factor_ldlt +
    rbt_solve(refine) against LU_rep + lu_svx, at nrhs = 1 and 64, alternating, medians; with the backward error
    max_i |b - A x|_i / (|A| |x| + |b|)_i of both solutions on A and their largest relative forward difference.
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


def wall(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def berr(A, X, B):
    X2, B2 = X.reshape(len(B), -1), B.reshape(len(B), -1)
    return float(np.max(np.abs(A @ X2 - B2) / (np.abs(A) @ np.abs(X2) + np.abs(B2))))


def part_a(comm, N, v, reps):
    ch = cb.cholesky(N, v, (1, 1, 1), comm)
    ch.parallelCholesky()
    ch.factor_ldlt()       # warm-up of both
    chol, ldlt = [], []
    for _ in range(reps):
        chol.append(ch.parallelCholesky(upload=False))
        ldlt.append(ch.factor_ldlt(upload=False)[3])
    ch.finalize()
    return dict(N=N, v=v, chol_ms=statistics.median(chol), ldlt_ms=statistics.median(ldlt), chol_all=chol, ldlt_all=ldlt)


def part_b(comm, N, v, reps):
    ch = cb.cholesky(N, v, (1, 1, 1), comm)
    sigma = float(ch.data[0, 0])
    low = np.tril(ch.data)
    low[np.diag_indices(N)] -= sigma
    ch.data[...] = low
    A = low + np.tril(low, -1).T
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    gv.data[...] = A
    rng = np.random.default_rng(0)
    out = dict(N=N, v=v, sigma=sigma)
    for nrhs in (1, 64):
        B = rng.standard_normal((N, nrhs))

        def rbt():
            ch.rbt(depth=2, seed=0, upload=False)
            r = ch.factor_ldlt(upload=False)
            X, _, _ = ch.rbt_solve(B)
            return X, r

        def lu():
            cb.LU_rep(gv, upload=False)
            X, d = cb.lu_svx(gv, B)
            return X
        t_r, t_l = [], []
        ca, la = np.ascontiguousarray(ch.data), np.ascontiguousarray(gv.data)
        for _ in range(reps + 1):                      # the first run of each is a warm-up
            cb._lib.check(cb._lib.lib().cflx_chol_set_local(ch._h, ca.ctypes.data), "chol_set_local")
            dt, (Xr, fac) = wall(rbt)
            t_r.append(dt)
            cb._lib.check(cb._lib.lib().cflx_lu_set_local(gv._h, la.ctypes.data), "lu_set_local")
            dt, Xl = wall(lu)
            t_l.append(dt)
        out[f"nrhs{nrhs}"] = dict(rbt_ms=statistics.median(t_r[1:]), lu_ms=statistics.median(t_l[1:]),
                                  rbt_berr=berr(A, Xr, B), lu_berr=berr(A, Xl, B),
                                  fwd_diff=float(np.max(np.abs(Xr - Xl)) / np.max(np.abs(Xl))),
                                  ldlt=dict(nrepl=fac[0], inertia=fac[1], info=fac[2]))
    gv.free_comms()
    ch.finalize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json")
    a = ap.parse_args()
    res = dict(card=card(), a=[], b=None)
    print("card:", res["card"])
    comm = cb.Comm(1, 0, None, 0)
    for v in (256, 512):
        r = part_a(comm, a.N, v, a.reps)
        res["a"].append(r)
        print(f"(a) N={r['N']} v={v}: chol_factor {r['chol_ms']:.2f} ms  factor_ldlt {r['ldlt_ms']:.2f} ms  "
              f"({100 * (r['ldlt_ms'] / r['chol_ms'] - 1):+.1f} %)")
    res["b"] = part_b(comm, a.N, 256, a.reps)
    for k in ("nrhs1", "nrhs64"):
        r = res["b"][k]
        print(f"(b) {k}: rbt+ldlt+rbt_solve {r['rbt_ms']:.1f} ms  LU_rep+lu_svx {r['lu_ms']:.1f} ms  "
              f"berr {r['rbt_berr']:.1e} / {r['lu_berr']:.1e}  fwd diff {r['fwd_diff']:.1e}  {r['ldlt']}")
    comm.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
