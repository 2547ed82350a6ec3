"""tools/cond_speed.py -- the transposed LU solve and the condition estimates at the C2 size (N=16384, v=256, one GPU).

Prints the card, its power limit and SM clocks; then, after one LU factorisation, the median of 10 plain and 10
transposed solves (alternating, host clock around the synchronous call) for nrhs = 1, 16, 64, 256; then the wall time of
cflx_lu_rcond and cflx_chol_rcond (median of 5), split into the 1-norm pass (device time of its two kernels, from one
profiled call) and the rest, which is the estimator's solves with one right-hand side."""
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import conflux_b200 as cb


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def wall(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def norm_kernel_ms(fn):
    """device time of the 1-norm kernels in one call of fn"""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = 0.0
    for e in prof.events():
        if "abs_sums_kernel" in e.name or "column_sums_kernel" in e.name:
            ms += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return ms


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
        cb.lu_solve(gv, B)
        X = cb.lu_solve(gv, B, trans=True)
        plain, trans = [], []
        for _ in range(10):
            plain.append(wall(lambda: cb.lu_solve(gv, B), 1))
            trans.append(wall(lambda: cb.lu_solve(gv, B, trans=True), 1))
        b, x = B[:, :4], X[:, :4]
        eta = np.linalg.norm(b - gv.data.T @ x) / (np.linalg.norm(gv.data) * np.linalg.norm(x) + np.linalg.norm(b))
        p, t = statistics.median(plain), statistics.median(trans)
        print(f"nrhs={nrhs:4d}: solve {p:7.2f} ms, transposed solve {t:7.2f} ms ({t / p:.2f}x), transposed eta {eta:.1e}")
    cb.lu_rcond(gv)
    r_ms = wall(lambda: cb.lu_rcond(gv), 5)
    n_ms = norm_kernel_ms(lambda: cb.lu_rcond(gv))
    rcond, anorm = cb.lu_rcond(gv)
    gbs = 8.0 * gv.Ml * gv.Nl / (n_ms * 1e-3) / 1e9 if n_ms > 0 else float("nan")
    print(f"lu_rcond: {r_ms:.2f} ms (1-norm kernels {n_ms:.3f} ms = {gbs:.0f} GB/s of the input; the rest: estimator "
          f"solves and host work), rcond {rcond:.3e}, anorm {anorm:.6e}")
    gv.free_comms()

    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    print(f"Cholesky factor N={N} v={v}: {ch.parallelCholesky():.1f} ms")
    b = rng.standard_normal(ch.N)
    ch.solve(b)
    s_ms = wall(lambda: ch.solve(b), 10)
    ch.rcond()
    r_ms = wall(lambda: ch.rcond(), 5)
    n_ms = norm_kernel_ms(lambda: ch.rcond())
    rcond, anorm = ch.rcond()
    gbs = 8.0 * ch.Ml * ch.Nl / (n_ms * 1e-3) / 1e9 if n_ms > 0 else float("nan")
    print(f"chol_rcond: {r_ms:.2f} ms (1-norm kernels {n_ms:.3f} ms = {gbs:.0f} GB/s of the local share; one solve "
          f"with nrhs=1 {s_ms:.2f} ms), rcond {rcond:.3e}, anorm {anorm:.6e}")
    ch.finalize()
    comm.close()


if __name__ == "__main__":
    main()
