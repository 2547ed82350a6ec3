"""Times cflx_lu_equilibrate_b against cflx_lu_equilibrate on the same row-graded input, the per-column pivot growth
pass, and cflx_lu_svxx against cflx_lu_solve + cflx_lu_refine_x on the same factors, at C2 (N = 16384, v = 256, one
GPU).  Prints the card and its power limit first.  The growth pass is timed from the kernel records of torch.profiler
(CUDA activities) over svxx calls.

    python tools/svxx_speed.py [--N 16384] [--v 256] [--reps 5]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch  # noqa: F401  (first: conflux_b200 then shares torch's NCCL)
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import conflux_b200 as cb  # noqa: E402


def timed(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps * 1e3


def kernel_ms(fn, reps, name):
    """mean device ms of the kernels whose name contains `name`, over reps calls of fn, and their count per call"""
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    tot, cnt = 0.0, 0
    for e in prof.key_averages():
        if name in e.key:
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            cnt += e.count
    return (tot / cnt / 1e3 if cnt else float("nan")), cnt / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--v", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(a.N, a.N, a.v, 1, 1, 1, comm)
    rng = np.random.default_rng(0)
    gv.data *= np.exp2(rng.uniform(-20, 20, gv.M))[:, None]             # row-graded: both scalings apply 'R'
    data = np.ascontiguousarray(gv.data)
    print(f"equilibration, one call with apply = 1 after an untimed upload (ms), N = {a.N}:")
    for what, fn in (("equilibrate  ", cb.lu_equilibrate), ("equilibrate_b", cb.lu_equilibrate_b)):
        ts = []
        for _ in range(a.reps + 1):
            cb.check(cb.lib().cflx_lu_set_local(gv._h, data.ctypes.data), "lu_set_local")
            t = time.perf_counter()
            e = fn(gv, upload=False)
            ts.append((time.perf_counter() - t) * 1e3)
        print(f"  {what}  min {min(ts[1:]):7.2f}  median {float(np.median(ts[1:])):7.2f}  equed {e['equed']}")
    cb.LU_rep(gv, upload=False)                                          # the factors of the last scaled input
    B1 = rng.standard_normal((gv.M, 1))
    try:
        ms, per_call = kernel_ms(lambda: cb.lu_svxx(gv, B1), a.reps, "growth_cols_kernel")
        gb = 1.5 * gv.Ml * gv.Nl * 8 / 1e9                               # A0, and U: the factor's upper triangle
        print(f"growth pass (kernel, {per_call:.0f} per svxx call): {ms:.3f} ms, {gb / ms * 1e3:.0f} GB/s of A0 and U")
    except Exception as ex:                                              # the profiler is unavailable: not measured
        print(f"growth pass: not measured ({ex})")
    print("end to end (ms per call):")
    for nrhs in (1, 16, 64):
        B = rng.standard_normal((gv.M, nrhs))
        t_x = timed(lambda: cb.lu_svxx(gv, B), a.reps)
        Bs = e["r"][:, None] * B if e["equed"] in "RB" else B            # the system svxx solves: the same rounds
        X0 = cb.lu_solve(gv, Bs)
        t_s = timed(lambda: cb.lu_solve(gv, Bs), a.reps)
        t_r = timed(lambda: cb.lu_refine_x(gv, Bs, X0), a.reps)
        print(f"  nrhs={nrhs:3d}  svxx {t_x:8.2f}  solve {t_s:8.2f}  refine_x {t_r:8.2f}  solve + refine_x {t_s + t_r:8.2f}")
    gv.free_comms()
    comm.close()


if __name__ == "__main__":
    main()
