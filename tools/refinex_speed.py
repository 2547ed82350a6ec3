"""Times cflx_*_refine_x against the working-precision refinement and the plain solve, and the double-double residual
kernel against the FP64 one, at C2 (N = 16384, v = 256, one GPU).  Prints the card and its power limit first.

    python tools/refinex_speed.py [--N 16384] [--v 256] [--reps 10]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import conflux_b200 as cb  # noqa: E402


def timed(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--v", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(a.N, a.N, a.v, 1, 1, 1, comm)
    A = gv.data
    rng = np.random.default_rng(0)
    print("kernel (one share, Ml = Nl = %d): ms, GB/s of A, FP64 Gop/s (10 per entry and column)" % a.N)
    for nrhs in (1, 16, 64):
        X = rng.standard_normal((a.N, nrhs))
        _, _, ms_w = cb.dbg.residual(A, "nn", a.v, Xc=X, reps=a.reps)
        _, _, ms_x = cb.dbg.residual_x(A, "nn", a.v, Xc=X, Xc_tail=X * 1e-17, reps=a.reps)
        _, _, ms_t = cb.dbg.residual_x(A, "tn", a.v, Xr=X, Xr_tail=X * 1e-17, reps=a.reps)
        gb = A.size * 8 / 1e9
        ops = 10.0 * A.size * nrhs / 1e9
        print(f"  nrhs={nrhs:3d}  fp64 nn {ms_w:8.3f}  dd nn {ms_x:8.3f} ({gb / ms_x * 1e3:6.0f} GB/s, "
              f"{ops / ms_x * 1e3:7.0f} Gop/s)  dd tn {ms_t:8.3f} ({gb / ms_t * 1e3:6.0f} GB/s, {ops / ms_t * 1e3:7.0f} Gop/s)")
    cb.LU_rep(gv)
    print("end to end (ms per call):")
    for nrhs in (1, 16):
        B = rng.standard_normal((gv.M, nrhs))
        X0 = cb.lu_solve(gv, B)
        t_s = timed(lambda: cb.lu_solve(gv, B), a.reps)
        t_r = timed(lambda: cb.lu_refine(gv, B, X0), a.reps)
        t_x = timed(lambda: cb.lu_refine_x(gv, B, X0), a.reps)
        t_n = timed(lambda: cb.lu_refine_x(gv, B, X0, cwise=False), a.reps)
        print(f"  nrhs={nrhs:3d}  solve {t_s:8.2f}  refine(ferr) {t_r:8.2f}  refine_x {t_x:8.2f}  refine_x(cwise=False) {t_n:8.2f}")
    gv.free_comms()
    comm.close()


if __name__ == "__main__":
    main()
