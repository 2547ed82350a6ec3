"""tools/chol_solve_speed.py -- cflx_chol_solve at N=16384 on one GPU (v=256 and v=512) and its transposed narrow GEMM
against the NN one.

Prints the card and its power limit; per tile size the factorisation time, then for several right-hand-side counts the
first solve after the factorisation (prepare included) and the median of 10 later solves (host clock around the
synchronous call, upload of B and download of X included) with the backward error over the first 4 columns; and the two
narrow GEMMs at 16128 x {8, 16, 32, 64} x 256, which read the same bytes of their matrix operand (A, or AT in place)."""
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import conflux_b200 as cb
from oracle import chol_ref


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main():
    print(f"card: {card()}")
    N = 16384
    rng = np.random.default_rng(0)
    for v in (256, 512):
        comm = cb.Comm(1, 0, None, 0)
        ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
        ms = ch.parallelCholesky()
        S = chol_ref.lower_sym(ch.data)
        print(f"factor N={N} v={v}: {ms:.1f} ms")
        first = True
        for nrhs in (1, 16, 64, 256):
            B = rng.standard_normal((ch.N, nrhs))
            t0 = time.perf_counter()
            X = ch.solve(B)
            t_first = (time.perf_counter() - t0) * 1e3
            ts = []
            for _ in range(10):
                t0 = time.perf_counter()
                ch.solve(B)
                ts.append((time.perf_counter() - t0) * 1e3)
            b, x = B[:, :4], X[:, :4]
            eta = np.linalg.norm(b - S @ x) / (np.linalg.norm(S) * np.linalg.norm(x) + np.linalg.norm(b))
            label = "first call (prepare included)" if first else "first call with this nrhs"
            print(f"  solve nrhs={nrhs:4d}: {label} {t_first:8.2f} ms, median of 10 {statistics.median(ts):7.2f} ms "
                  f"(min {min(ts):.2f}), eta {eta:.1e}")
            first = False
        ch.finalize()
        comm.close()

    M, K = 16128, 256
    A = rng.standard_normal((M, K))
    AT = np.ascontiguousarray(A.T)
    a_bytes = A.nbytes
    for Nn in (8, 16, 32, 64):
        Bn = rng.standard_normal((K, Nn))
        C = rng.standard_normal((M, Nn))
        _, ms_nn = cb.dbg.gemm_narrow(A, Bn, C, -1.0, 1.0, reps=50)
        _, ms_tn = cb.dbg.gemm_narrow_tn(AT, Bn, C, -1.0, 1.0, reps=50)
        print(f"{M} x {Nn} x {K} (D = C - A B): NN {ms_nn * 1e3:6.1f} us, A at {a_bytes / (ms_nn * 1e-3) / 1e9:5.0f} GB/s;  "
              f"TN {ms_tn * 1e3:6.1f} us, AT at {a_bytes / (ms_tn * 1e-3) / 1e9:5.0f} GB/s")


if __name__ == "__main__":
    main()
