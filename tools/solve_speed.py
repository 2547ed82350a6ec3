"""tools/solve_speed.py -- cflx_lu_solve at the C2 size (N=16384, v=256, one GPU) and its narrow GEMM alone.

Prints the card and its power limit, the first solve after the factorisation (prepare included) and the median of 10
later solves for several right-hand-side counts (host clock around the synchronous call), and the narrow GEMM at
16128 x 64 x 256 against a device-to-device copy measured in the same run."""
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import conflux_b200 as cb


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q or torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def copy_gbs(nbytes, reps=20):
    src = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")
    dst = torch.empty_like(src)
    dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dst.copy_(src)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return 2 * nbytes / (ms * 1e-3) / 1e9        # read + write


def main():
    print(f"card: {card()}")
    N, v = 16384, 256
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    ms = cb.LU_rep(gv)
    print(f"factor C2: {ms:.1f} ms")
    rng = np.random.default_rng(0)
    first = True
    for nrhs in (1, 16, 64, 256):
        B = rng.standard_normal((gv.M, nrhs))
        t0 = time.perf_counter()
        X = cb.lu_solve(gv, B)
        t_first = (time.perf_counter() - t0) * 1e3
        ts = []
        for _ in range(10):
            t0 = time.perf_counter()
            cb.lu_solve(gv, B)
            ts.append((time.perf_counter() - t0) * 1e3)
        b, x = B[:, :4], X[:, :4]
        eta = np.linalg.norm(b - gv.data @ x) / (np.linalg.norm(gv.data) * np.linalg.norm(x) + np.linalg.norm(b))
        label = "first call (prepare included)" if first else "first call with this nrhs"
        print(f"solve nrhs={nrhs:4d}: {label} {t_first:8.2f} ms, median of 10 {statistics.median(ts):7.2f} ms "
              f"(min {min(ts):.2f}), eta {eta:.1e}")
        first = False
    gv.free_comms()
    comm.close()

    M, Nn, K = 16128, 64, 256
    A = rng.standard_normal((M, K))
    Bn = rng.standard_normal((K, Nn))
    C = rng.standard_normal((M, Nn))
    _, ms = cb.dbg.gemm_narrow(A, Bn, C, -1.0, 1.0, reps=50)
    a_bytes = A.nbytes
    total = a_bytes + 2 * C.nbytes + Bn.nbytes
    cp = copy_gbs(a_bytes)
    print(f"gemm_narrow {M} x {Nn} x {K} (D = C - A B): {ms * 1e3:.1f} us, A at {a_bytes / (ms * 1e-3) / 1e9:.0f} GB/s, "
          f"all operands {total / (ms * 1e-3) / 1e9:.0f} GB/s, {2.0 * M * Nn * K / (ms * 1e-3) / 1e12:.1f} TFLOP/s; "
          f"device-to-device copy of {a_bytes / 2**20:.0f} MiB: {cp:.0f} GB/s (read + write)")
    for Nn in (8, 16, 32):
        Bn = rng.standard_normal((K, Nn))
        C = rng.standard_normal((M, Nn))
        _, ms = cb.dbg.gemm_narrow(A, Bn, C, -1.0, 1.0, reps=50)
        print(f"gemm_narrow {M} x {Nn} x {K}: {ms * 1e3:.1f} us, A at {a_bytes / (ms * 1e-3) / 1e9:.0f} GB/s")


if __name__ == "__main__":
    main()
