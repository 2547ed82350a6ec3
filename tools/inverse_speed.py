"""tools/inverse_speed.py -- the explicit inverse at the C2 size (N=16384, v=256, one GPU).

Prints the card, its power limit and SM clocks; then for the LU (v = 256) and the Cholesky (v = 256 and 512): the
factorisation's time (host clock around the synchronous call), and the median host-clock time of lu_inverse /
cholesky.inverse writing into a torch CUDA tensor (device output) and into a NumPy array (host output), with the rate at
LAPACK's flop counts (4/3 M^3 for dgetri, 2/3 M^3 for dpotri) and the ratio to the factorisation.

The block width is the compiled constant CFLX_INV_NC (csrc/lu_state.h).  To compare widths, build the library with
`-DCFLX_INV_NC=<n>` added to the nvcc flags and pass it with --lib <path to libconflux_b200.so>; --label names the run."""
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


def run(kind, N, v, reps, comm):
    if kind == "lu":
        h = cb.lu_params(N, N, v, 1, 1, 1, comm)
        M, shape = h.M, (h.Ml, h.Nl)
        fac = timed(lambda: cb.LU_rep(h))
        inv = lambda out: cb.lu_inverse(h, out)                     # noqa: E731
        flops = 4.0 / 3.0 * M ** 3
    else:
        h = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
        M, shape = h.N, (h.Ml, h.Nl)
        fac = timed(lambda: h.parallelCholesky())
        inv = lambda out: h.inverse(out)                            # noqa: E731
        flops = 2.0 / 3.0 * M ** 3
    dev = torch.empty(shape, dtype=torch.float64, device="cuda")
    host = np.empty(shape)
    inv(dev)                                                        # warm-up: the solve cache and every launch shape
    t_dev = statistics.median(timed(lambda: inv(dev)) for _ in range(reps))
    t_host = statistics.median(timed(lambda: inv(host)) for _ in range(reps))
    assert np.array_equal(dev.cpu().numpy(), host)
    print(f"{kind:4s} N={M} v={v}: factor {fac:8.1f} ms | inverse device out {t_dev:8.1f} ms "
          f"({flops / (t_dev * 1e-3) / 1e12:5.2f} TFLOP/s, {t_dev / fac:5.2f}x factor) | host out {t_host:8.1f} ms "
          f"({flops / (t_host * 1e-3) / 1e12:5.2f} TFLOP/s)", flush=True)
    if kind == "lu":
        h.free_comms()
    else:
        h.finalize()
    del dev
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="a libconflux_b200.so built with another -DCFLX_INV_NC")
    ap.add_argument("--label", default="")
    ap.add_argument("--N", type=int, default=16384)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="lu,chol256,chol512")
    a = ap.parse_args()
    if a.lib:
        cb._lib.LIB_PATH = os.path.abspath(a.lib)
    torch.cuda.init()
    print(f"card: {card()}  library: {cb._lib.LIB_PATH} {a.label}", flush=True)
    comm = cb.Comm(1, 0, None, 0)
    for what in a.only.split(","):
        if what == "lu":
            run("lu", a.N, 256, a.reps, comm)
        else:
            run("chol", a.N, int(what[4:]), a.reps, comm)
    comm.close()


if __name__ == "__main__":
    main()
