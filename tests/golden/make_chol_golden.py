"""tests/golden/make_chol_golden.py -- pins the Cholesky factor of the default update path (FP64 DMMA, one GPU) bit for
bit: for every input of oracle.chol_ref.BITS_CASES, the sha256 of the lower triangle of the factor and the launch count
of one factorisation, written to tests/golden/chol_factor_bits.json.  tests/test_gpu_cholesky_edges.py checks against
it, so a change that alters the rounding of the default path has to say so by regenerating this file.
Run on a GPU:  python tests/golden/make_chol_golden.py [OUT.json]
"""
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import conflux_b200 as cb  # noqa: E402
from conflux_b200 import _lib  # noqa: E402
from oracle import chol_ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "chol_factor_bits.json")


def factor_bits(kind, N, v):
    A = chol_ref.bits_case_input(kind, N)
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    if A is not None:
        ch.data[...] = A
    cnt = ctypes.c_int64()
    _lib.lib().cflx_chol_launch_count(ch._h, ctypes.byref(cnt), 1)
    ch.parallelCholesky()
    _lib.lib().cflx_chol_launch_count(ch._h, ctypes.byref(cnt), 1)
    digest = chol_ref.factor_digest(ch.local_factor())
    ch.finalize()
    comm.close()
    return dict(sha256=digest, launches=cnt.value)


if __name__ == "__main__":
    out = {f"{k}_{N}_{v}": factor_bits(k, N, v) for k, N, v in chol_ref.BITS_CASES}
    with open(sys.argv[1] if len(sys.argv) > 1 else OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
