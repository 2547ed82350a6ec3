"""tests/golden/make_solve_golden.py -- pins the solves (cflx_lu_solve, cflx_chol_solve) on one GPU bit for bit: for each
case, the sha256 of X for integer right-hand sides of 1, 3, 64 and 130 columns, written to tests/golden/solve_bits.json.
The LU cases factor the library's generated matrix at (N, v) = (1024, 128) and (100, 16); the Cholesky cases are the
inputs of oracle.chol_ref.BITS_CASES at v = 128 and 512.  The right-hand sides have integer entries, so every input has
the same bits on every machine.  tests/test_gpu_solve.py and tests/test_gpu_chol_solve.py check against it, so a change
that alters the rounding of a solve has to say so by regenerating this file.
Run on a GPU:  python tests/golden/make_solve_golden.py [OUT.json]
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import conflux_b200 as cb  # noqa: E402
from oracle import chol_ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "solve_bits.json")
NRHS = (1, 3, 64, 130)
LU_CASES = [(1024, 128), (100, 16)]
CHOL_CASES = [(k, N, v) for k, N, v in chol_ref.BITS_CASES if v in (128, 512)]


def rhs(M, nrhs):
    """integer right-hand sides, exact in float64"""
    return np.random.default_rng(M + nrhs).integers(-8, 9, (M, nrhs)).astype(np.float64)


def digest(X):
    return hashlib.sha256(np.ascontiguousarray(X, dtype=np.float64).tobytes()).hexdigest()


def lu_solve_bits(N, v):
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    cb.LU_rep(gv)
    out = {str(n): digest(cb.lu_solve(gv, rhs(gv.M, n))) for n in NRHS}
    gv.free_comms()
    comm.close()
    return out


def chol_solve_bits(kind, N, v):
    A = chol_ref.bits_case_input(kind, N)
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    if A is not None:
        ch.data[...] = A
    ch.parallelCholesky()
    out = {str(n): digest(ch.solve(rhs(ch.N, n))) for n in NRHS}
    ch.finalize()
    comm.close()
    return out


if __name__ == "__main__":
    out = {f"lu_{N}_{v}": lu_solve_bits(N, v) for N, v in LU_CASES}
    out.update({f"chol_{k}_{N}_{v}": chol_solve_bits(k, N, v) for k, N, v in CHOL_CASES})
    with open(sys.argv[1] if len(sys.argv) > 1 else OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
