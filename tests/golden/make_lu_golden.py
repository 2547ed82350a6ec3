"""tests/golden/make_lu_golden.py -- pins the LU factor of the default path (FP64 DMMA update, one GPU) bit for bit: for
every case of CASES, the sha256 of the layer-0 share of L\\U, of the permutation, and the launch count of one
factorisation, written to tests/golden/lu_factor_bits.json.  tests/test_gpu_lu_edges.py checks against it, so a change
that alters the rounding of the default path has to say so by regenerating this file.
Run on a GPU:  python tests/golden/make_lu_golden.py [OUT.json]
"""
import ctypes
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import conflux_b200 as cb  # noqa: E402
from conflux_b200 import _lib  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lu_factor_bits.json")

# the library's generator at the single-GPU shapes of tests/test_gpu_lu_edges.py, and integer matrices with a dominant
# diagonal (the input is the same bits on every machine)
CASES = [("gen", 240, 12), ("gen", 960, 48), ("gen", 1000, 80), ("gen", 1536, 96), ("gen", 1536, 384), ("gen", 2048, 512),
         ("gen", 2048, 256), ("int", 960, 48), ("int", 1536, 128), ("int", 2048, 256)]


def case_input(kind, M):
    """None = the library's generator; else the M x M integer matrix of the case (float64, exact)"""
    if kind == "gen":
        return None
    A = np.random.default_rng(M).integers(-8, 9, (M, M)).astype(np.float64)
    return A + np.diag(np.full(M, 16.0 * M))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def factor(N, v, A=None):
    """one factorisation on one GPU: (L\\U share, perm, launch count, uses the int8 update)"""
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    if A is not None:
        gv.data[...] = A
    cnt = ctypes.c_int64()
    _lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(cnt), 1)
    C = np.zeros((gv.Ml, gv.Nl))
    perm = np.zeros(gv.M, dtype=np.int32)
    cb.LU_rep(gv, C, perm)
    _lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(cnt), 1)
    oz = _lib.lib().cflx_lu_uses_ozaki(gv._h)
    gv.free_comms()
    comm.close()
    return C, perm, cnt.value, oz


def factor_bits(kind, N, v):
    M = cb.lu_dims(N, N, v, 1, 1, 1)["M"]
    C, perm, launches, _ = factor(N, v, case_input(kind, M))
    return dict(factor=digest(C), perm=digest(perm), launches=launches)


if __name__ == "__main__":
    out = {f"{k}_{N}_{v}": factor_bits(k, N, v) for k, N, v in CASES}
    with open(sys.argv[1] if len(sys.argv) > 1 else OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
