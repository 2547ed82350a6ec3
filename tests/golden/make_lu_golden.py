"""tests/golden/make_lu_golden.py -- pins the LU factor of every trailing-update kind (one GPU) bit for bit: for every case
of update_cases(update), the sha256 of the layer-0 share of L\\U, of the permutation, and the launch count of one
factorisation.  The default FP64 DMMA update is written to tests/golden/lu_factor_bits.json, the int8 (CFLX_GEMM=ozaki)
and TF32 / TF32x3 (cflx_lu_sv_mixed) updates to the "lu" section of tests/golden/update_factor_bits.json.
tests/test_gpu_lu_edges.py checks against them, so a change that alters the rounding of an update has to say so by
regenerating these files.
Run on a GPU:  python tests/golden/make_lu_golden.py [OUT_DIR]
"""
import contextlib
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

GOLDEN = os.path.dirname(os.path.abspath(__file__))
FP64_FILE, UPDATE_FILE = "lu_factor_bits.json", "update_factor_bits.json"

# the library's generator at the single-GPU shapes of tests/test_gpu_lu_edges.py, and integer matrices with a dominant
# diagonal (the input is the same bits on every machine)
CASES = [("gen", 240, 12), ("gen", 960, 48), ("gen", 1000, 80), ("gen", 1536, 96), ("gen", 1536, 384), ("gen", 2048, 512),
         ("gen", 2048, 256), ("int", 960, 48), ("int", 1536, 128), ("int", 2048, 256)]
UPDATES = ("fp64", "int8", "tf32", "tf32x3")
# cases whose TF32 factors leave the mixed driver's refinement unconverged (it falls back to FP64): not pinned
MIXED_FALLBACK = {"tf32": [("gen", 2048, 512), ("gen", 2048, 256)], "tf32x3": []}


def update_cases(update):
    """the cases an update kind is pinned on: int8 where its kernel runs (v a multiple of 128, at most 512), TF32 where
    the mixed driver converges"""
    if update == "int8":
        return [c for c in CASES if c[2] % 128 == 0 and c[2] <= 512]
    if update in MIXED_FALLBACK:
        return [c for c in CASES if c not in MIXED_FALLBACK[update]]
    return list(CASES)


@contextlib.contextmanager
def update_env(update):
    """CFLX_GEMM=ozaki while a handle of the int8 kind is created (read at creation)"""
    old = os.environ.get("CFLX_GEMM")
    if update == "int8":
        os.environ["CFLX_GEMM"] = "ozaki"
    try:
        yield
    finally:
        if update == "int8":
            if old is None:
                del os.environ["CFLX_GEMM"]
            else:
                os.environ["CFLX_GEMM"] = old


def case_input(kind, M):
    """None = the library's generator; else the M x M integer matrix of the case (float64, exact)"""
    if kind == "gen":
        return None
    A = np.random.default_rng(M).integers(-8, 9, (M, M)).astype(np.float64)
    return A + np.diag(np.full(M, 16.0 * M))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def factor(N, v, A=None, update="fp64"):
    """one factorisation on one GPU: (L\\U share, perm, launch count, uses the int8 update).  fp64 / int8: cflx_lu_factor;
    tf32 / tf32x3: cflx_lu_sv_mixed with one right-hand side, its launches included, asserted to have converged (the
    factors are the TF32 ones, not those of the FP64 fallback)"""
    comm = cb.Comm(1, 0, None, 0)
    with update_env(update):
        gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    if A is not None:
        gv.data[...] = A
    cnt = ctypes.c_int64()
    _lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(cnt), 1)
    C = np.zeros((gv.Ml, gv.Nl))
    perm = np.zeros(gv.M, dtype=np.int32)
    if update in ("tf32", "tf32x3"):
        _, it, _ = cb.lu_sv_mixed(gv, np.random.default_rng(gv.M).standard_normal(gv.M), prec=update)
        assert it >= 0, f"{update} N={N} v={v}: the mixed driver fell back to FP64 (iter {it})"
        cb.check(_lib.lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "lu_get_factors")
    else:
        cb.LU_rep(gv, C, perm)
    _lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(cnt), 1)
    oz = _lib.lib().cflx_lu_uses_ozaki(gv._h)
    gv.free_comms()
    comm.close()
    assert oz == (update == "int8"), f"{update} N={N} v={v}: cflx_lu_uses_ozaki = {oz}"
    return C, perm, cnt.value, oz


def factor_bits(kind, N, v, update="fp64"):
    M = cb.lu_dims(N, N, v, 1, 1, 1)["M"]
    C, perm, launches, _ = factor(N, v, case_input(kind, M), update)
    return dict(factor=digest(C), perm=digest(perm), launches=launches)


def golden(update, golden_dir=GOLDEN):
    """the recorded bits of one update kind, by case key"""
    if update == "fp64":
        with open(os.path.join(golden_dir, FP64_FILE)) as f:
            return json.load(f)
    with open(os.path.join(golden_dir, UPDATE_FILE)) as f:
        return json.load(f)["lu"][update]


def write_section(path, section, data):
    """data into section `section` of the JSON file at path, the other sections kept"""
    out = {}
    if os.path.exists(path):
        with open(path) as f:
            out = json.load(f)
    out[section] = data
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    out_dir = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
    bits = {u: {f"{k}_{N}_{v}": factor_bits(k, N, v, u) for k, N, v in update_cases(u)} for u in UPDATES}
    with open(os.path.join(out_dir, FP64_FILE), "w") as f:
        json.dump(bits.pop("fp64"), f, indent=1, sort_keys=True)
    write_section(os.path.join(out_dir, UPDATE_FILE), "lu", bits)
