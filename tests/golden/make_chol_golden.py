"""tests/golden/make_chol_golden.py -- pins the Cholesky factor of every trailing-update kind (one GPU) bit for bit: for
every input of update_cases(update), the sha256 of the lower triangle of the factor and the launch count of one
factorisation.  The default FP64 DMMA update is written to tests/golden/chol_factor_bits.json, the int8
(CFLX_GEMM=ozaki) and TF32 / TF32x3 (cflx_chol_sv_mixed) updates to the "chol" section of
tests/golden/update_factor_bits.json.  tests/test_gpu_cholesky_edges.py checks against them, so a change that alters the
rounding of an update has to say so by regenerating these files.
Run on a GPU:  python tests/golden/make_chol_golden.py [OUT_DIR]
"""
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import conflux_b200 as cb  # noqa: E402
from conflux_b200 import _lib  # noqa: E402
from oracle import chol_ref  # noqa: E402
from tests.golden.make_lu_golden import GOLDEN, UPDATES, update_env, write_section  # noqa: E402

FP64_FILE, UPDATE_FILE = "chol_factor_bits.json", "update_factor_bits.json"
# inputs whose TF32 factor leaves the mixed driver's refinement unconverged (it falls back to FP64): not pinned
MIXED_FALLBACK = {"tf32": [], "tf32x3": []}


def update_cases(update):
    """the inputs of chol_ref.BITS_CASES an update kind is pinned on: int8 where its kernel runs (v a multiple of 128, at
    most 512), TF32 where the mixed driver converges"""
    if update == "int8":
        return [c for c in chol_ref.BITS_CASES if c[2] % 128 == 0 and c[2] <= 512]
    if update in MIXED_FALLBACK:
        return [c for c in chol_ref.BITS_CASES if c not in MIXED_FALLBACK[update]]
    return list(chol_ref.BITS_CASES)


def factor_bits(kind, N, v, update="fp64"):
    """fp64 / int8: cflx_chol_factor; tf32 / tf32x3: cflx_chol_sv_mixed with one right-hand side, its launches
    included, asserted to have converged (the factor is the TF32 one, not that of the FP64 fallback)"""
    A = chol_ref.bits_case_input(kind, N)
    comm = cb.Comm(1, 0, None, 0)
    with update_env(update):
        ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    if A is not None:
        ch.data[...] = A
    cnt = ctypes.c_int64()
    _lib.lib().cflx_chol_launch_count(ch._h, ctypes.byref(cnt), 1)
    if update in ("tf32", "tf32x3"):
        _, it, _ = ch.sv_mixed(np.random.default_rng(ch.N).standard_normal(ch.N), prec=update)
        assert it >= 0, f"{update} N={N} v={v}: the mixed driver fell back to FP64 (iter {it})"
    else:
        ch.parallelCholesky()
    _lib.lib().cflx_chol_launch_count(ch._h, ctypes.byref(cnt), 1)
    digest = chol_ref.factor_digest(ch.local_factor())
    ch.finalize()
    comm.close()
    return dict(sha256=digest, launches=cnt.value)


def golden(update, golden_dir=GOLDEN):
    """the recorded bits of one update kind, by case key"""
    if update == "fp64":
        with open(os.path.join(golden_dir, FP64_FILE)) as f:
            return json.load(f)
    with open(os.path.join(golden_dir, UPDATE_FILE)) as f:
        return json.load(f)["chol"][update]


if __name__ == "__main__":
    out_dir = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
    bits = {u: {f"{k}_{N}_{v}": factor_bits(k, N, v, u) for k, N, v in update_cases(u)} for u in UPDATES}
    with open(os.path.join(out_dir, FP64_FILE), "w") as f:
        json.dump(bits.pop("fp64"), f, indent=1, sort_keys=True)
    write_section(os.path.join(out_dir, UPDATE_FILE), "chol", bits)
