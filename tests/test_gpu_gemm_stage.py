"""GPU: the 128x128 tile of gemm_tn_kernel, whose epilogue reads C from the drained operand ring, against the 64x128
tile, whose epilogue reads C straight from HBM: bit for bit (both accumulate every element over k in the same m16n8k8
order and finish it with one fma(alpha, acc, beta * c)).  CFLX_GEMM_TILE is read once per process, so the 64 tile runs
in a child interpreter.

The windows cover the C2 benchmark's update shapes at steps 32 and 60, every row count modulo 16 (slabs of 16 rows
partly or not at all inside M), N below one tile and not a multiple of 32, K below one trip around the 4-stage ring
(stages the main loop never used), at one trip and past it with a tail, beta = 0 with NaN in C, general alpha and beta,
in place and out of place.  The smaller windows are also checked on their own: NaN canaries around every operand
block, nothing written outside the window, the hp_ref error bound (graded inputs) or the exact product (integers)."""
import json
import os
import subprocess
import sys

import pytest

import conflux_b200 as cb  # noqa: F401
from tests import test_gpu_lu_edges as edges

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = (4, 12, 16, 60, 64, 68, 256)
NS = (2, 34, 98, 126, 130, 222, 382)
AB = ((-1.0, 1.0), (0.7, -0.3), (-1.0, 0.0))           # (alpha, beta); beta = 0 puts NaN in C


def _small_cases():
    cases = []
    for i, K in enumerate(KS):
        for j, (alpha, beta) in enumerate(AB):
            r = (3 * i + j) % 15 + 1                    # M % 16 takes every value 1..15
            M = 128 * (1 + j % 2) + 64 * (i % 2) + r    # the partial slabs fall in either warp row
            N = NS[(i + 2 * j) % len(NS)]
            cases.append((f"K{K}_M{M}_N{N}_a{alpha}_b{beta}",
                          dict(M=M, N=N, K=K, ldat=edges._rup2(M) + 2, at_rows=K + 2, at_off=(1, 2), ldb=N + 4,
                               b_rows=K + 2, b_off=(1, 2), c_rows=M + 3, ldc=N + 6, c_off=(2, 4), alpha=alpha,
                               beta=beta, in_place=(i + j) % 2 == 0)))
    return cases


def _c2_cases():
    """parts 0 (the look-ahead columns) and 1 of the trailing update at steps 32 and 60 of N = 16384, v = 256"""
    cases = []
    for k in (32, 60):
        n_act = 16384 - 256 * (k + 1)
        for part, (N, col) in enumerate(((256, 256), (n_act - 256, 512))):
            cases.append((f"c2_step{k}_part{part}",
                          dict(M=n_act, N=N, K=256, ldat=n_act, at_rows=258, at_off=(1, 0), ldb=n_act + 2, b_rows=258,
                               b_off=(1, col - 256), c_rows=n_act + 1, ldc=n_act + 258, c_off=(1, col), alpha=-1.0,
                               beta=1.0, in_place=True)))
    return cases


def _small_runs():
    """integer inputs where alpha = -1 (the product and the update are exact), graded inputs everywhere"""
    return [(n, c, kind) for n, c in _small_cases() for kind in ("int", "graded") if kind == "graded" or c["alpha"] == -1]


def _runs():
    return _small_runs() + [(n, c, "graded") for n, c in _c2_cases()]


def stage_digests(_):
    """sha256 of the whole D buffer of every run (also called in a child under CFLX_GEMM_TILE=64)"""
    out = {}
    for name, c, kind in _runs():
        AT, B, C, *_ = edges._window_buffers(c, kind, edges._seed(name, kind))
        out[f"{name}_{kind}"] = edges._digest(edges._run_window(c, AT, B, C)[0])
    return out


def _child_64(tmp_path):
    out = os.path.join(str(tmp_path), "stage_digests.json")
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); import json; from tests import test_gpu_gemm_stage as t; "
            f"json.dump(t.stage_digests(None), open({out!r}, 'w'))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=dict(os.environ, CFLX_GEMM_TILE="64"), cwd=ROOT,
                       timeout=900, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    with open(out) as f:
        return json.load(f)


@pytest.mark.parametrize("name,c,kind", _small_runs(), ids=[f"{n}_{k}" for n, _, k in _small_runs()])
def test_gemm_stage_window(name, c, kind):
    edges._check_window(name, c, kind, edges._seed(name, kind))


def test_gemm_stage_is_bit_identical_to_the_64_tile(tmp_path):
    want = stage_digests(None)
    got = _child_64(tmp_path)
    assert sorted(got) == sorted(want)
    diff = [k for k in want if got[k] != want[k]]
    assert not diff, diff
