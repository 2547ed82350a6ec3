"""GPU: the 192x128 tile of the trailing-update GEMM (gemm_tn_wide_kernel: a producer warpgroup that hands registers to
8 consumer warps of 96x32, C staged below and inside the drained operand ring) against the 64x128 tile, bit for bit.
CFLX_GEMM_TILE is read once per process, so each tile runs in a child interpreter.

The windows are those of test_gpu_gemm_stage (every M % 16, N below one tile, K below, at and past one trip around
the ring, beta = 0 with NaN in C, in place and out of place, the C2 update shapes at steps 32 and 60), those of the
factorisation (test_gpu_lu_edges), and windows around the 192-row block: M on both sides of 192 and 384, and K whose
last k-tile falls in each of the 4 ring stages, so the C slabs wait for every drain order.  Under the 192 tile every
small window is also checked on its own: NaN canaries, nothing written outside the window, the error bound or the
exact product."""
import json
import os
import subprocess
import sys

import pytest

import conflux_b200 as cb  # noqa: F401
from tests import test_gpu_gemm_stage as stage
from tests import test_gpu_lu_edges as edges

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = (8, 28, 40, 64, 84, 116, 132)                     # k-tiles 1, 2, 3, 4, 6, 8, 9: the last one in every ring stage


def _wide_cases():
    cases = []
    for i, K in enumerate(KS):
        for j, (alpha, beta) in enumerate(stage.AB):
            r = (5 * i + j) % 16                        # M % 16 == 0 included: whole slabs up to the tile edge
            M = (176, 192, 368, 384)[(i + j) % 4] + r   # one or two 192-row blocks, the second partly in M
            N = stage.NS[(2 * i + j) % len(stage.NS)]
            cases.append((f"K{K}_M{M}_N{N}_a{alpha}_b{beta}",
                          dict(M=M, N=N, K=K, ldat=edges._rup2(M) + 4, at_rows=K + 1, at_off=(1, 0), ldb=N + 2,
                               b_rows=K + 3, b_off=(2, 2), c_rows=M + 2, ldc=N + 4, c_off=(1, 2), alpha=alpha,
                               beta=beta, in_place=(i + j) % 2 == 1)))
    return cases


def _runs():
    return ([(n, c, "graded") for n, c in _wide_cases()] + stage._small_runs()
            + [(n, c, k) for n, c in edges._window_cases() for k in ("int", "graded")])


def _big_runs():
    return [(n, c, "graded") for n, c in stage._c2_cases()]


def digests(check):
    """sha256 of the whole D buffer of every run; check: each small window is also checked on its own"""
    out = {}
    for small, runs in ((True, _runs()), (False, _big_runs())):
        for name, c, kind in runs:
            seed = edges._seed(name, kind)
            if check and small:
                edges._check_window(name, c, kind, seed)
            AT, B, C, *_ = edges._window_buffers(c, kind, seed)
            out[f"{name}_{kind}"] = edges._digest(edges._run_window(c, AT, B, C)[0])
    return out


def _child(tile, check, tmp_path):
    out = os.path.join(str(tmp_path), f"digests_{tile}.json")
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); import json; from tests import test_gpu_gemm_wide as t; "
            f"json.dump(t.digests({check!r}), open({out!r}, 'w'))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=dict(os.environ, CFLX_GEMM_TILE=tile), cwd=ROOT,
                       timeout=900, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    with open(out) as f:
        return json.load(f)


def test_gemm_tile_192_windows_and_bits(tmp_path):
    got = _child("192", True, tmp_path)
    want = _child("64", False, tmp_path)
    assert sorted(got) == sorted(want)
    diff = [k for k in want if got[k] != want[k]]
    assert not diff, diff


def test_gemm_tile_128_is_bit_identical_to_192(tmp_path):
    """the two tiles the launcher chooses between: the choice never changes a bit"""
    assert _child("128", False, tmp_path) == _child("192", False, tmp_path)
