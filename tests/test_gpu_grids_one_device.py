"""GPU: every multi-rank test of the suite, on one device.  Each module's grid tests run in a child pytest under the NCCL
loopback (tests/loopback/nccl_loopback.cpp, LD_PRELOAD) with the tests._loopback plugin, so the P ranks of a grid are
P threads on device 0 and every collective, split and tournament message is staged and schedule-checked.  The
child's tests check their results against their own oracles; this test asserts that all of them ran and passed, and
that the collectives really went through the loopback.

Not run here: the bench-size C3 pivots (N = 32768 on 2 x 2 x 1, minutes of staged panels), the 4-GPU miniapp (a
separate program that needs four devices), the `cuda:1` pointer check of test_gpu_solve_local (a second physical
device), and CFLX_GEMM=ozaki on grids (its persistent update sizes itself to the whole device)."""
import json
import os
import subprocess
import sys
import time
import xml.etree.ElementTree as ET

import pytest

from tests import _loopback

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# module -> node selectors (a test name stands for all its parameters; "-k" narrows the module's selection)
MODULES = {
    "solve": ["test_multi_gpu_solve"],
    "solve_trans": ["test_multi_gpu_transposed_solve"],
    "rcond": ["test_multi_gpu_lu_rcond", "test_multi_gpu_chol_rcond"],
    "refine": ["test_multi_gpu_lu_refine", "test_multi_gpu_chol_refine"],
    "refinex": ["test_multi_gpu_lu_refine_x"],
    "svx": ["test_multi_gpu_lu_svx", "test_multi_gpu_chol_svx"],
    "svxx": ["test_multi_gpu_lu_svxx", "test_multi_gpu_chol_svxx"],
    "inverse": ["test_multi_gpu_lu_inverse", "test_multi_gpu_chol_inverse"],
    "det": ["test_multi_gpu_lu_det", "test_multi_gpu_chol_det"],
    "lu_fixed": ["test_multi_gpu_same_input_refactor", "test_multi_gpu_zero_and_tiny_pivots_on_every_rank"],
    "rbt": ["test_multi_gpu_matches_one_gpu"],
    "chol_solve": ["test_multi_gpu_solve"],
    "solve_local": ["test_multi_gpu_lu_solve_local", "test_multi_gpu_chol_solve_local"],
    "cholesky": ["test_cholesky_multi_gpu_matches_lapack"],
    "cholesky_edges": ["test_not_positive_definite_same_error_on_every_rank"],
    "grid_shares": ["test_multi_gpu_chol_padded_grid"],
    "lu": ["test_multi_gpu_matches_oracle", "test_multi_gpu_golden_fixtures"],
    # the grid cases of the switch tests; the digest tests run (1,1,1) and both grids, partly in children of their own
    "lu_edges": ["test_switch_is_bit_identical", "test_gemm_tile_64_is_bit_identical", "test_trsm_block_size_switch",
                 "-k", "not test_switch_is_bit_identical or grid1 or grid2"],
}
RUNS = [(m, {}) for m in MODULES] + [(m, {"CFLX_LOOKAHEAD": "0"}) for m in ("lu", "lu_edges", "lu_fixed")]
COLLECTIVES = ("ncclAllReduce", "ncclReduce", "ncclBroadcast", "ncclAllGather", "ncclSend")


def _selectors(module):
    f = f"tests/test_gpu_{module}.py"
    out, it = [], iter(MODULES[module])
    for s in it:
        out += [s, next(it)] if s == "-k" else [f"{f}::{s}"]
    return out


@pytest.fixture(scope="module")
def loopback():
    return _loopback.build()


@pytest.mark.parametrize("module,env", RUNS, ids=lambda x: x if isinstance(x, str) else
                         ("-".join(f"{k}={v}" for k, v in x.items()) or "default"))
def test_multi_rank_tests_pass_on_one_device(module, env, loopback, tmp_path):
    xml, stats_out = tmp_path / "junit.xml", tmp_path / "stats.json"
    preload = " ".join(p for p in (loopback, os.environ.get("LD_PRELOAD")) if p)
    cenv = dict(os.environ, LD_PRELOAD=preload, **{_loopback.STATS_ENV: str(stats_out)}, **env)
    flags = ["-s"] if sys.flags.no_user_site else []
    cmd = [sys.executable] + flags + ["-m", "pytest", "-p", "tests._loopback", "-p", "no:cacheprovider", "-q", "-rA",
                                      f"--junitxml={xml}"] + _selectors(module)
    t0 = time.perf_counter()
    r = subprocess.run(cmd, cwd=ROOT, env=cenv, capture_output=True, text=True, timeout=1800)
    dt = time.perf_counter() - t0
    tail = (r.stdout[-6000:] + "\n--- stderr ---\n" + r.stderr[-6000:])
    assert r.returncode == 0, tail
    cases = [(c.get("classname", "") + "::" + c.get("name", ""), [e.tag for e in c]) for c in ET.parse(xml).iter("testcase")]
    skipped = [n for n, tags in cases if "skipped" in tags]
    failed = [n for n, tags in cases if "failure" in tags or "error" in tags]
    assert cases and not skipped and not failed, (skipped, failed, tail)
    with open(stats_out) as f:
        calls = json.load(f)
    assert calls["ncclCommInitRank"] > 0 and calls["ncclCommSplit"] > 0, calls
    assert sum(calls[k] for k in COLLECTIVES) > 0, calls
    print(f"\n[{module} {env or ''}] {len(cases)} passed in {dt:.1f} s; loopback calls "
          + ", ".join(f"{k}={v}" for k, v in calls.items() if v))
    for n, _ in cases:
        print(f"    PASSED {n}")
