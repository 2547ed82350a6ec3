"""CPU: bench.py's host-side contract pieces -- the workloads are BASELINE.json's configurations, the reference arm runs
the STATED configuration (never a smaller N under the big config's name; the 8-GPU one is labelled as extrapolated), both
arms describe the workload with the same `config` keys, golden pivot sequences exist for C2 and C3."""
import importlib.util
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bench)


def test_workloads_are_the_baseline_configs():
    cfg = json.load(open(os.path.join(ROOT, "BASELINE.json")))["configs"]
    assert bench.WORKLOADS[1] == (16384, 256, (1, 1, 1)) and "N=16384, b=256" in cfg[1]
    assert bench.WORKLOADS[4] == (32768, 512, (2, 2, 1)) and "N=32768, b=512" in cfg[2]
    assert bench.WORKLOADS[8] == (65536, 512, (2, 2, 2)) and "N=65536, b=512" in cfg[3]
    assert bench.CHOL_WORKLOAD == (32768, 512) and "--dim=32768 --tile=512" in cfg[4]


def test_reference_arm_runs_the_stated_configuration():
    for gpus in (1, 2, 4):
        N, v, grid, note = bench.reference_plan(gpus)
        assert (N, v) == bench.WORKLOADS[gpus][:2]                      # never a smaller N under the config's name
        assert grid in (bench.WORKLOADS[gpus][2], (1, 1, 1))             # the rank-thread grid, or 1x1x1 if memory forbids
    N, v, grid, note = bench.reference_plan(8)
    assert N == 32768 and v == 512 and "rate measured at N=32768" in note   # C4 is labelled, not silently substituted


def test_both_arms_use_the_same_config_description():
    N, v, grid = bench.WORKLOADS[4]
    ours = {"workload": bench.workload_string(N, v, grid), "generator": bench.GENERATOR, "l2": bench.l2_string(N, v, grid)}
    assert ours["workload"] == "LU N=32768 v=512 grid 2x2x1" and "2.0 GiB" in ours["l2"]


def test_bench_golden_pivots_present():
    for (N, v, grid) in [(16384, 256, (1, 1, 1)), (32768, 512, (2, 2, 1))]:
        g = bench.load_golden_perm(N, v, grid)
        assert g is not None and sorted(np.asarray(g).tolist()) == list(range(N))
    assert bench.load_golden_perm(65536, 512, (2, 2, 2)) is None


def test_reference_arm_prints_the_contract_line_on_a_small_override():
    """`bench.py --impl reference` end to end (size override, a few seconds): one JSON line with impl/metric/config/
    cpu_baseline/e2e, timed inside ONE child process; also guards the threading set-up of that child (OMP_PROC_BIND made
    OpenBLAS' threads inherit a one-CPU mask: 40x slower)."""
    import subprocess
    import sys
    import time
    import pytest
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    t0 = time.time()
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "1",
                          "--warmup", "0", "--N", "1024", "--v", "128"], capture_output=True, text=True, timeout=300,
                         env=dict(os.environ, CFLX_REF_BUDGET_S="5"))
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and "unavailable" not in line, line
    assert line["metric"].startswith("LU GFLOP/s") and line["unit"] == "GFLOP/s" and line["higher_is_better"] is True
    assert line["cpu_baseline"]["kind"] == "reference" and line["cpu_baseline"]["value"] == line["value"]
    assert line["e2e"] == {"value": line["value"], "unit": "GFLOP/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "size override" in line["config"]["workload"] and line["steps_done"] == 1
    assert time.time() - t0 < 120


def test_dump_outputs_is_seeded_float64_and_within_budget(tmp_path):
    loc = np.arange(3000 * 3000, dtype=np.float64).reshape(3000, 3000)
    perm = np.arange(3000, dtype=np.int32)[::-1].copy()
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), 0, 1, loc, perm)
    files = sorted(os.listdir(tmp_path / "a"))
    assert files == ["factor_sample.npy", "factor_sample_index.npy", "permutation.npy"]
    assert sum(os.path.getsize(tmp_path / "a" / f) for f in files) <= 64 * 10 ** 6
    for f in files:
        a, b = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert a.dtype == np.float64 and np.array_equal(a, b)
    idx = np.load(tmp_path / "a" / "factor_sample_index.npy").astype(np.int64)
    assert np.array_equal(np.load(tmp_path / "a" / "factor_sample.npy"), loc.reshape(-1)[idx])
