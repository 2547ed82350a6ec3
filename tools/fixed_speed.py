"""tools/fixed_speed.py -- the LU in a prescribed row order (LU_rep_fixed) against the pivoted LU (LU_rep) on one GPU, at
N = 16384 with v = 256 (C2) and v = 512.

Prints the card, its power limit and SM clocks; per tile size the device time of the main loop of LU_rep and of
LU_rep_fixed with the last permutation on the same input, alternating, `--reps` each, medians; one non-serialising
timeline of each (profiling mode 2: per-region totals by stream, the side stream's step1_* and the main stream's
step6_dgemm); and the tile LU alone through its test hook (cflx_dbg_getrf_nopiv_tile), timed from the kernels
torch.profiler records: per call the span from the first kernel's start to the last kernel's end (host copies
excluded), with the one-CTA kernel's share of it.  --json PATH also writes everything as JSON."""
import argparse
import json
import os
import statistics
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import conflux_b200 as cb
from conflux_b200._lib import lib
from tools.cond_speed import card


def summary(tl):
    keep = {}
    for side in ("main", "side"):
        for name, (ms, cnt) in tl[side].items():
            if name.startswith("step1_") or name == "step6_dgemm":
                keep[f"{side}:{name}"] = [round(ms, 3), cnt]
    return keep


def compare(comm, N, v, reps):
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    cb.LU_rep(gv)
    p0 = np.zeros(gv.M, dtype=np.int32)
    cb.LU_rep_fixed(gv, upload=False, permutation=p0)        # warm-up of both paths
    piv, fix = [], []
    for _ in range(reps):
        piv.append(cb.LU_rep(gv, upload=False))
        fix.append(cb.LU_rep_fixed(gv, upload=False)[0])
    p1 = np.zeros(gv.M, dtype=np.int32)
    cb.LU_rep(gv, upload=False, permutation=p1)
    out = dict(pivoted_ms=piv, fixed_ms=fix, pivoted_median=statistics.median(piv), fixed_median=statistics.median(fix),
               same_permutation=bool(np.array_equal(p0, p1)))
    cb.LU_rep_fixed(gv, upload=False)
    out["resid_fixed"] = cb.validate(gv)[1]
    print(f"N={N} v={v}: LU_rep median {out['pivoted_median']:.2f} ms {['%.2f' % x for x in piv]}")
    print(f"    LU_rep_fixed median {out['fixed_median']:.2f} ms {['%.2f' % x for x in fix]}  "
          f"(same permutation {out['same_permutation']}, residual {out['resid_fixed']:.2e})")
    for name, fn in (("pivoted", lambda: cb.LU_rep(gv, upload=False)),
                     ("fixed", lambda: cb.LU_rep_fixed(gv, upload=False))):
        lib().cflx_lu_set_profiling(gv._h, 2)
        fn()
        tl = cb.timeline(gv)
        lib().cflx_lu_set_profiling(gv._h, 0)
        out[f"timeline_{name}"] = summary(tl)
        lup = sorted(r[3] for r in tl["records"] if r[0] == "step1_lup")
        out[f"step1_lup_median_{name}"] = statistics.median(lup)
        print(f"    timeline {name}:", json.dumps(out[f"timeline_{name}"]),
              f"step1_lup median {out[f'step1_lup_median_{name}']:.3f} ms")
    gv.free_comms()
    return out


def hook_ms(v, variant, reps):
    """(median span, median share of getrf_nopiv_block_kernel) in ms of the tile's kernels per hook call"""
    A = np.random.default_rng(v).standard_normal((v, v)) + 2.0 * v * np.eye(v)
    cb.dbg.getrf_nopiv_tile(A, variant=variant)              # warm-up: module load, shared-memory attribute
    spans, block = [], []
    for _ in range(reps):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            cb.dbg.getrf_nopiv_tile(A, variant=variant)
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
        spans.append((max(e["ts"] + e["dur"] for e in ev) - min(e["ts"] for e in ev)) / 1e3)
        block.append(sum(e["dur"] for e in ev if "getrf_nopiv_block_kernel" in e["name"]) / 1e3)
    return statistics.median(spans), statistics.median(block)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    out = {"card": card(), "N": a.n}
    print("card:", out["card"])
    torch.cuda.init()
    for v, variant in ((256, 0), (256, 1), (512, 0), (512, 1)):
        span, blk = hook_ms(v, variant, a.reps)
        out[f"hook_v{v}_variant{variant}"] = dict(span_ms=span, one_cta_kernel_ms=blk)
        print(f"tile hook v={v} variant {variant} ({'128-block driver' if variant else 'one-CTA kernel'}): "
              f"{span:.3f} ms, of which the one-CTA kernel {blk:.3f} ms")
    comm = cb.Comm(1, 0, None, 0)
    for v in (256, 512):
        out[f"v{v}"] = compare(comm, a.n, v, a.reps)
    comm.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
