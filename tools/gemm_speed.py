"""tools/gemm_speed.py -- anatomy of the trailing-update GEMM (gemm_tn_kernel) at the shapes the C2 benchmark runs
(N = 16384, v = 256, grid 1x1x1), timed through the factorisation's in-place launch (cb.dbg.gemm_tn_window, CUDA events
over `reps` launches, mean ms of one launch):
  * 16128 x 16128 x 256 (the whole update of step 0), with K = 16 as well: K = 256 minus K = 16 is the main loop, the
    rest is the per-tile fixed cost (operand fill, epilogue);
  * part 0 (n_act x 256, the look-ahead columns) and part 1 (n_act x (n_act - 256)) of steps k = 0, 16, 32, 48, 60,
    n_act = 16384 - 256 (k + 1), and the local pivot search (cb.dbg.panel) on the n_act x 256 panel of the same step;
  * the GEMMs of the U solve at the same steps (M = 128, K = 128, the TRSM sweep with nb = 128): the look-ahead
    columns (N = 256) and the rest (N = n_act - 256), beta = 0 the diagonal block, beta = 1 the update below it.
Every GEMM shape runs with beta = 1 and beta = 0; beta = 0 reads no C, so the difference is what the C read costs.
C has the factorisation's leading dimension (Nl = 16384).  Prints one JSON line with the card's name, power limit and
SM clock, and the tile CFLX_GEMM_TILE fixes (empty: chosen per launch).
    python tools/gemm_speed.py [--root TREE] [--out FILE]
--root imports conflux_b200 from another checkout (to compare two builds in one process each)."""
import argparse
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--out", default="")
ap.add_argument("--reps", type=int, default=20)
a = ap.parse_args()
sys.path.insert(0, os.path.abspath(a.root))
import numpy as np  # noqa: E402
import conflux_b200 as cb  # noqa: E402

N, V, NL = 16384, 256, 16384
STEPS = (0, 16, 32, 48, 60)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    name, plim, sm, smax = [x.strip() for x in r.stdout.strip().split(",")[:4]]
    return {"gpu": name, "power_limit_w": plim, "sm_mhz": sm, "sm_max_mhz": smax}


rng = np.random.default_rng(2024)
Cbig = rng.uniform(-1, 1, (N - V, NL))            # rows of the largest trailing matrix, factorisation leading dim.
AT = rng.uniform(-1, 1, (V, N))
B = rng.uniform(-1, 1, (V, NL))


def gemm(M, Ncols, K, beta, col_off):
    C = Cbig[:M]                                   # contiguous row block: no copy
    _, _, ms = cb.dbg.gemm_tn_window(AT, B, C, M, Ncols, K, -1.0, beta, at_off=(0, 0), b_off=(0, col_off),
                                     c_off=(0, col_off), in_place=True, reps=a.reps)
    return {"M": M, "N": Ncols, "K": K, "beta": beta, "ms": round(ms, 4),
            "tflops": round(2.0 * M * Ncols * K / (ms * 1e-3) / 1e12, 2)}


rec = {"tool": "gemm_speed", "root": os.path.abspath(a.root), "tile": os.environ.get("CFLX_GEMM_TILE", ""),
       "card": card(), "shapes": [], "panel": []}
M0 = N - V
for K in (256, 16):
    for beta in (1.0, 0.0):
        rec["shapes"].append(dict(gemm(M0, M0, K, beta, 0), name=f"full_K{K}"))
for k in STEPS:
    n_act = N - V * (k + 1)
    for part, (cols, off) in enumerate(((V, 0), (n_act - V, V))):
        for beta in (1.0, 0.0):
            rec["shapes"].append(dict(gemm(n_act, cols, V, beta, off), name=f"step{k}_part{part}"))
    for cols in (V, n_act - V):
        for beta in (1.0, 0.0):
            rec["shapes"].append(dict(gemm(128, cols, 128, beta, 0), name=f"step{k}_usolve_N{cols}"))
    _, _, _, pms = cb.dbg.panel(np.ascontiguousarray(Cbig[:n_act, :V]), reps=5)
    rec["panel"].append({"step": k, "n_act": n_act, "ms": round(pms, 4)})
rec["card_after"] = card()
line = json.dumps(rec)
print(line)
if a.out:
    with open(a.out, "w") as f:
        f.write(line + "\n")
