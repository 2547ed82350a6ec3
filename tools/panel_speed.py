"""tools/panel_speed.py -- the row-owner pivot search (panel_getrf_kernel) timed as the factorisation launches it: the
n_act x 256 panels of the C2 benchmark (N = 16384, v = 256, grid 1x1x1; n_act = N - v (k + 1)) under the look-ahead's
SM budget.  cb.dbg.panel honours CFLX_PANEL_CTAS, so every cap is one call; CUDA events around each of `reps` launches
after one warm-up launch, mean ms of one launch.
  * steps 0, 8, ..., 56 x caps 8, 16, 32, 64, 132: ms per launch, us per column, and the launch geometry (G CTAs x R rows,
    inner block NB), computed here with the launcher's arithmetic;
  * v = 512 at n = 16384 - 512 (k + 1), k = 0 and 16 (the shape of the 2- and 4-GPU panels), caps 32 and 48;
  * a phase split by differences: v = 256 against v = 32 at equal n (no trailing columns at v = NB: what is left is the
    per-column exchange and elimination), and one CTA on a 2048-row panel (no foreign CTA to wait for: the protocol's own
    store -> load latency plus the work inside the CTA).
Prints one JSON line with the card's name, power limit and SM clock.  Needs a GPU.
    python tools/panel_speed.py [--root TREE] [--out FILE] [--reps 20]
--root imports conflux_b200 from another checkout (to compare two builds, one process each)."""
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

N, V = 16384, 256
STEPS = (0, 8, 16, 24, 32, 40, 48, 56)
CAPS = (8, 16, 32, 64, 132)
SMS, ROW_THREADS, RPT_LIMIT = 132, 256, 8


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    name, plim, sm, smax = [x.strip() for x in r.stdout.strip().split(",")[:4]]
    return {"gpu": name, "power_limit_w": plim, "sm_mhz": sm, "sm_max_mhz": smax}


def geometry(n, v, cap):
    """(G, R, NB) of launch_panel_getrf_a00 for an n x v panel under CFLX_PANEL_CTAS = cap (panel.cu)."""
    G = min(max((n + 31) // 32, 1), SMS)
    if 0 < cap < G:
        need = -(-n // (RPT_LIMIT * ROW_THREADS))
        G = max(cap, min(need, SMS))
    R = -(-max(-(-n // G), 1) // 32) * 32
    G = -(-n // R) if n > 0 else 1
    for nb in (32, 16, 8, 4):
        if (nb <= v or nb == 4) and (8 * nb + 1) * R + 8 * nb * v <= 222 * 1024 - (8 * nb * nb + 796 * nb + 848):
            return G, R, nb
    return G, R, 0


rng = np.random.default_rng(2024)
Cbig = rng.uniform(-1, 1, (N - V, 512))


def run(n, v, cap, name):
    os.environ["CFLX_PANEL_CTAS"] = str(cap)
    _, _, _, ms = cb.dbg.panel(np.ascontiguousarray(Cbig[:n, :v]), reps=a.reps)
    G, R, nb = geometry(n, v, cap)
    return {"name": name, "n": n, "v": v, "cap": cap, "G": G, "R": R, "NB": nb, "ms": round(ms, 4),
            "us_per_col": round(ms * 1e3 / min(n, v), 3)}


rec = {"tool": "panel_speed", "root": os.path.abspath(a.root), "reps": a.reps, "card": card(), "c2": [], "v512": [],
       "split": []}
for k in STEPS:
    for cap in CAPS:
        rec["c2"].append(run(N - V * (k + 1), V, cap, f"step{k}"))
for k in (0, 16):
    for cap in (32, 48):
        rec["v512"].append(run(N - 512 * (k + 1), 512, cap, f"v512_step{k}"))
for k in (24, 48):
    n = N - V * (k + 1)
    rec["split"].append(run(n, 32, 32, f"step{k}_v32"))
rec["split"].append(run(2048, 256, 1, "one_cta_2048"))
rec["split"].append(run(2048, 32, 1, "one_cta_2048_v32"))
rec["card_after"] = card()
line = json.dumps(rec)
print(line)
if a.out:
    with open(a.out, "w") as f:
        f.write(line + "\n")
