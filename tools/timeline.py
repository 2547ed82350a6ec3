"""tools/timeline.py -- per-region device time of one factorisation at a bench configuration, WITHOUT serialising the run:
CUDA event pairs on the launching streams (cflx_lu_set_profiling mode 2), region names = the reference's semiprof regions.
    python tools/timeline.py --gpus 1 [--mode 2] [--out timeline.json]
With mode 2 it also prints, per look-ahead panel k + 1, the pivot search on the side stream (step1_lup) next to the part
of step k's trailing update it overlaps ("lookahead_per_step": start and duration in ms from the first recorded event).
    python -m torch.distributed.run --nproc-per-node 4 --master-addr 127.0.0.1 tools/timeline.py --gpus 4 ...
Every rank prints/saves its own table (roles differ: panel column, pivot row, other layers)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
WORKLOADS = {1: (16384, 256, (1, 1, 1)), 2: (32768, 512, (1, 1, 2)), 4: (32768, 512, (2, 2, 1)), 8: (65536, 512, (2, 2, 2))}

ap = argparse.ArgumentParser()
ap.add_argument("--gpus", type=int, default=1)
ap.add_argument("--mode", type=int, default=2)
ap.add_argument("--out", default="")
ap.add_argument("--N", type=int, default=0)
ap.add_argument("--v", type=int, default=0)
a = ap.parse_args()
rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
import conflux_b200 as cb  # noqa: E402
from conflux_b200 import _lib  # noqa: E402
if world > 1:
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("gloo", rank=rank, world_size=world)
N, v, g = WORKLOADS[a.gpus]
N, v = a.N or N, a.v or v
comm = cb.Comm.from_torch_distributed(device=int(os.environ.get("LOCAL_RANK", "0"))) if world > 1 else cb.Comm(1, 0, None, 0)
gv = cb.lu_params(N, N, v, *g, comm)
cb.LU_rep(gv, None, None, upload=True)
cb.LU_rep(gv, None, None, upload=False)
ms_plain = cb.LU_rep(gv, None, None, upload=False)
_lib.lib().cflx_lu_set_profiling(gv._h, a.mode)
ms = cb.LU_rep(gv, None, None, upload=False)
tl = cb.timeline(gv)
# per step: the look-ahead pivot search on the side stream against the part of the trailing update it overlaps (the next
# step6_dgemm launched on the main stream), traced from the per-instance records
records = tl.pop("records", [])
per_step = []
for i, (region, stream, start, dur) in enumerate(records):
    if region != "step1_lup" or stream != "side":
        continue
    nxt = next((r for r in records[i + 1:] if r[0] == "step6_dgemm" and r[1] == "main"), None)
    per_step.append({"panel": len(per_step) + 1, "lup_start_ms": start, "lup_ms": dur,
                     "update_start_ms": nxt[2] if nxt else None, "update_ms": nxt[3] if nxt else None})
_lib.lib().cflx_lu_set_profiling(gv._h, 0)
rec = {"workload": f"LU N={gv.N} v={gv.v} grid {g[0]}x{g[1]}x{g[2]}", "rank": gv.rank, "coords": [gv.pi, gv.pj, gv.pk],
       "mode": "serialising timers" if a.mode == 1 else "event pairs on the launching streams (not serialised)",
       "factor_ms_unprofiled": ms_plain, "factor_ms_profiled": ms, "gemm": "ozaki (int8 wgmma)" if _lib.lib().cflx_lu_uses_ozaki(gv._h) else "dmma", "regions": tl,
       "lookahead_per_step": per_step}
out = a.out or ""
if out:
    path = out.replace(".json", f"_rank{gv.rank}.json") if world > 1 else out
    json.dump(rec, open(path, "w"), indent=1)
print(json.dumps(rec))
gv.free_comms()
comm.close()
if world > 1:
    dist.destroy_process_group()
