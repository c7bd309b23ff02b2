#!/usr/bin/env python
"""bench_table_fit.py — how the headline's hash-aggregate kernel slows as its table outgrows the L2 (DESIGN §5).

The input is the headline's: 1e9 (u64,u64) AoS rows resident in HBM, SUM, 8 map x 8 reduce partitions, the maps
borrowed into one shared table as bench.py does.  Only the table changes between points:

  footprint  n_distinct 1.25e5 .. 2e6, each with a hint that gives a table at load ~0.48, so every row issues the
             same requests and only the table's size (4 .. 64 MB) moves;
  load       1e6 keys with hints that force a table size: 0.8e6 gives 2^21 slots (load 0.48), 1.6e6 gives 2^22 slots
             (load 0.24), and no hint gives the size bench.py gets from the sample estimate.  --load-hints takes
             other hints, for a library built with another sizing rule (VEGA_B200_LIB).

Each point is timed with CUDA events on the library's stream (hot_kernel_ms: the hash_agg launches alone) over
--steps steps after --warmup, and prints one JSON line: table slots and bytes, load, ns per row of the hot kernel
and the whole step.  The card's name and power limit are read in the same run.

  python tools/bench_table_fit.py [--rows 1e9] [--steps 10] [--warmup 2] [--points footprint,load]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vega_b200 as vb
from vega_b200 import _lib as L
from vega_b200 import dist as vdist

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=float, default=1e9)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--points", default="footprint,load")
ap.add_argument("--load-hints", default="0.8,1.6",
                help="load points: hint = this x 1e6 (1e6 keys; the table the library chooses for each hint is reported)")
args = ap.parse_args()
assert torch.cuda.is_available(), "bench_table_fit.py needs a GPU"
N, M, R = int(args.rows), 8, 8


def card():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        info["power_limit_w"], info["sm_max_mhz"] = float(out[0]), float(out[1])
    except Exception:
        pass
    return info


sc = vb.Context(0, profile=True)
engine = vdist.CudaEngine(sc)
stream = sc.stream()
rows = torch.empty((N, 2), dtype=torch.int64, device="cuda")
gpu = card()


def point(kind, D, hint):
    sc.gen_pairs(out_rows=rows, first=0, n=N, mode="uniform", n_distinct=D, seed_k=1, seed_v=2)
    starts = vb.slice_starts(N, M)
    maps = [(m, rows[int(starts[m]):int(starts[m + 1])], None) for m in range(M)]

    def step():
        return vdist.run_shuffle(engine, maps, M, R, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, 0, 1, hint=hint)

    for _ in range(args.warmup):
        step().free()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    hot, st = [], None
    e0.record(stream)
    for _ in range(args.steps):
        sh = step()
        st = sh.stats()
        hot.append(st["hot_kernel_ms"])
        sh.free()
    e1.record(stream)
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps
    hot.sort()
    slots = st["table_slots"]
    line = {"kind": kind, "n_distinct": D, "hint": hint, "table_slots": slots, "table_mb": slots * 16 / 2 ** 20,
            "load": D / slots if slots else None, "restarts": st["table_restarts"],
            "hot_ms_median": hot[len(hot) // 2], "hot_ms_min": hot[0], "hot_ms_max": hot[-1],
            "hot_ns_per_row": hot[len(hot) // 2] * 1e6 / N, "step_ms": step_ms, "rows": N, "steps": args.steps, "gpu": gpu}
    print(json.dumps(line), flush=True)


kinds = args.points.split(",")
if "footprint" in kinds:
    for D in (125_000, 250_000, 500_000, 1_000_000, 2_000_000):
        cap = 1 << (int(D / 0.48) - 1).bit_length()        # the power of two just above D / 0.48
        point("footprint", D, int(cap * 0.4))               # choose_log_cap: 2.5 x hint rounded up to a power of two
if "load" in kinds:
    for x in (float(v) for v in args.load_hints.split(",")):
        point("load", 1_000_000, int(x * 1e6))
    point("load", 1_000_000, 0)                              # no hint: the size bench.py gets from the sample estimate
