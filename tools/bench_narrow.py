#!/usr/bin/env python
"""bench_narrow.py — aggregate, then join (not the bench.py contract; feeds DESIGN.md §5).

Two sides of --rows device rows each over --keys keys per side, --shared of them on both sides.  SUM on both sides,
then the inner join and the cogroup of every partition, outputs on the device.  Three arms, one JSON line each:
  views      the sums joined through vb_shuffle_create_narrow views (no second shuffle)
  reshuffle  the sums shuffled again on the device (each result partition one map task of a COGROUP shuffle)
  host       today's workaround: collect the sums to the host, parallelize them, join
Wall time per arm (host clock around work that ends in a device synchronise), median of --reps after one warm-up run,
and the device ms per kernel class of one extra profiled run, with the card, power limit and SM clock read in the same
process."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vega_b200 as vb
from vega_b200 import _lib as L

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=float, default=5e8)
ap.add_argument("--keys", type=float, default=1e7)
ap.add_argument("--shared", type=float, default=0.02)
ap.add_argument("--splits", type=int, default=16)
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
N, D, R = int(args.rows), int(args.keys), args.splits

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
g = torch.Generator(device="cuda").manual_seed(1)
MUL = 0x9E3779B97F4A7C15 - (1 << 64)
ka = torch.randint(0, D, (N,), device="cuda", generator=g) * MUL + 12345
kb = (torch.randint(0, D, (N,), device="cuda", generator=g) + int(D * (1 - args.shared))) * MUL + 12345
va = torch.randint(0, 1 << 40, (N,), device="cuda", generator=g)
vb_ = torch.randint(0, 1 << 40, (N,), device="cuda", generator=g)
torch.cuda.synchronize()


def joins(sc, a, b):
    """Inner join and cogroup of every partition of two sealed COGROUP-kind sides, into device tensors."""
    lib, rows = sc._lib, 0
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    for r in range(R):
        n = ctypes.c_uint64()
        L.check(lib.vb_join_size(a._h, b._h, r, ctypes.byref(n)))
        out = [torch.empty(n.value, dtype=torch.int64, device="cuda") for _ in range(3)]
        L.check(lib.vb_join(a._h, b._h, r, *[p(t) for t in out], L.VB_DEVICE))
        nk, nl, nr = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        L.check(lib.vb_cogroup_size(a._h, b._h, r, ctypes.byref(nk), ctypes.byref(nl), ctypes.byref(nr)))
        cg = [torch.empty(x, dtype=torch.int64, device="cuda") for x in (nk.value, nk.value + 1, nl.value, nk.value + 1, nr.value)]
        L.check(lib.vb_cogroup(a._h, b._h, r, *[p(t) for t in cg], L.VB_DEVICE))
        rows += n.value
    return rows


def arm(sc, name):
    """One run of the pipeline; returns (joined rows, every shuffle it made)."""
    sa = sc.parallelize((ka, va), R).reduce_by_key("sum", R)
    sb = sc.parallelize((kb, vb_), R).reduce_by_key("sum", R)
    if name == "views":
        a, b = sa._cogroup_side(R), sb._cogroup_side(R)
    elif name == "reshuffle":
        a, b = sa._reshuffled(R), sb._reshuffled(R)
    else:
        ha, hb = (sc.parallelize(s.collect(), R) for s in (sa, sb))
        a, b = vb.JoinedRdd(ha, hb, R)._run()
    rows = joins(sc, a, b)
    torch.cuda.synchronize()
    return rows, [sa._sh, sb._sh, a, b]


for name in ("views", "reshuffle", "host"):
    with vb.Context(0) as sc:
        arm(sc, name)                                       # warm-up
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rows, shs = arm(sc, name)
            times.append((time.perf_counter() - t0) * 1e3)
            for s in shs:
                s.free()
        sc.set_profile(True)
        _, shs = arm(sc, name)
        kms = {c: round(sum(s.stats()["kernels"][c]["ms"] for s in shs), 3) for c in L.KERNEL_CLASSES}
    print(json.dumps({"arm": name, "rows": N, "keys": D, "shared": args.shared, "splits": R, "joined_rows": rows,
                      "ms_median": round(sorted(times)[len(times) // 2], 2), "ms_all": [round(t, 2) for t in times],
                      "kernel_ms": kms, "gpu": card}), flush=True)
