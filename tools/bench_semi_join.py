#!/usr/bin/env python
"""bench_semi_join.py — subtract_by_key and semi_join on the device (not the bench.py contract; feeds DESIGN.md §5).

Side 0: --rows (u64, u64) device rows over --keys keys, uniform or Zipf (--zipf s); the filter side: --filter-rows rows
over --filter-keys keys, half of them side-0 keys.  Two arms per op, on the same input, one JSON line each:
  semi     vb_semi_join_n over the two lazy COGROUP shuffles, every partition written to device tensors
  cogroup  the route without it: vb_cogroup_n of both sides to the host, then the rows kept by a numpy filter
Each arm shuffles the sides itself (map + seal are in the time).  Wall time (host clock around work that ends in a
device synchronise), median of --reps after one warm-up run; the rows each arm keeps must agree.  The card, its power
limit and SM clocks are read in the same process."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import vega_b200 as vb
from vega_b200 import _lib as L

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=float, default=1e8)
ap.add_argument("--keys", type=float, default=1e7)
ap.add_argument("--filter-rows", type=float, default=2e6)
ap.add_argument("--filter-keys", type=float, default=1e6)
ap.add_argument("--zipf", type=float, default=0.0, help="Zipf exponent of side 0's keys (0: uniform)")
ap.add_argument("--splits", type=int, default=16)
ap.add_argument("--reps", type=int, default=2)
args = ap.parse_args()
N, D, NF, DF, R = int(args.rows), int(args.keys), int(args.filter_rows), int(args.filter_keys), args.splits

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
MUL = 0x9E3779B97F4A7C15 - (1 << 64)
g = torch.Generator(device="cuda").manual_seed(1)
if args.zipf > 0:
    ranks = torch.from_numpy((np.random.default_rng(1).zipf(args.zipf, N) - 1) % D).cuda()
else:
    ranks = torch.randint(0, D, (N,), device="cuda", generator=g)
k0 = ranks * MUL + 12345
v0 = torch.randint(0, 1 << 40, (N,), device="cuda", generator=g)
# the filter side's keys: ranks D - DF/2 .. D + DF/2, so half of them are side-0 keys (the hottest Zipf ranks are not)
kf = (torch.randint(0, DF, (NF,), device="cuda", generator=g) + (D - DF // 2)) * MUL + 12345
vf = torch.zeros(NF, dtype=torch.int64, device="cuda")
del ranks
torch.cuda.synchronize()


def sides(sc):
    return vb.CoGroupedRdd([sc.parallelize((k0, v0), R), sc.parallelize((kf, vf), R)], R)._sides()


def semi(sc, req, exc):
    shs, arr = sides(sc)
    lib, rows, check = sc._lib, 0, 0
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    for r in range(R):
        n = ctypes.c_uint64()
        L.check(lib.vb_semi_join_n_size(arr, 2, r, req, exc, ctypes.byref(n)))
        k, v = (torch.empty(n.value, dtype=torch.int64, device="cuda") for _ in range(2))
        L.check(lib.vb_semi_join_n(arr, 2, r, req, exc, p(k), p(v), L.VB_DEVICE))
        rows += n.value
        check += int(v.sum()) if n.value else 0
    torch.cuda.synchronize()
    return rows, check, shs


def cogroup(sc, req, exc):
    shs, arr = sides(sc)
    lib, rows, check = sc._lib, 0, 0
    for r in range(R):
        nk, nv = ctypes.c_uint64(), (ctypes.c_uint64 * 2)()
        L.check(lib.vb_cogroup_n_size(arr, 2, r, ctypes.byref(nk), nv))
        keys = np.empty(nk.value, np.uint64)
        offs = [np.empty(nk.value + 1, np.uint64) for _ in range(2)]
        vals = [np.empty(nv[j], np.uint64) for j in range(2)]
        ptrs = lambda xs: (ctypes.c_void_p * 2)(*[x.ctypes.data for x in xs])
        L.check(lib.vb_cogroup_n(arr, 2, r, keys.ctypes.data_as(ctypes.c_void_p), ptrs(offs), ptrs(vals), L.VB_HOST))
        l0, l1 = (np.diff(o.astype(np.int64)) for o in offs)
        keep = (l0 > 0) & ((l1 > 0) if req else (l1 == 0))
        out_k = np.repeat(keys[keep], l0[keep])
        sel = np.repeat(keep, l0)
        out_v = vals[0][sel]
        rows += len(out_k)
        check += int(out_v.astype(np.int64).sum())
    return rows, check, shs


def run(fn, req, exc):
    with vb.Context(0) as sc:
        res = fn(sc, req, exc)                              # warm-up: module load, pools
        times = []
        for _ in range(args.reps):
            for s in res[2]:
                s.free()
            torch.cuda.synchronize()
            t = time.perf_counter()
            res = fn(sc, req, exc)
            times.append(time.perf_counter() - t)
        for s in res[2]:
            s.free()
    return float(np.median(times)), res[0], res[1]


for op, req, exc in (("subtract_by_key", 0, 0b10), ("semi_join", 0b10, 0)):
    got = {}
    for name, fn in (("semi", semi), ("cogroup", cogroup)):
        t, rows, check = run(fn, req, exc)
        got[name] = (rows, check)
        print(json.dumps({"op": op, "arm": name, "keys": "zipf %.2f" % args.zipf if args.zipf else "uniform", "rows": N,
                          "distinct": D, "filter_rows": NF, "filter_keys": DF, "splits": R, "rows_out": rows, "s": round(t, 4),
                          "rows_per_s": round(N / t), "card": card}), flush=True)
    assert got["semi"] == got["cogroup"], (op, got)
