#!/usr/bin/env python
"""bench_str_narrow.py — aggregate by word, then join by word (not the bench.py contract; feeds DESIGN.md §5).

Two sides of --rows device rows each with word-like keys ('w' + the hex digits of a rank, built on the device by
tests/test_gpu_str_keys._device_words) over --keys words per side, --shared of them on both sides.  SUM on both sides,
then the inner join (vb_join_n_str) and the cogroup (vb_cogroup_n_str) of every partition, outputs on the device.
Three arms, one JSON line each:
  views      the sums joined through vb_shuffle_create_narrow_str views (StrCoGroupedRdd under the same num_splits)
  reshuffle  the sums shuffled again on the device (StrCoGroupedRdd._reshuffled: each result partition one map task of a
             String GROUP shuffle), the path a String reduce parent took before views
  host       collect the sums to the host, parallelize them, join
Wall time per arm (host clock around work that ends in a device synchronise), median of --reps after one warm-up run,
and the device ms per kernel class of one extra profiled run, with the card, power limit and SM clock read in the same
process.  Writes nothing."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import vega_b200 as vb  # noqa: E402
from tests.test_gpu_str_keys import _device_words  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=float, default=5e7)
ap.add_argument("--keys", type=float, default=1e6)
ap.add_argument("--shared", type=float, default=0.02)
ap.add_argument("--splits", type=int, default=16)
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
N, D, R = int(args.rows), int(args.keys), args.splits

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
g = torch.Generator(device="cuda").manual_seed(1)
ka = _device_words(torch.randint(0, D, (N,), device="cuda", generator=g))
kb = _device_words(torch.randint(0, D, (N,), device="cuda", generator=g) + int(D * (1 - args.shared)))
va = torch.randint(0, 1 << 40, (N,), device="cuda", generator=g)
vb_ = torch.randint(0, 1 << 40, (N,), device="cuda", generator=g)
torch.cuda.synchronize()


def joins(sc, a, b):
    """Inner join and cogroup of every partition of two sealed String GROUP-kind sides, into device tensors."""
    lib, rows = sc._lib, 0
    sides = (ctypes.c_void_p * 2)(a._h.value, b._h.value)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    dev = lambda n, dt=torch.int64: torch.empty(n, dtype=dt, device="cuda")
    for r in range(R):
        nr, nk, nb = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        L.check(lib.vb_join_n_str_size(sides, 2, r, 0b11, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)))
        ko, kbs, ro, v, w = dev(nk.value + 1), dev(nb.value, torch.uint8), dev(nk.value + 1), dev(nr.value), dev(nr.value)
        L.check(lib.vb_join_n_str(sides, 2, r, 0b11, p(ko), p(kbs), p(ro), (ctypes.c_void_p * 2)(p(v), p(w)), None, L.VB_DEVICE))
        nv = (ctypes.c_uint64 * 2)()
        L.check(lib.vb_cogroup_n_str_size(sides, 2, r, ctypes.byref(nk), ctypes.byref(nb), nv))
        ko, kbs = dev(nk.value + 1), dev(nb.value, torch.uint8)
        offs, vals = [dev(nk.value + 1) for _ in range(2)], [dev(nv[j]) for j in range(2)]
        L.check(lib.vb_cogroup_n_str(sides, 2, r, p(ko), p(kbs), (ctypes.c_void_p * 2)(*[p(o) for o in offs]),
                                     (ctypes.c_void_p * 2)(*[p(x) for x in vals]), L.VB_DEVICE))
        rows += nr.value
    return rows


def arm(sc, name):
    """One run of the pipeline; returns (joined rows, every shuffle it made)."""
    sa = sc.parallelize(ka, R, values=va).reduce_by_key("sum", R)
    sb = sc.parallelize(kb, R, values=vb_).reduce_by_key("sum", R)
    if name == "views":
        a, b = vb.StrCoGroupedRdd([sa, sb], R)._sides()[0]
    elif name == "reshuffle":
        cg = vb.StrCoGroupedRdd([sa, sb], R)
        a, b = (cg._reshuffled(s._run(), 0, None, L.VB_I64) for s in (sa, sb))
    else:
        ha, hb = (sc.parallelize(k, R, values=v) for k, v in (s.collect() for s in (sa, sb)))
        a, b = vb.StrCoGroupedRdd([ha, hb], R)._sides()[0]
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
