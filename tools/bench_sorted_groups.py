"""group_by_key with each key's values in input order and sorted on the device (vb_shuffle_set_value_order), timed in
the same process, alternating the two orders.

    python tools/bench_sorted_groups.py [--reps 3] [--scale 1.0] [--only NAME]

Workloads (rows and keys times --scale):
  medium   10^9 rows over 10^6 uniform keys: ~1000 values per list, the shared-memory path
  tiny     10^8 rows over 5 x 10^7 uniform keys: lists of 1 to ~10 values, the smallest size classes
  zipf     10^8 rows over 10^7 keys, Zipf 1.1: a few very long lists (radix path) and a long tail of short ones
  large    one key with 10^8 values: the radix path alone
One JSON line per workload:
  map_seal_ms_input / _sorted   median wall time of the map call and the seal (device input, one map task, 64
                                partitions), synchronised; the orders alternate, after one warm-up of each
  sort_cost_ms                  the difference of the two medians
  segsort_kernel_ms             device time of the segmented sort's own kernels (seg_*, narrow_u32) in one sorted
                                seal under torch.profiler, a run of its own; the radix passes of the large lists are
                                counted in sort_cost_ms only, since they share their kernels with the grouping
  segsort_gbps                  16 B (read and write) per value in a list of 2 or more, over segsort_kernel_ms, and
                                hbm_share its share of 3.35 TB/s (HBM bound)
  check                         partition 0 of the sorted result equals the input-order one sorted by numpy
The card's name and power limit are read in the same process.  Nothing is written."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import vega_b200 as vb  # noqa: E402
from tests import sorted_groups_ref as S  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402
from vega_b200.rdd import Shuffle, _Col  # noqa: E402

M, R = 1, 64                      # one map task over the device input: no gathered copy, so 10^9 rows fit in 80 GB
WORKLOADS = {                      # name: (rows, distinct keys, generator, zipf s)
    "medium": (10 ** 9, 10 ** 6, "uniform", 0.0),
    "tiny": (10 ** 8, 5 * 10 ** 7, "uniform", 0.0),
    "zipf": (10 ** 8, 10 ** 7, "zipf", 1.1),
    "large": (10 ** 8, 1, "uniform", 0.0),
}
HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")][:2]
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def col(t, code):
    c = _Col(t, role="key")
    c.code = code
    return c


def seal(sc, kc, vc, n, order, keep=False):
    """Map and seal one GROUP shuffle; (wall ms, the shuffle if keep else None)."""
    starts = vb.slice_starts(n, M)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sh = Shuffle(sc, M, R, L.VB_U64, L.VB_I64, L.VB_AGG_GROUP, value_order=order)
    for m in range(M):
        sh.map(m, kc, vc, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    ms = (time.perf_counter() - t0) * 1e3
    if keep:
        return ms, sh
    sh.free()
    return ms, None


def sorted_values(sh):
    """Values in lists of 2 or more, over every partition."""
    total = 0
    for r in range(R):
        nk, nv = sh.reduce_size(r)
        if nv > nk:
            _, o, _ = sh.reduce(r)
            lens = np.diff(o.astype(np.int64))
            total += int(lens[lens >= 2].sum())
    return total


def run(sc, name, reps, scale):
    rows, distinct, mode, s = WORKLOADS[name]
    n, d = int(rows * scale), max(1, int(distinct * scale))
    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    vals = torch.empty(n, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=keys, out_vals=vals, n=n, mode=mode, n_distinct=d, zipf_s=s)
    kc, vc = col(keys, L.VB_U64), col(vals, L.VB_I64)
    t = {L.VB_VALORDER_INPUT: [], L.VB_VALORDER_ASC: []}
    for order in t:
        seal(sc, kc, vc, n, order)                           # warm-up
    for _ in range(reps):
        for order in t:
            t[order].append(seal(sc, kc, vc, n, order)[0])
    # check and bytes from one kept pair
    _, a = seal(sc, kc, vc, n, L.VB_VALORDER_INPUT, keep=True)
    pk, po, pv = a.reduce(0)
    a.free()
    _, b = seal(sc, kc, vc, n, L.VB_VALORDER_ASC, keep=True)
    sk, so, sv = b.reduce(0)
    touched = sorted_values(b)
    b.free()
    want, got = S.triples(pk, po, S.sort_lists(po, pv)), S.triples(sk, so, sv)
    ok = all(np.array_equal(x, y) for x, y in zip(want, got))
    # the segmented sort's kernels, profiled in a run of their own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        seal(sc, kc, vc, n, L.VB_VALORDER_ASC)
        torch.cuda.synchronize()
    names = ("seg_classify", "seg_sort_cta", "seg_bounds", "seg_move", "narrow_u32")
    kus = sum(e.device_time_total for e in prof.key_averages() if any(x in e.key for x in names))
    med = {o: float(np.median(v)) for o, v in t.items()}
    kms = kus / 1e3
    gbps = 16 * touched / (kms / 1e3) / 1e9 if kms else None
    return {"workload": name, "rows": n, "distinct": d, "zipf_s": s, "map_seal_ms_input": round(med[L.VB_VALORDER_INPUT], 2),
            "map_seal_ms_sorted": round(med[L.VB_VALORDER_ASC], 2),
            "sort_cost_ms": round(med[L.VB_VALORDER_ASC] - med[L.VB_VALORDER_INPUT], 2),
            "runs_input": [round(x, 2) for x in t[L.VB_VALORDER_INPUT]], "runs_sorted": [round(x, 2) for x in t[L.VB_VALORDER_ASC]],
            "values_in_lists_of_2_plus": touched, "segsort_kernel_ms": round(kms, 3),
            "segsort_gbps": None if gbps is None else round(gbps, 1), "hbm_share": None if gbps is None else round(gbps * 1e9 / HBM, 3),
            "check": ok}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--only", choices=list(WORKLOADS), action="append")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sorted_groups needs a GPU")
    name, limit = card()
    with vb.Context(0) as sc:
        for w in a.only or list(WORKLOADS):
            out = run(sc, w, a.reps, a.scale)
            out.update(gpu=name, power_limit=limit)
            print(json.dumps(out), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
