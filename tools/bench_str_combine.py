"""combine_by_key over String keys against the ways to get the same results without it (DESIGN.md §5.6).

`rows` rows (default 5e7) of word-like device keys ('w' + hex digits of a rank, built on the device by
tests/test_gpu_str_keys._device_words) over uniform ranks with 1e4 and 1e6 distinct keys, and Zipf(1.1) ranks over 1e6,
with the combine spec of tools/bench_ops.py: sum(v0), min(v1), max(v1), mean(v2) and count (v0 = gen_pairs' values,
v1 = 7 v0 - 3e6 as i64, v2 = v0 / 2 as f64), 8 map slices -> 8 partitions.  Arms, each the median wall time of 3 runs
after a warm-up, from the first map call to the end of the seal:
  (a) the String combine, at W = 1, 2 and 8 ranks in one process (every rank's map, export, an in-process column swap,
      import and seal, as tests/test_gpu_str_combine_multirank.py runs them);
  (b) the same results from five single-column String shuffles (sum v0, min v1, max v1, sum v2, count);
  (c) the integer combine over the ranks themselves (what a caller who already has integer ids runs).
Then one profiled run of (a) at W = 1 and of (b) on a profiling context: device ms per kernel class.  Prints one JSON line
with the card name and power limit read in the same process; writes nothing.
    python tools/bench_str_combine.py [rows=5e7]
"""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vega_b200 as vb  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402
from vega_b200 import dist as vdist  # noqa: E402
from vega_b200.rdd import Shuffle, StrShuffle, _Col, _StrCol  # noqa: E402
from tests import multirank as MR  # noqa: E402
from tests.test_gpu_str_keys import _device_words  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
M = R = 8
SPEC = [(L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 1), (L.VB_AGG_MEAN, 2), (L.VB_AGG_COUNT, 0)]
SINGLES = [(L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 1), (L.VB_AGG_SUM, 2), (L.VB_AGG_COUNT, None)]
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip(), "rows": n, "map_slices": M, "partitions": R,
       "spec": "sum(v0) min(v1) max(v1) mean(v2) count", "cases": {}}


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def med3(f):
    timed(f)                                        # warm-up
    return round(statistics.median(timed(f)[0] for _ in range(3)), 2)


def kernels(stats):
    tot = {}
    for st in stats:
        for k, v in st["kernels"].items():
            tot[k] = tot.get(k, 0.0) + v["ms"]
    return {k: round(v, 2) for k, v in tot.items() if v}


def str_combine(sc, K, cols, W, hint):
    multi = ([c.code for c in cols], SPEC)
    starts = vb.slice_starts(n, M)
    shs = [StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, hint=hint, rank=r, world=W, multi=multi) for r in range(W)]
    for r in range(W):
        lo, hi = vdist.map_block(r, W, M)
        for m in range(lo, hi):
            shs[r].map_cols(m, K, cols, int(starts[m]), int(starts[m + 1]))
    if W > 1:
        exports = [sh.export_cols() for sh in shs]
        recv = MR.swap_columns([([ln, b, a.t()], [nk, nb, nk]) for (nk, nb), (ln, b, a) in exports])
        for sh, (rc, rs) in zip(shs, recv):
            sh.import_cols(rc[0], rc[1], rc[2].t().contiguous(), rs[0], rs[1])
    for sh in shs:
        sh.seal()
    stats = [sh.stats() for sh in shs]
    for sh in shs:
        sh.free()
    return stats


def str_singles(sc, K, cols, hint):
    starts = vb.slice_starts(n, M)
    stats = []
    for agg, c in SINGLES:
        col = cols[c] if c is not None else None
        sh = StrShuffle(sc, M, R, col.code if col is not None else L.VB_U64, agg, hint=hint)
        for m in range(M):
            sh.map(m, K, col, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        stats.append(sh.stats())
        sh.free()
    return stats


def int_combine(sc, ranks, cols, hint):
    starts = vb.slice_starts(n, M)
    k = _Col(ranks)
    k.code = L.VB_U64
    sh = Shuffle(sc, M, R, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, hint=hint, multi=([c.code for c in cols], SPEC))
    for m in range(M):
        sh.map_cols(m, k, cols, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    st = sh.stats()
    sh.free()
    return [st]


sc = vb.Context(0)
prof = vb.Context(0, profile=True)
for name, mode, D, s in [("uniform 1e4", "uniform", 10_000, 0.0), ("uniform 1e6", "uniform", 1_000_000, 0.0),
                         ("zipf 1.1 over 1e6", "zipf", 1_000_000, 1.1)]:
    ranks = torch.empty(n, dtype=torch.int64, device="cuda")
    v0 = torch.empty(n, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=ranks, out_vals=v0, n=n, mode=mode, n_distinct=D, seed_k=5, zipf_s=s)
    ranks &= (1 << 40) - 1
    v1 = v0 * 7 - 3_000_000
    v2 = v0.to(torch.float64) * 0.5
    keys = _device_words(ranks)
    torch.cuda.synchronize()
    K = _StrCol(keys)
    cols = (_Col(v0, role="value"), _Col(v1, role="value"), _Col(v2, role="value"))
    cols[0].code = L.VB_U64
    hint = D if mode == "uniform" else 0
    case = {"key_bytes": int(keys.data.numel()), "distinct": int(torch.unique(ranks).numel())}
    for W in (1, 2, 8):
        case[f"str_combine_W{W}_ms"] = med3(lambda: str_combine(sc, K, cols, W, hint))
    case["five_str_shuffles_ms"] = med3(lambda: str_singles(sc, K, cols, hint))
    case["int_rank_combine_ms"] = med3(lambda: int_combine(sc, ranks, cols, hint))
    case["device_ms_str_combine_W1"] = kernels(str_combine(prof, K, cols, 1, hint))
    case["device_ms_five_str_shuffles"] = kernels(str_singles(prof, K, cols, hint))
    case["device_ms_int_rank_combine"] = kernels(int_combine(prof, ranks, cols, hint))
    out["cases"][name] = case
    del ranks, v0, v1, v2, keys, K, cols
    torch.cuda.empty_cache()
prof.close()
sc.close()
print(json.dumps(out))
