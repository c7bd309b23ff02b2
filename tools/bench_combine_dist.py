"""combine_by_key across ranks on one GPU (DESIGN.md §5): the one-process combine shuffle (map + seal, W = 1) against
W = 2 and 8 ranks of the same shuffle in one process (map + export + import + seal, summed over the ranks).

2e8 device rows with tools/bench_ops.py's three value columns and its spec: sum(v0), min(v1), max(v1), mean(v2), count
(5 accumulators), uniform over 10^4 and 10^6 keys, 8 map tasks and 8 partitions.  Per (D, W): the wall time of map +
export + import + seal summed over the ranks, median of 3 after a warm-up (the column swap between the ranks is not
counted: it is the exchange, which NCCL does between GPUs); device ms per kernel class summed over the ranks, from one
separate profiled run; and the exported rows and bytes per row (8 (1 + n_acc) per distinct key and rank).  Prints one
JSON line with the card's name and power limit; writes nothing.
    python tools/bench_combine_dist.py [rows=2e8]
"""
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vega_b200 as vb  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402
from vega_b200 import dist as vdist  # noqa: E402
from bench import gpu_info  # noqa: E402
from tests.test_gpu_combine_multirank import swap  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 200_000_000
M = R = 8
SPEC = ([L.VB_U64, L.VB_I64, L.VB_F64],
        [(L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 1), (L.VB_AGG_MEAN, 2), (L.VB_AGG_COUNT, 0)])


def one_run(sc, W, K, cols, starts):
    """(wall ms of map + export + import + seal over the ranks, kernel ms by class, exported rows, n_acc)"""
    shs = [vb.Shuffle.combine_dist(sc, M, R, L.VB_U64, SPEC, r, W) for r in range(W)]
    wall, rows, n_acc, exports = 0.0, 0, 0, []
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for m in range(lo, hi):
            sh.map_cols(m, K, cols, int(starts[m]), int(starts[m + 1]))
        if W == 1:
            sh.seal()
        else:
            exports.append(sh.export_cols())
        torch.cuda.synchronize()
        wall += (time.perf_counter() - t0) * 1e3
    if W > 1:
        rows = sum(sum(c) for c, _, _ in exports)
        n_acc = exports[0][2].shape[0]
        recv = swap(exports)
        for sh, (k, a, c) in zip(shs, recv):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sh.import_cols(k, a, c)
            sh.seal()
            torch.cuda.synchronize()
            wall += (time.perf_counter() - t0) * 1e3
        del recv, exports
    kt = {}
    for sh in shs:
        for name, v in sh.stats()["kernels"].items():
            if v["ms"]:
                kt[name] = round(kt.get(name, 0.0) + v["ms"], 2)
    for sh in shs:
        sh.free()
    return wall, kt, rows, n_acc


card = gpu_info(0)
out = {"gpu": card.get("name"), "power_limit_w": card.get("power_limit_w"), "rows": n, "maps": M, "partitions": R,
       "spec": "sum(v0) min(v1) max(v1) mean(v2) count"}
with vb.Context(0) as sc:
    for label, D in [("1e4", 10_000), ("1e6", 1_000_000)]:
        keys = torch.empty(n, dtype=torch.int64, device="cuda")
        v0 = torch.empty(n, dtype=torch.int64, device="cuda")
        sc.gen_pairs(out_keys=keys, out_vals=v0, n=n, mode="uniform", n_distinct=D)
        v1 = v0 * 7 - 3_000_000
        v2 = v0.to(torch.float64) * 0.5
        torch.cuda.synchronize()
        K = vb.rdd._Col(keys)
        K.code = L.VB_U64
        cols = (vb.rdd._Col(v0), vb.rdd._Col(v1), vb.rdd._Col(v2))
        cols[0].code = L.VB_U64
        starts = vb.slice_starts(n, M)
        res = {}
        for W in [1, 2, 8]:
            one_run(sc, W, K, cols, starts)                                   # warm-up: pool, table sizes
            runs = [one_run(sc, W, K, cols, starts) for _ in range(3)]
            sc.set_profile(True)
            _, kt, rows, n_acc = one_run(sc, W, K, cols, starts)
            sc.set_profile(False)
            r = {"wall_ms_median": round(statistics.median(x[0] for x in runs), 2),
                 "wall_ms_runs": [round(x[0], 2) for x in runs], "kernels_ms": kt}
            if W > 1:
                r["export_rows"] = rows
                r["export_bytes_per_row"] = 8 * (1 + n_acc)
                r["export_bytes"] = 8 * (1 + n_acc) * rows
            res[f"W{W}"] = r
        out[label] = res
        del keys, v0, v1, v2, K, cols
        torch.cuda.empty_cache()
print(json.dumps(out))
