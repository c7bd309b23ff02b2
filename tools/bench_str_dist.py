"""String keys across ranks on one GPU (DESIGN.md §5.4): the one-process string shuffle (map + seal, W = 1) against
W = 2 and 8 ranks of the same shuffle in one process (map + export + import + seal, summed over the ranks).

Keys are the word-like keys of tools/bench_str_ops.py ('w' + hex digits of a vb_gen_pairs rank, 2-12 bytes), built
on the device, uniform over 10^4 and 10^6 ranks, 8 map tasks and 8 partitions.  For count_by_key, reduce_by_key(sum)
and group_by_key: wall time of the second of two runs (the column swap between the ranks is not counted: it is the
exchange, which NCCL does between GPUs), device ms per kernel class summed over the ranks, and the bytes each rank
exports (4 B per key length, the key bytes, 4 B per GROUP value count, 8 B per value), per exported row (a combined
row for reduce ops, a value for GROUP) against the 16 B per row an integer-key rank exports.  Prints one JSON line with the card's name and power limit; writes nothing.
    python tools/bench_str_dist.py [rows=5e7]
"""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vega_b200 as vb  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402
from vega_b200 import dist as vdist  # noqa: E402
from tests.test_gpu_str_keys import _device_words  # noqa: E402
from tests.test_gpu_str_multirank import swap  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
M = R = 8
AGG = {"count": L.VB_AGG_COUNT, "sum": L.VB_AGG_SUM, "group": L.VB_AGG_GROUP}


def power_limit():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def kernels(shs):
    tot = {}
    for sh in shs:
        for k, v in sh.stats()["kernels"].items():
            if v["ms"]:
                tot[k] = round(tot.get(k, 0.0) + v["ms"], 2)
    return tot


def one_run(sc, W, op, col, vcol, starts):
    """(wall ms of map + export + import + seal over the ranks, kernel ms by class, bytes exported per rank)"""
    shs = [vb.StrShuffle(sc, M, R, L.VB_U64, AGG[op], rank=r, world=W) for r in range(W)]
    wall, sent, rows = 0.0, [], 0
    exports = []
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for m in range(lo, hi):
            sh.map(m, col, None if op == "count" else vcol, int(starts[m]), int(starts[m + 1]))
        if W == 1:
            sh.seal()
        else:
            exports.append(sh.export())
        torch.cuda.synchronize()
        wall += (time.perf_counter() - t0) * 1e3
    if W > 1:
        for (nk, nb, nv), _ in exports:
            sent.append(4 * sum(nk) + sum(nb) + (4 * sum(nk) if op == "group" else 0) + 8 * sum(nv))
            rows += sum(nv)
        recv = swap(exports)
        for sh, (cols, counts) in zip(shs, recv):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sh.import_(*cols, *counts)
            sh.seal()
            torch.cuda.synchronize()
            wall += (time.perf_counter() - t0) * 1e3
        del recv, exports
    kt = kernels(shs)
    for sh in shs:
        sh.free()
    return wall, kt, sent, rows


out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "rows": n, "maps": M, "partitions": R}
with vb.Context(0, profile=True) as sc:
    for label, D in [("1e4", 10_000), ("1e6", 1_000_000)]:
        ranks = torch.empty(n, dtype=torch.int64, device="cuda")
        vals = torch.empty(n, dtype=torch.int64, device="cuda")
        sc.gen_pairs(out_keys=ranks, out_vals=vals, n=n, mode="uniform", n_distinct=D)
        keys = _device_words(ranks & ((1 << 40) - 1))
        torch.cuda.synchronize()
        col, vcol = vb.rdd._StrCol(keys), vb.rdd._Col(vals, role="value")
        starts = vb.slice_starts(n, M)
        res = {"key_bytes": int(keys.data.numel())}
        for op in ["count", "sum", "group"]:
            for W in [1, 2, 8]:
                one_run(sc, W, op, col, vcol, starts)                     # warm-up: pool, index sizes
                wall, kt, sent, rows = one_run(sc, W, op, col, vcol, starts)
                r = {"wall_ms": round(wall, 2), "kernels_ms": kt}
                if sent:
                    r["export_bytes_per_rank_max"] = max(sent)
                    r["export_rows"] = rows
                    r["export_bytes_per_row"] = round(sum(sent) / max(rows, 1), 2)     # an integer key's row: 16 B
                res[f"{op}_W{W}"] = r
        out[label] = res
        del keys, ranks, vals, col, vcol
        torch.cuda.empty_cache()
print(json.dumps(out))
