"""String-key shuffles against the same ops on integer keys (DESIGN.md §5.2).

Keys are word-like ('w' + hex digits of a vb_gen_pairs rank, 2-12 bytes), built on the device; uniform over 10^4 and
10^6 ranks and Zipf(1.1) over 10^6.  For count_by_key, reduce_by_key(sum) and group_by_key on the string keys and on
the integer ranks: median wall time of map + seal over 3 runs, and the per-kernel-class device split of the last run.
Then, at 10^7 rows, the workaround without string keys (host dictionary encoding + an integer shuffle) against
count_by_value over the Python strs.  Prints one JSON line; writes nothing.
    python tools/bench_str_ops.py [rows=5e7]
"""
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vega_b200 as vb  # noqa: E402
from tests.test_gpu_str_keys import _device_words  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
out = {"gpu": torch.cuda.get_device_name(0), "rows": n}
with vb.Context(0, profile=True) as sc:
    for label, mode, D in [("1e4", "uniform", 10_000), ("1e6", "uniform", 1_000_000), ("zipf1.1", "zipf", 1_000_000)]:
        ranks = torch.empty(n, dtype=torch.int64, device="cuda")
        vals = torch.empty(n, dtype=torch.int64, device="cuda")
        sc.gen_pairs(out_keys=ranks, out_vals=vals, n=n, mode=mode, n_distinct=D, zipf_s=1.1)
        ranks = ranks & ((1 << 40) - 1)
        keys = _device_words(ranks)
        torch.cuda.synchronize()
        real = int(torch.unique(ranks).numel())
        kb = int(keys.data.numel())
        res = {"distinct": real, "key_bytes": kb}
        for op in ["count", "sum", "group"]:
            for kind in ["str", "u64"]:
                ts, kt = [], None
                for rep in range(3):
                    if kind == "str":
                        rdd = sc.parallelize(keys, 8, values=vals)
                    else:
                        rdd = sc.parallelize(ranks, 8, values=vals)
                    s = rdd.group_by_key(8) if op == "group" else rdd.count_by_key(8) if op == "count" else rdd.reduce_by_key("sum", 8)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    sh = s._run()
                    torch.cuda.synchronize()
                    ts.append((time.perf_counter() - t0) * 1e3)
                    st = sh.stats()
                    kt = {k: round(v["ms"], 2) for k, v in st["kernels"].items() if v["ms"]}
                    sh.free()
                res[f"{op}_{kind}"] = {"median_ms": round(statistics.median(ts), 2), "kernels_ms": kt}
        out[label] = res
        del keys, ranks, vals
        torch.cuda.empty_cache()
    # workaround users have today at 1e7 rows: host dictionary encoding + integer shuffle
    m = 10_000_000
    ranks = torch.empty(m, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=ranks, n=m, mode="uniform", n_distinct=1_000_000)
    words = _device_words(ranks & ((1 << 40) - 1)).to_strs().tolist()
    t0 = time.perf_counter()
    d = {}
    ids = np.fromiter((d.setdefault(w, len(d)) for w in words), dtype=np.uint64, count=m)
    t1 = time.perf_counter()
    k, c = sc.parallelize(ids, 8).count_by_value().collect()
    t2 = time.perf_counter()
    k2, c2 = sc.parallelize(words, 8).count_by_value().collect()
    t3 = time.perf_counter()
    out["workaround_1e7"] = {"host_encode_ms": round((t1 - t0) * 1e3, 1), "int_count_by_value_ms": round((t2 - t1) * 1e3, 1),
                             "str_count_by_value_from_python_strs_ms": round((t3 - t2) * 1e3, 1)}
print(json.dumps(out))
