"""sort_by_key over String keys against the ways to get the same order without it (DESIGN.md §5.7).

`rows` rows (default 5e7) with i64 payloads (gen_pairs' values), 8 map slices -> 8 partitions, over five key sets built
on the device:
  uniform 1e4 / uniform 1e6 / zipf 1.1 over 1e6   word-like keys, 'w' + the hex digits of a rank
                                                 (tests/test_gpu_str_keys._device_words), 2 to 11 bytes;
  all distinct                                   the same words over 63-bit hashed ranks, 2 to 17 bytes;
  url, 32-byte shared prefix                     'https://example.com/catalog/item' + 8 hex digits of a 1e6-rank:
                                                 every key ties with every other for the prefix's rounds.
Per key set, one JSON line:
  str_sort_ms           median of 3 wall times (after a warm-up) from the first map call to the end of the seal;
  device_ms             one profiled run: device ms per kernel class; `dict` is the encode, `str_order` the ordering of
                        the distinct keys (radix passes included), rp_* the row sort;  str_order_launches;
  int_rank_sort_ms      the integer sort_by_key of the u64 ranks on the same rows (what a caller with ids runs);
  host_workaround_ms    at 1e7 rows, one run: np.unique over the keys as Python strs, then the integer sort of the
                        inverse indices (the encode of the strs themselves is not timed).
The card name and power limit are read in the same process; nothing is written.
    python tools/bench_str_sort.py [rows=5e7]
"""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vega_b200 as vb  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402
from vega_b200.rdd import Shuffle, StrShuffle, _Col, _StrCol  # noqa: E402
from tests.test_gpu_str_keys import _device_words  # noqa: E402

M = R = 8
PREFIX = b"https://example.com/catalog/item"
assert len(PREFIX) == 32


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def med3(f):
    timed(f)                                        # warm-up
    return round(statistics.median(timed(f)[0] for _ in range(3)), 2)


def url_keys(ranks):
    """PREFIX + 8 zero-padded hex digits of each rank: 40-byte keys, built on the device."""
    shift = 4 * torch.arange(7, -1, -1, device=ranks.device)
    hexc = torch.tensor(list(b"0123456789abcdef"), dtype=torch.uint8, device=ranks.device)
    data = torch.empty((len(ranks), 40), dtype=torch.uint8, device=ranks.device)
    data[:, :32] = torch.tensor(list(PREFIX), dtype=torch.uint8, device=ranks.device)
    data[:, 32:] = hexc[(ranks[:, None] >> shift[None, :]) & 15]
    return vb.StrKeys(torch.arange(len(ranks) + 1, dtype=torch.int64, device=ranks.device) * 40, data.reshape(-1))


def str_sort(sc, K, V, rows):
    starts = vb.slice_starts(rows, M)
    sh = StrShuffle(sc, M, R, L.VB_I64, L.VB_AGG_SORT, sort=True)
    for m in range(M):
        sh.map(m, K, V, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    st = sh.stats()
    sh.free()
    return st


def int_sort(sc, ranks, V, rows):
    starts = vb.slice_starts(rows, M)
    k = _Col(ranks)
    k.code = L.VB_U64
    sh = Shuffle(sc, M, R, L.VB_U64, L.VB_I64, L.VB_AGG_SORT)
    for m in range(M):
        sh.map(m, k, V, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    st = sh.stats()
    sh.free()
    return st


def host_workaround(sc, strs, vals):
    u, inv = np.unique(strs, return_inverse=True)
    ids = torch.from_numpy(inv.astype(np.int64)).cuda()
    return int_sort(sc, ids, _Col(torch.from_numpy(vals).cuda(), role="value"), len(strs))


def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
    host_rows = min(n, 10_000_000)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip(), "rows": n, "map_slices": M, "partitions": R}
    sc = vb.Context(0)
    prof = vb.Context(0, profile=True)
    for name, mode, D, s in [("uniform 1e4", "uniform", 10_000, 0.0), ("uniform 1e6", "uniform", 1_000_000, 0.0),
                             ("zipf 1.1 over 1e6", "zipf", 1_000_000, 1.1), ("all distinct", "unique", 0, 0.0),
                             ("url, 32-byte shared prefix", "uniform", 1_000_000, 0.0)]:
        ranks = torch.empty(n, dtype=torch.int64, device="cuda")
        vals = torch.empty(n, dtype=torch.int64, device="cuda")
        sc.gen_pairs(out_keys=ranks, out_vals=vals, n=n, mode=mode, n_distinct=max(D, 1), seed_k=5, zipf_s=s)
        ranks &= (1 << 63) - 1 if mode == "unique" else (1 << 28) - 1
        keys = url_keys(ranks) if name.startswith("url") else _device_words(ranks)
        torch.cuda.synchronize()
        K, V = _StrCol(keys), _Col(vals, role="value")
        case = {"keys": name, **gpu, "key_bytes": int(keys.data.numel()), "distinct": int(torch.unique(ranks).numel())}
        case["str_sort_ms"] = med3(lambda: str_sort(sc, K, V, n))
        st = str_sort(prof, K, V, n)
        case["device_ms"] = {k: round(v["ms"], 2) for k, v in st["kernels"].items() if v["ms"]}
        case["str_order_launches"] = st["kernels"]["str_order"]["launches"]
        case["int_rank_sort_ms"] = med3(lambda: int_sort(sc, ranks, V, n))
        hk = vb.StrKeys(keys.offsets[:host_rows + 1].cpu().numpy(), keys.data[:int(keys.offsets[host_rows])].cpu().numpy())
        strs = hk.to_strs()
        hv = vals[:host_rows].cpu().numpy()
        case["host_workaround_rows"] = host_rows
        case["host_workaround_ms"] = round(timed(lambda: host_workaround(sc, strs, hv))[0], 1)
        print(json.dumps(case), flush=True)
        del ranks, vals, keys, K, V, hk, strs, hv
        torch.cuda.empty_cache()
    prof.close()
    sc.close()


if __name__ == "__main__":
    main()
