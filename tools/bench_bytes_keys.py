"""Byte-slice keys against String keys (DESIGN.md §5.14): the same key bytes shuffled with the String placement
(MetroHash64_1(key ‖ 0xFF)) and with the Vec<u8> placement (MetroHash64_1(le64(len) ‖ key)), alternating in one process.

Workloads, 8 map tasks and 8 partitions, keys and values on the device (borrowed):
  words  5e7 rows over about 1e6 distinct words of 1 to 20 bytes (bench_str_blob.py's dictionary), uniform;
  uuid   5e7 rows over 1e6 distinct random 16-byte keys, uniform;
each through reduce_by_key(sum) over u64 values and group_by_key.  A run is host clock from the first map call to the end
of seal (a synchronise).  Medians of 5 runs of each kind after one warm-up of each.  Both kinds must give the same
(key, value) multiset over all partitions: reduce results as sorted (key, sum) pairs, group results as every key's value
list (input order) laid end to end in key order.  The card's name and power limit are read in the same process.  Prints
one JSON line; writes nothing.
    python tools/bench_bytes_keys.py [rows=5e7] [distinct=1e6]
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
from vega_b200 import _lib as L  # noqa: E402
from tools.bench_str_blob import card, dictionary  # noqa: E402

REPS = 5
M = R = 8


def uuid_dictionary(D, seed):
    rng = np.random.default_rng(seed)
    data = rng.integers(0, 256, (D, 16), dtype=np.uint8)
    offs = np.arange(D + 1, dtype=np.int64) * 16
    return torch.from_numpy(offs).cuda(), torch.from_numpy(data.reshape(-1).copy()).cuda()


def rows(doffs, dbytes, n, seed):
    """n keys drawn uniformly from the dictionary, built on the device: (offsets, bytes)."""
    D = doffs.numel() - 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    ranks = torch.randint(0, D, (n,), generator=g, device="cuda")
    lens = doffs[1:][ranks] - doffs[:-1][ranks]
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    total = int(offs[-1])
    row = torch.repeat_interleave(torch.arange(n, device="cuda"), lens, output_size=total)
    j = torch.arange(total, device="cuda") - offs[:-1][row]
    data = dbytes[doffs[:-1][ranks][row] + j]
    del row, j, ranks, lens
    return offs, data


def run(sc, offs, data, vals, kind, op):
    keys = (vb.BytesKeys if kind == L.VB_STRKEY_BYTES else vb.StrKeys)(offs, data)
    rdd = sc.parallelize(keys, M, values=vals)
    s = rdd.group_by_key(R) if op == "group" else rdd.reduce_by_key("sum", R)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sh = s._run()
    torch.cuda.synchronize()
    return sh, time.perf_counter() - t0


def contents(sh, op):
    """The shuffle's (key, value) multiset in a canonical form."""
    keys, parts = [], []
    for r in range(R):
        out = sh.reduce_raw(r)
        ko, kb = out[0].astype(np.int64), out[1].tobytes()
        ks = [kb[ko[i]:ko[i + 1]] for i in range(len(ko) - 1)]
        keys += ks
        if op == "group":
            o, v = out[2].astype(np.int64), out[3]
            parts += [v[o[i]:o[i + 1]] for i in range(len(ks))]
        else:
            parts.append(out[2].view(np.uint64))
    order = sorted(range(len(keys)), key=keys.__getitem__)
    if op == "group":
        return [keys[i] for i in order], np.concatenate([parts[i] for i in order]) if parts else np.empty(0)
    return [keys[i] for i in order], np.concatenate(parts)[np.array(order, dtype=np.int64)]


def main():
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
    D = int(float(sys.argv[2])) if len(sys.argv) > 2 else 1_000_000
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rows": n, "distinct": D, "maps": M, "partitions": R, "runs": REPS}
    vals = torch.from_numpy(np.random.default_rng(5).integers(0, 1 << 62, n, dtype=np.int64)).cuda()
    with vb.Context(0) as sc:
        for wl, dic in (("words", lambda: dictionary(D, np.random.default_rng(11))), ("uuid", lambda: uuid_dictionary(D, 12))):
            doffs, dbytes = dic()
            offs, data = rows(doffs, dbytes, n, 13)
            del doffs, dbytes
            torch.cuda.empty_cache()
            for op in ("reduce", "group"):
                t = {L.VB_STRKEY_STR: [], L.VB_STRKEY_BYTES: []}
                got = {}
                for rep in range(REPS + 1):           # alternated, so both kinds see the same machine state
                    for kind in (L.VB_STRKEY_STR, L.VB_STRKEY_BYTES):
                        sh, dt = run(sc, offs, data, vals, kind, op)
                        if rep:
                            t[kind].append(dt)
                        elif kind not in got:
                            got[kind] = contents(sh, op)
                        sh.free()
                a, b = got[L.VB_STRKEY_STR], got[L.VB_STRKEY_BYTES]
                assert a[0] == b[0] and np.array_equal(a[1], b[1]), f"{wl} {op}: the two kinds give different contents"
                ms = {k: statistics.median(v) * 1e3 for k, v in t.items()}
                spread = {k: (max(v) - min(v)) * 1e3 for k, v in t.items()}
                res[f"{wl}_{op}"] = {"str_ms": round(ms[L.VB_STRKEY_STR], 2), "bytes_ms": round(ms[L.VB_STRKEY_BYTES], 2),
                                     "bytes_over_str": round(ms[L.VB_STRKEY_BYTES] / ms[L.VB_STRKEY_STR], 3),
                                     "str_spread_ms": round(spread[L.VB_STRKEY_STR], 2),
                                     "bytes_spread_ms": round(spread[L.VB_STRKEY_BYTES], 2),
                                     "distinct_keys": len(a[0]), "same_contents": True}
            del offs, data
            torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
