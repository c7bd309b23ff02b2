"""repartition(n) = coalesce(n, shuffle = true) on one GPU (DESIGN.md §5.13): the map calls plus the seal of the new path,
device-resident, against (a) the route a user has without it, partition_by_key over (position, item) pairs with the
positions computed on the host, which gives the same multiset per partition, and (b) one device-to-device cudaMemcpy of
the item bytes.

Cases: 2e8 u64 items in 8 maps for R = 8, 64 and 1000, one and two columns; 5e7 byte-string items of 1 to 20 bytes
(uniform lengths) for R = 8 and 1000.  Starts are drawn per map from a fixed seed.  Host clock around map calls + seal
(the seal ends in a device synchronise); (b) is a torch copy followed by a synchronise.  Every shape is run once before
the timed runs, then the new path and (a) alternate, medians of 3.  The equality with (a) is checked at the timed size:
per partition the sorted items (one column), or the item and byte counts (byte strings).  The card's name and power limit
are read in the same process.  Prints one JSON line per case; writes nothing.
    python tools/bench_repartition.py [u64_items=2e8] [byte_items=5e7]
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
from vega_b200.rdd import RepShuffle, StrKeys, _BytesCol, _Col, slice_starts  # noqa: E402

REPS, M = 3, 8


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def dev_col(t):
    c = _Col(t, role="value")
    c.code = L.VB_U64
    return c


def run_new(sc, bounds, starts, R, cols, bcol):
    sh = RepShuffle(sc, M, R, [L.VB_U64] * len(cols), bcol is not None)
    t0 = time.perf_counter()
    for m in range(M):
        sh.map_items(m, starts[m], cols, bcol, bounds[m], bounds[m + 1])
    sh.seal()
    return time.perf_counter() - t0, sh


def run_old(sc, bounds, R, pos, vals):
    vcode = L.VB_BYTES if isinstance(vals, _BytesCol) else L.VB_U64
    sh = vb.Shuffle(sc, M, R, L.VB_U64, vcode, L.VB_AGG_GROUP)
    t0 = time.perf_counter()
    for m in range(M):
        sh.map(m, pos, vals, bounds[m], bounds[m + 1])
    sh.seal()
    return time.perf_counter() - t0, sh


def positions(bounds, starts):
    """Host-computed positions start_m + 1 + i (u64 wrap-around), copied to the device before the timed calls."""
    parts = [(np.arange(1, bounds[m + 1] - bounds[m] + 1, dtype=np.uint64) + np.uint64(starts[m])) for m in range(M)]
    return torch.from_numpy(np.concatenate(parts).view(np.int64)).cuda()


def check_u64(sh_new, sh_old, R):
    for r in range(R):
        n, _ = sh_new.reduce_size(r)
        a = torch.empty(n, dtype=torch.int64, device="cuda")
        sh_new.reduce_device(r, [a])
        nk, nv = sh_old.reduce_size(r)
        b = torch.empty(nv, dtype=torch.int64, device="cuda")
        offs = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
        keys = torch.empty(nk, dtype=torch.int64, device="cuda")
        sh_old.reduce_device(r, out_keys=keys, out_offs=offs, out_vals=b)
        assert n == nv and torch.equal(torch.sort(a).values, torch.sort(b).values), f"partition {r} differs from partition_by_key"


def check_bytes(sh_new, sh_old, R):
    import ctypes
    lib = L.lib()
    for r in range(R):
        n, nb = sh_new.reduce_size(r)
        nk, nv = sh_old.reduce_size(r)
        refs = torch.empty(nv, dtype=torch.int64, device="cuda")
        sh_old.reduce_device(r, out_keys=torch.empty(nk, dtype=torch.int64, device="cuda"),
                             out_offs=torch.empty(nk + 1, dtype=torch.int64, device="cuda"), out_vals=refs)
        tot = ctypes.c_uint64()
        L.check(lib.vb_shuffle_gather_bytes_size(sh_old._h, ctypes.c_void_p(refs.data_ptr()), nv, L.VB_DEVICE, ctypes.byref(tot)))
        assert (n, nb) == (nv, tot.value), f"partition {r}: ({n}, {nb}) items / bytes, partition_by_key ({nv}, {tot.value})"


def memcpy_s(nbytes):
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    dst.copy_(src)
    torch.cuda.synchronize()
    ts = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        dst.copy_(src)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    n_u64 = int(float(sys.argv[1])) if len(sys.argv) > 1 else 200_000_000
    n_b = int(float(sys.argv[2])) if len(sys.argv) > 2 else 50_000_000
    name, limit = card()
    rng = np.random.default_rng(1)
    starts = [int(x) for x in rng.integers(0, 1 << 63, size=M, dtype=np.int64)]
    with vb.Context(0) as sc:
        g = torch.Generator(device="cuda").manual_seed(2)
        bounds = [int(x) for x in slice_starts(n_u64, M)]
        a = torch.randint(-(1 << 62), 1 << 62, (n_u64,), device="cuda", generator=g)
        b = torch.randint(-(1 << 62), 1 << 62, (n_u64,), device="cuda", generator=g)
        pos = dev_col(positions(bounds, starts))
        copy_1 = memcpy_s(8 * n_u64)
        for n_cols in (1, 2):
            cols = [dev_col(a), dev_col(b)][:n_cols]
            for R in (8, 64, 1000):
                new_t, old_t = [], []
                for rep in range(REPS + 1):
                    t, sh = run_new(sc, bounds, starts, R, cols, None)
                    if rep:
                        new_t.append(t)
                    if n_cols == 1:
                        t2, sh2 = run_old(sc, bounds, R, pos, cols[0])
                        if rep:
                            old_t.append(t2)
                        if rep == REPS:
                            check_u64(sh, sh2, R)
                        sh2.free()
                    sh.free()
                res = {"case": f"u64 x{n_cols}", "items": n_u64, "maps": M, "R": R, "new_ms": 1e3 * statistics.median(new_t),
                       "memcpy_ms": 1e3 * n_cols * copy_1, "gpu": name, "power_limit": limit}
                if old_t:
                    res["partition_by_key_ms"] = 1e3 * statistics.median(old_t)
                print(json.dumps(res), flush=True)
        del a, b, pos
        torch.cuda.empty_cache()
        lens = torch.randint(1, 21, (n_b,), device="cuda", generator=g)
        offs = torch.zeros(n_b + 1, dtype=torch.int64, device="cuda")
        offs[1:] = torch.cumsum(lens, 0)
        data = torch.randint(0, 256, (int(offs[-1]),), dtype=torch.uint8, device="cuda", generator=g)
        bcol = _BytesCol(StrKeys(offs, data))
        bounds = [int(x) for x in slice_starts(n_b, M)]
        pos = dev_col(positions(bounds, starts))
        copy_b = memcpy_s(int(offs[-1]))
        for R in (8, 1000):
            new_t, old_t = [], []
            for rep in range(REPS + 1):
                t, sh = run_new(sc, bounds, starts, R, [], bcol)
                t2, sh2 = run_old(sc, bounds, R, pos, bcol)
                if rep:
                    new_t.append(t)
                    old_t.append(t2)
                if rep == REPS:
                    check_bytes(sh, sh2, R)
                sh.free()
                sh2.free()
            print(json.dumps({"case": "bytes 1-20", "items": n_b, "item_bytes": int(offs[-1]), "maps": M, "R": R,
                              "new_ms": 1e3 * statistics.median(new_t), "partition_by_key_ms": 1e3 * statistics.median(old_t),
                              "memcpy_ms": 1e3 * copy_b, "gpu": name, "power_limit": limit}), flush=True)


if __name__ == "__main__":
    main()
