"""group_by_key and join with byte-string values (VB_BYTES) against the same keys with u64 values, and the gather that
turns references back into bytes, against a device-to-device memcpy of the same byte count.

    python tools/bench_bytes_values.py [--rows 50000000] [--distinct 1000000] [--maps 8] [--reduce 8]

One JSON line per value shape (fixed 16 B, uniform 0-64 B, 1 % at 4 KiB and the rest 0-64 B):
  map_ms / seal_ms       vb_shuffle_map_bytes vs vb_shuffle_map_soa over device input, and the seal; median of 3 runs
                         after a warm-up run (wall clock around calls that synchronise); seal_device_ms is the device
                         time of the seal (profiling on), seal_pool_growth_bytes what the seal added to the memory pool
  gather_ms              vb_shuffle_gather_bytes of every reference of the result, device to device (lengths, scan and
                         copy), median of 3; gather_gbps is the algorithmic bytes over that time: per value 8 (reference)
                         + 16 (source offsets) + 8 (length) + 16 (scan) + 8 (output offset) + 8 (reference) + 8 (source
                         offset) read or written by the three passes, plus 2 x the value's bytes
  memcpy_ms              cudaMemcpy device to device of the gathered byte count (torch copy_), the ceiling of the copy
  join_ms                a two-side inner join with byte-string values on both sides (join_size + join + both gathers)
  host_workaround_ms     at 10^7 rows: group row ids on the GPU, copy them out, gather the strings with numpy on the host
The card's name and power limit are read in the same process.  Nothing is written."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vega_b200 as vb  # noqa: E402
from vega_b200 import _lib as L  # noqa: E402

P = lambda t: ctypes.c_void_p(t.data_ptr())


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def lengths(shape, n, gen):
    if shape == "fixed16":
        return torch.full((n,), 16, dtype=torch.int64, device="cuda")
    lens = torch.randint(0, 65, (n,), generator=gen, device="cuda")
    if shape == "tail4k":
        lens[torch.rand(n, generator=gen, device="cuda") < 0.01] = 4096
    return lens


def values(shape, n, gen):
    lens = lengths(shape, n, gen)
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    data = torch.randint(0, 256, (int(offs[-1]),), dtype=torch.uint8, generator=gen, device="cuda")
    return offs, data


def keys_of(sc, n, D, seed):
    k = torch.empty(n, dtype=torch.int64, device="cuda")
    L.check(sc._lib.vb_gen_pairs(sc._h, None, P(k), None, 0, n, L.VB_GEN_UNIFORM, D, 0, seed, 0, 0.0))
    torch.cuda.synchronize()
    return k


def timed(f):
    t = time.perf_counter()
    r = f()
    return (time.perf_counter() - t) * 1e3, r


def group_run(sc, keys, offs, data, M, R, u64):
    """map ms, seal ms, shuffle"""
    lib, n = sc._lib, keys.numel()
    sh = vb.Shuffle(sc, M, R, L.VB_U64, L.VB_U64 if u64 else L.VB_BYTES, L.VB_AGG_GROUP)
    starts = np.linspace(0, n, M + 1).astype(np.int64)
    ids = torch.arange(n, dtype=torch.int64, device="cuda") if u64 else None
    torch.cuda.synchronize()

    def maps():
        for m in range(M):
            a, b = int(starts[m]), int(starts[m + 1])
            kp = ctypes.c_void_p(keys.data_ptr() + 8 * a)
            if u64:
                L.check(lib.vb_shuffle_map_soa(sh._h, m, kp, ctypes.c_void_p(ids.data_ptr() + 8 * a), b - a, L.VB_DEVICE))
            else:
                L.check(lib.vb_shuffle_map_bytes(sh._h, m, kp, ctypes.c_void_p(offs.data_ptr() + 8 * a), P(data), data.numel(),
                                                 b - a, L.VB_DEVICE))
    map_ms, _ = timed(maps)
    reserved0 = sc.mem_info()[0]
    seal_ms, _ = timed(sh.seal)
    sh.seal_dev_ms = sh.stats()["seal_ms"]               # device time of the seal's kernels and copies (profiling on)
    sh.seal_pool_growth = sc.mem_info()[0] - reserved0   # bytes the seal added to the context's pool
    return map_ms, seal_ms, sh


def all_vals(sh, R):
    out = []
    for r in range(R):
        nk, nv = sh.reduce_size(r)
        v = torch.empty(nv, dtype=torch.int64, device="cuda")
        sh.reduce_device(r, out_vals=v)
        out.append(v)
    return torch.cat(out)


def gather(sc, sh, refs):
    lib, n = sc._lib, refs.numel()
    nb = ctypes.c_uint64()
    L.check(lib.vb_shuffle_gather_bytes_size(sh._h, P(refs), n, L.VB_DEVICE, ctypes.byref(nb)))
    go = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    gb = torch.empty(max(nb.value, 1), dtype=torch.uint8, device="cuda")
    ms, _ = timed(lambda: L.check(lib.vb_shuffle_gather_bytes(sh._h, P(refs), n, L.VB_DEVICE, P(go), P(gb), L.VB_DEVICE)))
    return ms, nb.value, go, gb


def memcpy_ms(nbytes):
    a = torch.empty(max(nbytes, 1), dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    b.copy_(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(3):
        e0.record()
        b.copy_(a)
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def join_ms(sc, shape, n, D, R, gen):
    lib = sc._lib
    sides = []
    for s in range(2):
        k = keys_of(sc, n, D, 100 + s)
        o, d = values(shape, n, gen)
        sh = vb.Shuffle(sc, 1, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_COGROUP)
        torch.cuda.synchronize()
        L.check(lib.vb_shuffle_map_bytes(sh._h, 0, P(k), P(o), P(d), d.numel(), n, L.VB_DEVICE))
        sh.seal()
        sides.append(sh)
    torch.cuda.synchronize()
    t = time.perf_counter()
    rows = 0
    for r in range(R):
        nn = ctypes.c_uint64()
        L.check(lib.vb_join_size(sides[0]._h, sides[1]._h, r, ctypes.byref(nn)))
        k, v, w = (torch.empty(nn.value, dtype=torch.int64, device="cuda") for _ in range(3))
        L.check(lib.vb_join(sides[0]._h, sides[1]._h, r, P(k), P(v), P(w), L.VB_DEVICE))
        gather(sc, sides[0], v)
        gather(sc, sides[1], w)
        rows += nn.value
    ms = (time.perf_counter() - t) * 1e3
    for sh in sides:
        sh.free()
    return ms, rows


def host_workaround_ms(sc, shape, n, D, M, R, gen):
    keys = keys_of(sc, n, D, 7)
    offs, data = values(shape, n, gen)
    h_offs, h_data = offs.cpu().numpy(), data.cpu().numpy()
    torch.cuda.synchronize()
    t = time.perf_counter()
    _, _, sh = group_run(sc, keys, offs, data, M, R, True)
    ids = all_vals(sh, R).cpu().numpy()
    starts, lens = h_offs[:-1][ids], np.diff(h_offs)[ids]
    out_off = np.zeros(len(ids) + 1, dtype=np.int64)
    np.cumsum(lens, out=out_off[1:])
    src = np.repeat(starts - out_off[:-1], lens) + np.arange(out_off[-1], dtype=np.int64)
    out = h_data[src]
    ms = (time.perf_counter() - t) * 1e3
    sh.free()
    return ms, int(out.size)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--distinct", type=int, default=1_000_000)
    ap.add_argument("--maps", type=int, default=8)
    ap.add_argument("--reduce", type=int, default=8)
    ap.add_argument("--join-rows", type=int, default=2_000_000)
    ap.add_argument("--host-rows", type=int, default=10_000_000)
    ap.add_argument("--shapes", default="fixed16,uniform64,tail4k")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bytes_values needs a GPU")
    name, limit = card()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    with vb.Context(0) as sc:
        keys = keys_of(sc, a.rows, a.distinct, 1)
        for shape in a.shapes.split(","):
            offs, data = values(shape, a.rows, gen)
            res = {"u64": [], "bytes": [], "gather": []}
            nbytes = 0
            for it in range(4):                       # run 0 warms up
                sc.set_profile(True)
                mu, su, shu = group_run(sc, keys, offs, data, a.maps, a.reduce, True)
                du, gu = shu.seal_dev_ms, shu.seal_pool_growth
                shu.free()
                mb, sb, shb = group_run(sc, keys, offs, data, a.maps, a.reduce, False)
                db, gbw = shb.seal_dev_ms, shb.seal_pool_growth
                sc.set_profile(False)
                refs = all_vals(shb, a.reduce)
                gms, nbytes, go, gb = gather(sc, shb, refs)
                del go, gb, refs
                shb.free()
                if it:
                    res["u64"].append((mu, su, du, gu))
                    res["bytes"].append((mb, sb, db, gbw))
                    res["gather"].append(gms)
            med = lambda xs: float(np.median(xs))
            n = a.rows
            algo = n * 72 + 2 * nbytes
            jm, jrows = join_ms(sc, shape, a.join_rows, a.join_rows, a.reduce, gen)
            hm, hbytes = host_workaround_ms(sc, shape, min(a.host_rows, n), a.distinct, a.maps, a.reduce, gen)
            print(json.dumps({
                "shape": shape, "rows": n, "distinct": a.distinct, "maps": a.maps, "reduce": a.reduce, "value_bytes": nbytes,
                "u64_map_ms": med([x[0] for x in res["u64"]]), "u64_seal_ms": med([x[1] for x in res["u64"]]),
                "bytes_map_ms": med([x[0] for x in res["bytes"]]), "bytes_seal_ms": med([x[1] for x in res["bytes"]]),
                "u64_seal_device_ms": med([x[2] for x in res["u64"]]), "bytes_seal_device_ms": med([x[2] for x in res["bytes"]]),
                "u64_seal_pool_growth_bytes": max(x[3] for x in res["u64"]),
                "bytes_seal_pool_growth_bytes": max(x[3] for x in res["bytes"]),
                "gather_ms": med(res["gather"]), "gather_gbps": algo / med(res["gather"]) / 1e6,
                "memcpy_ms": memcpy_ms(nbytes), "memcpy_gbps": 2 * nbytes / memcpy_ms(nbytes) / 1e6,
                "join_rows_per_side": a.join_rows, "join_out_rows": jrows, "join_ms": jm,
                "host_workaround_rows": min(a.host_rows, n), "host_workaround_ms": hm, "host_workaround_bytes": hbytes,
                "gpu": name, "power_limit": limit}), flush=True)
            del offs, data


if __name__ == "__main__":
    main()
