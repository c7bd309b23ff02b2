"""group_by_key with byte-string values across W ranks in one process (vb_shuffle_create_bytes_dist and the bytes export /
import calls), the ranks' columns swapped with torch.cat as an all-to-all-v would deliver them.

    python tools/bench_bytes_dist.py [--rows 50000000] [--distinct 1000000] [--maps 8] [--reduce 8] [--worlds 1,2,8]

One JSON line per (value shape, W), the shapes of bench_bytes_values.py (fixed 16 B, uniform 0-64 B, 1 % at 4 KiB and
the rest 0-64 B), keys uniform over --distinct:
  wall_ms          map + export + import + seal, each call timed on the wall clock (they synchronise) and summed over the
                   ranks; the swap between export and import is not included.  Median of 3 runs after a warm-up run.
  map_ms / export_ms / import_ms / seal_ms   each phase alone, summed over the ranks (median of the same runs)
  pack_device_ms   device time of the pack inside the exports (bytes_len_kernel, the scan, bytes_gather_kernel, the u32
                   lengths and the read of the byte counts at the destination cuts), from torch.profiler in a separate
                   run, summed over the ranks
  exported_bytes_per_row  what the exports wrote (keys 8 B + value length 4 B + the value's bytes) over the rows
Cross-GPU exchange time is not measured: every rank runs on the one GPU.  The card's name and power limit are read in
the same process.  Nothing is written."""
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
from vega_b200 import dist as vdist  # noqa: E402

P = lambda t: ctypes.c_void_p(t.data_ptr())
PACK_KERNELS = ("bytes_len_kernel", "scan_reduce_kernel", "scan_apply_kernel", "bytes_gather_kernel", "str_diff_u32_kernel",
                "gather_u64_kernel")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def values(shape, n, gen):
    if shape == "fixed16":
        lens = torch.full((n,), 16, dtype=torch.int64, device="cuda")
    else:
        lens = torch.randint(0, 65, (n,), generator=gen, device="cuda")
        if shape == "tail4k":
            lens[torch.rand(n, generator=gen, device="cuda") < 0.01] = 4096
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    data = torch.randint(0, 256, (int(offs[-1]),), dtype=torch.uint8, generator=gen, device="cuda")
    return offs, data


def swap(exports, W):
    """exports[src] = ((counts, n_val_bytes), (keys, val_lens, val_bytes)) -> per destination the received columns and
    what every source sent, source-rank major."""
    out = []
    for d in range(W):
        cols = []
        for i, vec in ((0, 0), (1, 0), (2, 1)):
            parts = [torch.split(c[i], list(n[vec]))[d] for n, c in exports]
            cols.append(torch.cat(parts))
        out.append((cols, ([n[0][d] for n, _ in exports], [n[1][d] for n, _ in exports])))
    return out


def run(sc, keys, offs, data, W, M, R, profile=None):
    """One shuffle on W ranks -> (wall ms summed over ranks, {phase: ms summed over ranks}, exported bytes)."""
    lib, n = sc._lib, keys.numel()
    starts = np.linspace(0, n, M + 1).astype(np.int64)
    shs = [vb.Shuffle.bytes_dist(sc, M, R, L.VB_U64, L.VB_AGG_GROUP, r, W) for r in range(W)]
    torch.cuda.synchronize()
    t = {"map": 0.0, "export": 0.0, "import": 0.0, "seal": 0.0}

    def timed(k, f):
        t0 = time.perf_counter()
        r = f()
        t[k] += (time.perf_counter() - t0) * 1e3
        return r
    for sh in shs:
        lo, hi = vdist.map_block(sh.rank, W, M)
        for m in range(lo, hi):
            a, b = int(starts[m]), int(starts[m + 1])
            timed("map", lambda: L.check(lib.vb_shuffle_map_bytes(sh._h, m, ctypes.c_void_p(keys.data_ptr() + 8 * a),
                                                                  ctypes.c_void_p(offs.data_ptr() + 8 * a), P(data), data.numel(),
                                                                  b - a, L.VB_DEVICE)))
    exported = 0
    if W > 1:
        if profile is not None:
            profile.start()
        exports = [timed("export", sh.export_bytes) for sh in shs]
        if profile is not None:
            torch.cuda.synchronize()
            profile.stop()
        exported = sum(8 * sum(c[0]) + 4 * sum(c[0]) + sum(c[1]) for c, _ in exports)
        recv = swap(exports, W)
        del exports
        for sh, (cols, counts) in zip(shs, recv):
            timed("import", lambda: sh.import_bytes(*cols, *counts))
        del recv, cols
    for sh in shs:
        timed("seal", sh.seal)
    for sh in shs:
        sh.free()
    return sum(t.values()), t, exported


def pack_ms(sc, keys, offs, data, W, M, R):
    from torch.profiler import ProfilerActivity, profile
    prof = profile(activities=[ProfilerActivity.CUDA])
    run(sc, keys, offs, data, W, M, R, profile=prof)
    total = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and any(k in e.name for k in PACK_KERNELS):
            total += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--distinct", type=int, default=1_000_000)
    ap.add_argument("--maps", type=int, default=8)
    ap.add_argument("--reduce", type=int, default=8)
    ap.add_argument("--worlds", default="1,2,8")
    ap.add_argument("--shapes", default="fixed16,uniform64,tail4k")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bytes_dist needs a GPU")
    name, limit = card()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    with vb.Context(0) as sc:
        keys = torch.empty(a.rows, dtype=torch.int64, device="cuda")
        L.check(sc._lib.vb_gen_pairs(sc._h, None, P(keys), None, 0, a.rows, L.VB_GEN_UNIFORM, a.distinct, 0, 1, 0, 0.0))
        for shape in a.shapes.split(","):
            offs, data = values(shape, a.rows, gen)
            torch.cuda.synchronize()
            for W in [int(w) for w in a.worlds.split(",")]:
                runs = [run(sc, keys, offs, data, W, a.maps, a.reduce) for _ in range(4)][1:]   # run 0 warms up
                phase = lambda k: float(np.median([r[1][k] for r in runs]))
                print(json.dumps({
                    "shape": shape, "rows": a.rows, "distinct": a.distinct, "maps": a.maps, "reduce": a.reduce, "world": W,
                    "value_bytes": data.numel(), "wall_ms": float(np.median([r[0] for r in runs])),
                    **{f"{k}_ms": phase(k) for k in ("map", "export", "import", "seal")},
                    "pack_device_ms": pack_ms(sc, keys, offs, data, W, a.maps, a.reduce) if W > 1 else None,
                    "exported_bytes_per_row": runs[0][2] / a.rows if W > 1 else None,
                    "gpu": name, "power_limit": limit}), flush=True)
            del offs, data


if __name__ == "__main__":
    main()
