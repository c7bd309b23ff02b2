"""Join and cogroup of String-key shuffles against the same shapes on integer keys (DESIGN.md §5.2).

Two sides of `rows` rows each (default 5e7), word-like keys ('w' + hex digits of a rank, built on the device by
tests/test_gpu_str_keys._device_words), D = 1e6 and 1e7 distinct keys per side, 2 % of the keys on both sides, 8 map
slices -> 8 partitions.  For each D: the median wall time over 3 runs (after a warm-up) of vb_join_n_str (inner) and
vb_cogroup_n_str over every partition with device outputs, and of vb_join_n / vb_cogroup_n on the integer ranks; then
one profiled run on fresh shuffles for the device time per kernel class, with the lazy key-index build on its own.
Last, at 1e7 rows per side, the workaround without string joins: host dictionary encoding of both sides' words and an
integer join.  Prints one JSON line with the card name and power limit read in the same process; writes nothing.
    python tools/bench_str_join.py [rows=5e7]
"""
import ctypes
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
from tests.test_gpu_str_keys import _device_words  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 50_000_000
R = 8
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip(), "rows_per_side": n, "partitions": R}


def arr(shs):
    return (ctypes.c_void_p * len(shs))(*[s._h.value for s in shs])


def dev(k, dtype=torch.int64):
    return torch.empty(k, dtype=dtype, device="cuda")


def p(t):
    return ctypes.c_void_p(t.data_ptr())


def str_join(lib, shs):
    a, m = arr(shs), len(shs)
    nr, nk, nb = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    rows = 0
    for r in range(R):
        L.check(lib.vb_join_n_str_size(a, m, r, (1 << m) - 1, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)))
        ko, kb, ro = dev(nk.value + 1), dev(nb.value, torch.uint8), dev(nk.value + 1)
        vs = [dev(nr.value) for _ in shs]
        L.check(lib.vb_join_n_str(a, m, r, (1 << m) - 1, p(ko), p(kb), p(ro), (ctypes.c_void_p * m)(*[p(v) for v in vs]), None,
                                  L.VB_DEVICE))
        rows += nr.value
    return rows


def str_cogroup(lib, shs):
    a, m = arr(shs), len(shs)
    nk, nb, nv = ctypes.c_uint64(), ctypes.c_uint64(), (ctypes.c_uint64 * m)()
    keys = 0
    for r in range(R):
        L.check(lib.vb_cogroup_n_str_size(a, m, r, ctypes.byref(nk), ctypes.byref(nb), nv))
        ko, kb = dev(nk.value + 1), dev(nb.value, torch.uint8)
        offs, vals = [dev(nk.value + 1) for _ in shs], [dev(nv[j]) for j in range(m)]
        L.check(lib.vb_cogroup_n_str(a, m, r, p(ko), p(kb), (ctypes.c_void_p * m)(*[p(o) for o in offs]),
                                     (ctypes.c_void_p * m)(*[p(v) for v in vals]), L.VB_DEVICE))
        keys += nk.value
    return keys


def int_join(lib, shs):
    a, m = arr(shs), len(shs)
    nr = ctypes.c_uint64()
    rows = 0
    for r in range(R):
        L.check(lib.vb_join_n_size(a, m, r, ctypes.byref(nr)))
        k, vs = dev(nr.value), [dev(nr.value) for _ in shs]
        L.check(lib.vb_join_n(a, m, r, p(k), (ctypes.c_void_p * m)(*[p(v) for v in vs]), L.VB_DEVICE))
        rows += nr.value
    return rows


def int_cogroup(lib, shs):
    a, m = arr(shs), len(shs)
    nk, nv = ctypes.c_uint64(), (ctypes.c_uint64 * m)()
    keys = 0
    for r in range(R):
        L.check(lib.vb_cogroup_n_size(a, m, r, ctypes.byref(nk), nv))
        k = dev(nk.value)
        offs, vals = [dev(nk.value + 1) for _ in shs], [dev(nv[j]) for j in range(m)]
        L.check(lib.vb_cogroup_n(a, m, r, p(k), (ctypes.c_void_p * m)(*[p(o) for o in offs]),
                                 (ctypes.c_void_p * m)(*[p(v) for v in vals]), L.VB_DEVICE))
        keys += nk.value
    return keys


def timed(f, *a):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = f(*a)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, res


def kernels(sh):
    return {k: round(v["ms"], 2) for k, v in sh.stats()["kernels"].items() if v["ms"]}


def inputs(sc, m, D):
    """ranks, values of both sides: side 1's ranks are shifted so that 2 % of the keys are on both sides"""
    sides = []
    for j in range(2):
        r = dev(m)
        v = dev(m)
        sc.gen_pairs(out_keys=r, out_vals=v, n=m, mode="uniform", n_distinct=D, seed_k=1 + j * 1_000_000_007)
        sides.append((torch.remainder(r, D) + j * int(D * 0.98), v))
    torch.cuda.synchronize()
    return sides


with vb.Context(0) as sc:
    lib = sc._lib
    for D in (1_000_000, 10_000_000):
        sides = inputs(sc, n, D)
        words = [_device_words(r) for r, _ in sides]
        torch.cuda.synchronize()
        res = {"key_bytes_per_side": [int(w.data.numel()) for w in words]}
        s_sh = [sc.parallelize(w, 8, values=v).group_by_key(R)._run() for w, (_, v) in zip(words, sides)]
        i_sh = [sc.parallelize(r, 8, values=v).group_by_key(R)._run() for r, v in sides]
        for name, f, shs in [("join_str", str_join, s_sh), ("cogroup_str", str_cogroup, s_sh),
                             ("join_u64", int_join, i_sh), ("cogroup_u64", int_cogroup, i_sh)]:
            f(lib, shs)                                               # warm-up (builds the string key index once)
            runs = [timed(f, lib, shs) for _ in range(3)]
            res[name] = {"median_ms": round(statistics.median(t for t, _ in runs), 2), "out": runs[0][1]}
        for s in s_sh + i_sh:
            s.free()
        # one profiled run on fresh shuffles: device time per kernel class; the index build is the dict class
        sc.set_profile(True)
        for label, f, mk in [("str", (str_join, str_cogroup), lambda w, r, v: sc.parallelize(w, 8, values=v)),
                             ("u64", (int_join, int_cogroup), lambda w, r, v: sc.parallelize(r, 8, values=v))]:
            for g in f:
                shs = [mk(w, r, v).group_by_key(R)._run() for w, (r, v) in zip(words, sides)]
                before = [kernels(s).get("dict", 0.0) for s in shs]
                t, _ = timed(g, lib, shs)
                res[f"profiled_{g.__name__}"] = {
                    "wall_ms": round(t, 2), "side0_kernels_ms": kernels(shs[0]),
                    "index_build_ms": [round(kernels(s).get("dict", 0.0) - b, 2) for s, b in zip(shs, before)] if label == "str" else None}
                for s in shs:
                    s.free()
        sc.set_profile(False)
        out[f"D={D:.0e}"] = res
        del words, sides
        torch.cuda.empty_cache()
    # the workaround without string joins, at 1e7 rows per side: encode both sides' words on the host, join integers
    m = 10_000_000
    sides = inputs(sc, m, 1_000_000)
    strs = [_device_words(r).to_strs().tolist() for r, _ in sides]
    t0 = time.perf_counter()
    d = {}
    ids = [np.fromiter((d.setdefault(w, len(d)) for w in s), dtype=np.uint64, count=m) for s in strs]
    t1 = time.perf_counter()
    i_sh = [sc.parallelize(torch.from_numpy(x.view(np.int64)).cuda(), 8, values=v).group_by_key(R)._run() for x, (_, v) in zip(ids, sides)]
    rows_i = int_join(lib, i_sh)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    words = [_device_words(r) for r, _ in sides]
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    s_sh = [sc.parallelize(w, 8, values=v).group_by_key(R)._run() for w, (_, v) in zip(words, sides)]
    rows_s = str_join(lib, s_sh)
    torch.cuda.synchronize()
    t4 = time.perf_counter()
    assert rows_i == rows_s, (rows_i, rows_s)
    out["workaround_1e7"] = {"host_encode_ms": round((t1 - t0) * 1e3, 1), "int_shuffle_and_join_ms": round((t2 - t1) * 1e3, 1),
                             "str_shuffle_and_join_ms": round((t4 - t3) * 1e3, 1), "rows": rows_s}
print(json.dumps(out))
