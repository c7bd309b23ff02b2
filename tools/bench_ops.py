#!/usr/bin/env python
"""bench_ops.py — device-resident timing of every operator on the path at BASELINE.json sizes
(not the bench.py contract; feeds DESIGN.md).  One JSON line per operator."""
import argparse
import json
import sys
import time

import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import vega_b200 as vb
from vega_b200 import _lib as L

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=float, default=1e9)
ap.add_argument("--distinct", type=float, default=1e6)
ap.add_argument("--ops", default="reduce,group,sort,sortkv,join,count")   # also: zipf, zipfgroup, combine, combinezipf,
#                                                                             leftjoin, rightjoin, fulljoin, cogroup, cogroup3,
#                                                                             join3, join3outer
ap.add_argument("--reps", type=int, default=3)
# reduce partitions of join, leftjoin, rightjoin, fulljoin and cogroup; many partitions of a small input (--rows 1.6e6
# gives 2e5 rows per side) time the fixed cost of every partition's plan
ap.add_argument("--join-splits", type=int, default=8)
args = ap.parse_args()
N, D, JR = int(args.rows), int(args.distinct), args.join_splits
sc = vb.Context(0, profile=True)
stream = sc.stream()
PEAK = 3350.0      # GB/s, NVIDIA H100 SXM data sheet (HBM3); the fraction columns are of this peak


def timed(fn, reps):
    fn()  # warm-up
    out = []
    for _ in range(reps):
        torch.cuda.synchronize(); sc.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        st = fn()
        e1.record(stream)
        sc.synchronize(); torch.cuda.synchronize()
        out.append((e0.elapsed_time(e1), st))
    return out


def run_shuffle(agg, rows=None, keys=None, vals=None, M=8, R=8, hint=0, n=None):
    sh = vb.Shuffle(sc, M, R, L.VB_U64, L.VB_U64, agg, hint=hint)
    src = vb.rdd._Col(rows, allow_rows=True) if rows is not None else vb.rdd._Col(keys)
    vcol = vb.rdd._Col(vals) if vals is not None else None
    starts = vb.slice_starts(src.n, M)
    for m in range(M):
        sh.map(m, src, vcol, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    st = sh.stats()
    sh.free()
    return st


def report(name, n_rows, alg_bytes, res, extra=None):
    ms = sorted(r[0] for r in res)[len(res) // 2]
    st = res[-1][1]
    k = {kk: round(v["ms"], 3) for kk, v in st["kernels"].items() if v["launches"]}
    line = {"op": name, "rows": n_rows, "ms": round(ms, 3), "rows_per_s": n_rows / ms * 1e3,
            "alg_GBps": alg_bytes / ms / 1e6, "roofline_frac": alg_bytes / ms / 1e6 / PEAK, "kernel_ms": k,
            "launches": st["kernel_launches"], "table_slots": st["table_slots"], "restarts": st["table_restarts"]}
    if extra:
        line.update(extra)
    print(json.dumps(line), flush=True)


ops = args.ops.split(",")
rows = torch.empty((N, 2), dtype=torch.int64, device="cuda")
sc.gen_pairs(out_rows=rows, first=0, n=N, mode="uniform", n_distinct=D)
if "reduce" in ops:
    report("reduce_by_key(sum)", N, 16.0 * N + 16.0 * D, timed(lambda: run_shuffle(L.VB_AGG_SUM, rows=rows, hint=D), args.reps))
if "count" in ops:
    report("count_by_key", N, 16.0 * N + 16.0 * D, timed(lambda: run_shuffle(L.VB_AGG_COUNT, rows=rows, hint=D), args.reps))
if "group" in ops:
    report("group_by_key", N, 24.0 * N + 16.0 * D, timed(lambda: run_shuffle(L.VB_AGG_GROUP, rows=rows, hint=D), args.reps))
if "sortkv" in ops:
    report("sort_by_key(k,v)", N, 32.0 * N, timed(lambda: run_shuffle(L.VB_AGG_SORT, rows=rows), max(1, args.reps - 1)))
del rows
torch.cuda.empty_cache()
if "zipf" in ops:
    rows = torch.empty((N, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=0, n=N, mode="zipf", n_distinct=D, seed_k=5, zipf_s=1.1)
    report("reduce_by_key(sum) zipf(1.1)", N, 16.0 * N + 16.0 * D, timed(lambda: run_shuffle(L.VB_AGG_SUM, rows=rows), args.reps))
    if "zipfgroup" in ops:
        report("group_by_key zipf(1.1)", N, 24.0 * N + 16.0 * D, timed(lambda: run_shuffle(L.VB_AGG_GROUP, rows=rows), max(1, args.reps - 1)))
    del rows
    torch.cuda.empty_cache()
if "sort" in ops:
    keys = torch.empty(N, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=keys, first=0, n=N, mode="unique", rank_base=3)
    report("sort_by_key(keys only)", N, 16.0 * N, timed(lambda: run_shuffle(L.VB_AGG_SORT, keys=keys), max(1, args.reps - 1)))
    del keys
    torch.cuda.empty_cache()
join_ops = [o for o in ("join", "leftjoin", "rightjoin", "fulljoin", "cogroup", "cogroup3", "join3", "join3outer") if o in ops]
if join_ops:
    # BASELINE config 4, per-GPU share at 8 GPUs: 6.25e7 rows per side, each rank once per side,
    # 1.25e6 shared keys per GPU (1e7 / 8)
    import ctypes
    n_side = int(min(N, 5e8) // 8)
    shared = n_side // 50
    a = torch.empty((n_side, 2), dtype=torch.int64, device="cuda")
    b = torch.empty((n_side, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=a, first=0, n=n_side, mode="unique", rank_base=0)
    sc.gen_pairs(out_rows=b, first=0, n=n_side, mode="unique", rank_base=n_side - shared)

    def cogroup_pair():
        sa = vb.Shuffle(sc, 8, JR, L.VB_U64, L.VB_U64, L.VB_AGG_COGROUP)
        sb = vb.Shuffle(sc, 8, JR, L.VB_U64, L.VB_U64, L.VB_AGG_COGROUP)
        for s_, t in ((sa, a), (sb, b)):
            col = vb.rdd._Col(t, allow_rows=True)
            st = vb.slice_starts(col.n, 8)
            for m in range(8):
                s_.map(m, col, None, int(st[m]), int(st[m + 1]))
            s_.seal()
        return sa, sb

    def pair_stats(sa, sb):
        st = sa.stats()
        stb = sb.stats()
        for kk in st["kernels"]:
            st["kernels"][kk]["ms"] += stb["kernels"][kk]["ms"]; st["kernels"][kk]["launches"] += stb["kernels"][kk]["launches"]
        st["kernel_launches"] += stb["kernel_launches"]
        return st

    def join():
        sa, sb = cogroup_pair()
        tot = 0
        for r in range(JR):
            nn = ctypes.c_uint64()
            L.check(sc._lib.vb_join_size(sa._h, sb._h, r, ctypes.byref(nn)))
            k, v, w = (torch.empty(nn.value, dtype=torch.int64, device="cuda") for _ in range(3))
            p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
            L.check(sc._lib.vb_join(sa._h, sb._h, r, p(k), p(v), p(w), L.VB_DEVICE))
            tot += nn.value
        st = pair_stats(sa, sb)
        st["join_rows"] = tot
        sa.free(); sb.free()
        return st

if "join" in ops:
    res = timed(join, max(1, args.reps - 1))
    assert res[-1][1]["join_rows"] == shared, (res[-1][1]["join_rows"], shared)
    report("join", 2 * n_side, 32.0 * n_side + 24.0 * shared, res, {"join_rows": shared, "reduce_splits": JR})
if "leftjoin" in ops or "rightjoin" in ops or "fulljoin" in ops or "cogroup" in ops or "cogroup3" in ops:
    # Each outer join against the inner join of the same inputs and against the workaround without outer joins:
    # materialising the cogroup of both sides (vb_shuffle_reduce of every partition, device output), which the
    # caller then still has to expand.  All outputs stay on the device.
    from bench import gpu_info
    card = gpu_info(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    dev = lambda n, dt=torch.int64: torch.empty(n, dtype=dt, device="cuda")

    def outer(kind):
        def run():
            sa, sb = cogroup_pair()
            tot = 0
            for r in range(JR):
                nn = ctypes.c_uint64()
                L.check(sc._lib.vb_join_outer_size(sa._h, sb._h, r, kind, ctypes.byref(nn)))
                k, v, w = dev(nn.value), dev(nn.value), dev(nn.value)
                vv, wv = dev(nn.value, torch.uint8), dev(nn.value, torch.uint8)
                L.check(sc._lib.vb_join_outer(sa._h, sb._h, r, kind, p(k), p(v), p(w), p(vv), p(wv), L.VB_DEVICE))
                tot += nn.value
            st = pair_stats(sa, sb)
            st["join_rows"] = tot
            sa.free(); sb.free()
            return st
        return run

    def cogroup_both():
        sa, sb = cogroup_pair()
        for r in range(JR):
            for s_ in (sa, sb):
                nk, nv = ctypes.c_uint64(), ctypes.c_uint64()
                L.check(sc._lib.vb_shuffle_reduce_size(s_._h, r, ctypes.byref(nk), ctypes.byref(nv)))
                k, o, v = dev(nk.value), dev(nk.value + 1), dev(nv.value)
                L.check(sc._lib.vb_shuffle_reduce(s_._h, r, p(k), None, p(o), p(v), L.VB_DEVICE))
        st = pair_stats(sa, sb)
        sa.free(); sb.free()
        return st

    def cogroup():
        # vb_cogroup of every partition: both sides grouped and aligned by key, device output
        sa, sb = cogroup_pair()
        tot = 0
        for r in range(JR):
            nk, nl, nr = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
            L.check(sc._lib.vb_cogroup_size(sa._h, sb._h, r, ctypes.byref(nk), ctypes.byref(nl), ctypes.byref(nr)))
            k, lo, lv, ro, rv = dev(nk.value), dev(nk.value + 1), dev(nl.value), dev(nk.value + 1), dev(nr.value)
            L.check(sc._lib.vb_cogroup(sa._h, sb._h, r, p(k), p(lo), p(lv), p(ro), p(rv), L.VB_DEVICE))
            tot += nk.value
        st = pair_stats(sa, sb)
        st["cogroup_keys"] = tot
        sa.free(); sb.free()
        return st

    med = lambda r: sorted(x[0] for x in r)[len(r) // 2]
    reps = max(1, args.reps - 1)
    outer_ops = (("leftjoin", "left_outer_join", L.VB_JOIN_LEFT, n_side), ("rightjoin", "right_outer_join", L.VB_JOIN_RIGHT, n_side),
                 ("fulljoin", "full_outer_join", L.VB_JOIN_FULL, 2 * n_side - shared))
    r_inner = timed(join, reps) if any(o[0] in ops for o in outer_ops) else None
    r_cog = timed(cogroup_both, reps)
    for op, name, kind, want in outer_ops:
        if op not in ops:
            continue
        res = timed(outer(kind), reps)
        assert res[-1][1]["join_rows"] == want, (res[-1][1]["join_rows"], want)
        extra = {"gpu": card["name"], "power_limit_w": card["power_limit_w"], "join_rows": want, "reduce_splits": JR,
                 "inner_join_ms": round(med(r_inner), 3), "cogroup_both_sides_ms": round(med(r_cog), 3)}
        report(name, 2 * n_side, 32.0 * n_side + 26.0 * want, res, extra)
    if "cogroup" in ops:
        # against cogroup_both (two vb_shuffle_reduce per partition): the grouping alone, without the alignment by key
        res = timed(cogroup, reps)
        want = 2 * n_side - shared
        assert res[-1][1]["cogroup_keys"] == want, (res[-1][1]["cogroup_keys"], want)
        extra = {"gpu": card["name"], "power_limit_w": card["power_limit_w"], "cogroup_keys": want,
                 "cogroup_both_sides_ms": round(med(r_cog), 3)}
        report("cogroup", 2 * n_side, 32.0 * n_side + 24.0 * want, res, extra)
if "cogroup3" in ops or "join3" in ops or "join3outer" in ops:
    # The join shape with a third side that shares the same 2 % of the keys (its other keys are on no other side), 8 -> 8,
    # device outputs.  vb_cogroup_n of 3 sides against the grouping alone (vb_shuffle_reduce of every partition of the 3
    # sides); vb_cogroup_n of 2 sides against vb_cogroup of the same pair; vb_join_n of 3 sides against vb_join of 2.
    from bench import gpu_info
    card = gpu_info(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    dev = lambda n: torch.empty(n, dtype=torch.int64, device="cuda")
    c = torch.empty((n_side, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=c[:shared], first=0, n=shared, mode="unique", rank_base=n_side - shared)
    sc.gen_pairs(out_rows=c[shared:], first=shared, n=n_side - shared, mode="unique", rank_base=2 * n_side - shared)
    torch.cuda.synchronize()

    def sides_of(ts):
        shs = []
        for t in ts:
            s_ = vb.Shuffle(sc, 8, 8, L.VB_U64, L.VB_U64, L.VB_AGG_COGROUP)
            col = vb.rdd._Col(t, allow_rows=True)
            st = vb.slice_starts(col.n, 8)
            for m in range(8):
                s_.map(m, col, None, int(st[m]), int(st[m + 1]))
            s_.seal()
            shs.append(s_)
        return shs

    def finish(shs, **extra):
        st = shs[0].stats()          # kernel times and launches of every side, summed
        for s_ in shs[1:]:
            o = s_.stats()
            for kk in st["kernels"]:
                st["kernels"][kk]["ms"] += o["kernels"][kk]["ms"]; st["kernels"][kk]["launches"] += o["kernels"][kk]["launches"]
            st["kernel_launches"] += o["kernel_launches"]
        st.update(extra)
        for s_ in shs:
            s_.free()
        return st

    def group_only(ts):
        def run():
            shs = sides_of(ts)
            for r in range(8):
                for s_ in shs:
                    nk, nv = ctypes.c_uint64(), ctypes.c_uint64()
                    L.check(sc._lib.vb_shuffle_reduce_size(s_._h, r, ctypes.byref(nk), ctypes.byref(nv)))
                    k, o, v = dev(nk.value), dev(nk.value + 1), dev(nv.value)
                    L.check(sc._lib.vb_shuffle_reduce(s_._h, r, p(k), None, p(o), p(v), L.VB_DEVICE))
            return finish(shs)
        return run

    def cogroup_n(ts):
        def run():
            shs = sides_of(ts)
            n = len(shs)
            arr = (ctypes.c_void_p * n)(*[s_._h.value for s_ in shs])
            tot = 0
            for r in range(8):
                nk, nv = ctypes.c_uint64(), (ctypes.c_uint64 * n)()
                L.check(sc._lib.vb_cogroup_n_size(arr, n, r, ctypes.byref(nk), nv))
                k = dev(nk.value)
                offs = [dev(nk.value + 1) for _ in range(n)]
                vals = [dev(nv[j]) for j in range(n)]
                L.check(sc._lib.vb_cogroup_n(arr, n, r, p(k), (ctypes.c_void_p * n)(*[p(x) for x in offs]),
                                             (ctypes.c_void_p * n)(*[p(x) for x in vals]), L.VB_DEVICE))
                tot += nk.value
            return finish(shs, cogroup_keys=tot)
        return run

    def join_n(ts):
        def run():
            shs = sides_of(ts)
            n = len(shs)
            arr = (ctypes.c_void_p * n)(*[s_._h.value for s_ in shs])
            tot = 0
            for r in range(8):
                nn = ctypes.c_uint64()
                L.check(sc._lib.vb_join_n_size(arr, n, r, ctypes.byref(nn)))
                k, vs = dev(nn.value), [dev(nn.value) for _ in range(n)]
                L.check(sc._lib.vb_join_n(arr, n, r, p(k), (ctypes.c_void_p * n)(*[p(x) for x in vs]), L.VB_DEVICE))
                tot += nn.value
            return finish(shs, join_rows=tot)
        return run

    med = lambda r: sorted(x[0] for x in r)[len(r) // 2]
    info = {"gpu": card["name"], "power_limit_w": card["power_limit_w"]}
    rows3 = 3 * n_side
    if "cogroup3" in ops:
        keys3 = 3 * n_side - 2 * shared
        r_group = timed(group_only([a, b, c]), args.reps)
        res = timed(cogroup_n([a, b, c]), args.reps)
        assert res[-1][1]["cogroup_keys"] == keys3, (res[-1][1]["cogroup_keys"], keys3)
        # algorithmic bytes: the input rows (16 B), then per output key the key and one offset per side, and every value
        report("cogroup_n 3 sides", rows3, 16.0 * rows3 + (8.0 + 3 * 8.0) * keys3 + 8.0 * rows3, res,
               dict(info, cogroup_keys=keys3, group_3_sides_ms=round(med(r_group), 3)))
        keys2 = 2 * n_side - shared
        r_two = timed(cogroup, args.reps)
        res = timed(cogroup_n([a, b]), args.reps)
        assert res[-1][1]["cogroup_keys"] == keys2, (res[-1][1]["cogroup_keys"], keys2)
        report("cogroup_n 2 sides", 2 * n_side, 16.0 * 2 * n_side + (8.0 + 2 * 8.0) * keys2 + 8.0 * 2 * n_side, res,
               dict(info, cogroup_keys=keys2, vb_cogroup_ms=round(med(r_two), 3)))
    if "join3" in ops:
        r_two = timed(join, args.reps)
        res = timed(join_n([a, b, c]), args.reps)
        assert res[-1][1]["join_rows"] == shared, (res[-1][1]["join_rows"], shared)
        report("join_n 3 sides", rows3, 16.0 * rows3 + 8.0 * 4 * shared, res, dict(info, join_rows=shared, vb_join_2_sides_ms=round(med(r_two), 3)))
    if "join3outer" in ops:
        # vb_join_n_outer of the same 3 sides with every side required (the inner join's rows, plus validity) and
        # with side 0 required (a LEFT JOIN b LEFT JOIN c: every key of a once), against vb_join_n of the 3 sides.
        # Written bytes per row: the key, 3 values and 3 validity bytes.
        def join_n_outer(ts, mask):
            def run():
                shs = sides_of(ts)
                n = len(shs)
                arr = (ctypes.c_void_p * n)(*[s_._h.value for s_ in shs])
                tot = 0
                for r in range(8):
                    nn = ctypes.c_uint64()
                    L.check(sc._lib.vb_join_n_outer_size(arr, n, r, mask, ctypes.byref(nn)))
                    k, vs = dev(nn.value), [dev(nn.value) for _ in range(n)]
                    oks = [torch.empty(nn.value, dtype=torch.uint8, device="cuda") for _ in range(n)]
                    L.check(sc._lib.vb_join_n_outer(arr, n, r, mask, p(k), (ctypes.c_void_p * n)(*[p(x) for x in vs]),
                                                    (ctypes.c_void_p * n)(*[p(x) for x in oks]), L.VB_DEVICE))
                    tot += nn.value
                return finish(shs, join_rows=tot)
            return run

        r_inner = timed(join_n([a, b, c]), args.reps)
        for mask, want in ((0b111, shared), (0b001, n_side)):
            res = timed(join_n_outer([a, b, c], mask), args.reps)
            assert res[-1][1]["join_rows"] == want, (res[-1][1]["join_rows"], want)
            written = (8.0 + 3 * 8.0 + 3.0) * want
            report(f"join_n_outer 3 sides required={mask:#05b}", rows3, 16.0 * rows3 + written, res,
                   dict(info, join_rows=want, written_GBps=written / med(res) / 1e6, join_n_3_sides_ms=round(med(r_inner), 3)))
    del c
    torch.cuda.empty_cache()
if "combine" in ops or "combinezipf" in ops:
    # combine_by_key: sum(v0), min(v1), max(v1), mean(v2), count in one shuffle (5 accumulators) against the baseline a
    # user has without it, one single-column shuffle per aggregate (the mean from a sum and the count).  v0 is gen_pairs'
    # value column (< 2^20), v1 = 7 v0 - 3e6 (i64), v2 = v0 / 2 (f64), all on the device.
    from bench import gpu_info
    card = gpu_info(0)
    for zipf in ([False] if "combinezipf" not in ops else [False, True] if "combine" in ops else [True]):
        keys = torch.empty(N, dtype=torch.int64, device="cuda")
        v0 = torch.empty(N, dtype=torch.int64, device="cuda")
        sc.gen_pairs(out_keys=keys, out_vals=v0, first=0, n=N, mode="zipf" if zipf else "uniform", n_distinct=D,
                     seed_k=5 if zipf else 1, zipf_s=1.1 if zipf else 0.0)
        v1 = v0 * 7 - 3_000_000
        v2 = v0.to(torch.float64) * 0.5
        torch.cuda.synchronize()
        K = vb.rdd._Col(keys)
        K.code = L.VB_U64
        cols = (vb.rdd._Col(v0), vb.rdd._Col(v1), vb.rdd._Col(v2))
        cols[0].code = L.VB_U64
        spec = [(L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 1), (L.VB_AGG_MEAN, 2), (L.VB_AGG_COUNT, 0)]
        M, R = 8, 8
        starts = vb.slice_starts(N, M)

        def fused():
            sh = vb.Shuffle(sc, M, R, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, hint=0 if zipf else D, multi=([c.code for c in cols], spec))
            for m in range(M):
                sh.map_cols(m, K, cols, int(starts[m]), int(starts[m + 1]))
            sh.seal()
            st = sh.stats()
            sh.free()
            return st

        singles = [(L.VB_AGG_SUM, cols[0]), (L.VB_AGG_MIN, cols[1]), (L.VB_AGG_MAX, cols[1]), (L.VB_AGG_SUM, cols[2]),
                   (L.VB_AGG_COUNT, None)]

        def per_aggregate():
            tot = None
            for agg, col in singles:
                sh = vb.Shuffle(sc, M, R, L.VB_U64, col.code if col is not None else L.VB_U64, agg, hint=0 if zipf else D)
                for m in range(M):
                    sh.map(m, K, col, int(starts[m]), int(starts[m + 1]))
                sh.seal()
                st = sh.stats()
                sh.free()
                if tot is None:
                    tot = st
                else:
                    for kk in st["kernels"]:
                        tot["kernels"][kk]["ms"] += st["kernels"][kk]["ms"]
                        tot["kernels"][kk]["launches"] += st["kernels"][kk]["launches"]
                    for kk in ("kernel_launches", "table_restarts"):
                        tot[kk] += st[kk]
                    tot["table_slots"] = max(tot["table_slots"], st["table_slots"])
            return tot

        tag = " zipf(1.1)" if zipf else ""
        alg = 8.0 * (1 + 3) * N + 8.0 * (1 + 5) * D
        rf = timed(fused, args.reps)
        rb = timed(per_aggregate, args.reps)
        med = lambda r: sorted(x[0] for x in r)[len(r) // 2]
        extra = {"gpu": card["name"], "power_limit_w": card["power_limit_w"], "aggregates": 5, "accumulators": 5}
        report("combine_by_key 5 aggs" + tag, N, alg, rf, dict(extra, per_aggregate_ms=round(med(rb), 3)))
        report("5 x reduce_by_key" + tag, N, alg, rb, dict(extra, fused_ms=round(med(rf), 3)))
        del keys, v0, v1, v2, K, cols
        torch.cuda.empty_cache()
sc.close()
