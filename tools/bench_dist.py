#!/usr/bin/env python
"""bench_dist.py — the multi-GPU BASELINE.json configs, one rank per GPU under torchrun:

  zipf   configs[4]: reduce_by_key(sum), rows/GPU Zipf(1.1) pairs over 1e6 keys, 8 map partitions/GPU, 8*N reduce
  join   configs[3]: join of two RDDs with unique keys (rows/GPU per side), shared keys = rows/50, N map x 8 reduce... (R = max(8, N))
  group  group_by_key of rows/GPU uniform pairs: raw rows cross NVLink in ONE all-to-all-v (exchange GB/s)
  combine  combine_by_key of rows/GPU uniform rows, tools/bench_ops.py's spec (sum, min, max, mean, count: 5
         accumulators); one row per distinct key and rank crosses NVLink with its 5 partials

Each line: whole-job rows/s (max over ranks), exchange bytes/time, and a size-independent parity property."""
import argparse
import ctypes
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as tdist

import vega_b200 as vb
from vega_b200 import _lib as L
from vega_b200 import dist as vdist

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=float, default=1e9, help="rows per GPU")
ap.add_argument("--distinct", type=float, default=1e6)
ap.add_argument("--ops", default="zipf,join,group")   # + "sort"
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--p2p", action="store_true", help="fused partition+send over peer memory for group/join")
args = ap.parse_args()
rank, world, lrank = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(lrank)
dev = f"cuda:{lrank}"
if world > 1:
    tdist.init_process_group("nccl", device_id=torch.device(dev))
N, D = int(args.rows), int(args.distinct)
sc = vb.Context(lrank, profile=True)
if world > 1:
    sc.comm_init(rank, world)
eng = vdist.CudaEngine(sc)
stream = sc.stream()


def barrier():
    torch.cuda.synchronize(); sc.synchronize()
    if world > 1:
        tdist.barrier()
    torch.cuda.synchronize()


def allmax(x):
    if world == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    tdist.all_reduce(t, op=tdist.ReduceOp.MAX)
    return float(t[0])


def allsum(x):
    if world == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    tdist.all_reduce(t, op=tdist.ReduceOp.SUM)
    return float(t[0])


def shuffle(rows, maps_per_rank, R, agg, stats):
    starts = vb.slice_starts(rows.shape[0], maps_per_rank)
    lo, _ = vdist.map_block(rank, world, maps_per_rank * world)
    maps = [(lo + m, rows[int(starts[m]):int(starts[m + 1])], None) for m in range(maps_per_rank)]
    return vdist.run_shuffle(eng, maps, maps_per_rank * world, R, L.VB_U64, L.VB_U64, agg, rank, world, stats=stats, p2p=args.p2p)


def timed(fn):
    fn()
    best = None
    for _ in range(args.reps):
        barrier()
        t0 = time.perf_counter()
        out = fn()
        barrier()
        dt = allmax(time.perf_counter() - t0)
        if best is None or dt < best[0]:
            best = (dt, out)
    return best


def emit(d):
    if rank == 0:
        print(json.dumps(d), flush=True)


# ---- oracle-sampled parity at full size -------------------------------------------------------------------
# A key-closed sample: every row whose key has its low SAMPLE_BITS bits zero (keys are splitmix64 outputs, so this
# is a uniform ~2^-SAMPLE_BITS sample of the key universe).  Per-key results do not depend on the other keys, so the
# CPU oracle run on just those rows (all ranks' rows gathered on rank 0, in map-id order) must reproduce the GPU
# result restricted to those keys — sums, placement (hash(k) % R), ordered value lists, join rows.
def sample_mask(keys, bits):
    return (keys & ((1 << bits) - 1)) == 0


def gather_sample(rows, bits, cap=4_000_000):
    """This rank's sampled rows (host numpy, input order); None if the sample is too large to ship."""
    m = sample_mask(rows[:, 0], bits)
    n = int(m.sum().item())
    if n > cap:
        return None
    sub = rows[m].cpu().numpy().view(np.uint64)
    return sub


def gather_objs(obj):
    if world == 1:
        return [obj]
    out = [None] * world
    tdist.all_gather_object(out, obj)
    return out


def oracle_sampled_reduce(rows, bits, R, got_parts):
    """got_parts: {r: (keys u64, sums u64)} of the partitions this rank owns (already restricted to the sample).
    Returns (#keys compared, ok) on rank 0, (0, None) elsewhere."""
    subs = gather_objs(gather_sample(rows, bits))
    gots = gather_objs(got_parts)
    if rank != 0:
        return 0, None
    if any(x is None for x in subs):
        return 0, None
    from oracle import oracle as O
    allrows = np.concatenate(subs) if len(subs) else np.zeros((0, 2), np.uint64)
    want = O.shuffle("sum", np.ascontiguousarray(allrows[:, 0]), np.ascontiguousarray(allrows[:, 1]), 8, R, threads=8)
    got = {}
    for g in gots:
        got.update(g)
    n, ok = 0, True
    for r in range(R):
        w = dict(zip(want[r]["keys"].tolist(), want[r]["combined"].tolist()))
        gk, gc = got.get(r, (np.zeros(0, np.uint64), np.zeros(0, np.uint64)))
        g = dict(zip(gk.tolist(), gc.tolist()))
        ok = ok and (g == w)
        n += len(w)
    return n, ok


ops = args.ops.split(",")
if "zipf" in ops:
    rows = torch.empty((N, 2), dtype=torch.int64, device=dev)
    sc.gen_pairs(out_rows=rows, first=rank * N, n=N, mode="zipf", n_distinct=D, seed_k=5, seed_v=2, zipf_s=1.1)
    total_vals = allsum(float(rows[:, 1].sum().item()))
    R = 8 * world

    def run():
        st = {}
        sh = shuffle(rows, 8, R, L.VB_AGG_SUM, st)
        nk, sm = 0, 0
        samp = {}
        for r in vdist.owned_partitions(rank, world, R):
            k, c = sh.reduce(r)
            nk += len(k); sm += int(c.sum(dtype=np.uint64))
            ku = k.view(np.uint64)
            msk = (ku & np.uint64((1 << SB) - 1)) == 0
            samp[r] = (ku[msk].copy(), c.view(np.uint64)[msk].copy())
        sh.free()
        return nk, sm, st, samp

    SB = 10                                     # ~1/1024 of the keys; the Zipf head keys (millions of rows each) are
    while SB < 20 and int(sample_mask(rows[:, 0], SB).sum().item()) > 4_000_000:   # checked via the total-sum property
        SB += 1
    dt, (nk, sm, st, samp) = timed(run)
    keys_total, sum_total = allsum(float(nk)), allsum(float(sm))
    n_cmp, ok = oracle_sampled_reduce(rows, SB, R, samp)
    emit({"op": "reduce_by_key(sum) Zipf(1.1) [configs[4]]", "n_gpus": world, "rows_total": N * world, "partitions": R, "s": dt,
          "rows_per_s": N * world / dt, "distinct_keys_out": int(keys_total), "sum_matches_input": abs(sum_total - total_vals) < 0.5,
          "parity": "oracle-sampled", "parity_keys_compared": n_cmp, "parity_ok": ok, "parity_sample": f"keys with low {SB} bits zero: every row of those keys from all ranks -> oracle/vega_oracle.c on rank 0 -> per-partition (key, sum) dicts must be equal",
          "exchange_ms": st.get("exchange_ms"), "bytes_sent_per_rank": 16 * st.get("sent_rows", 0),
          "note": "time includes the D2H read-back of every owned partition"})
    del rows
    torch.cuda.empty_cache()

if "combine" in ops:
    keys = torch.empty(N, dtype=torch.int64, device=dev)
    v0 = torch.empty(N, dtype=torch.int64, device=dev)
    sc.gen_pairs(out_keys=keys, out_vals=v0, first=rank * N, n=N, mode="uniform", n_distinct=D)
    v1 = v0 * 7 - 3_000_000
    v2 = v0.to(torch.float64) * 0.5
    torch.cuda.synchronize()
    spec = ([L.VB_U64, L.VB_I64, L.VB_F64],
            [(L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MAX, 1), (L.VB_AGG_MEAN, 2), (L.VB_AGG_COUNT, 0)])
    ceng = vdist.CombineCudaEngine(sc)
    R = 8 * world
    starts = vb.slice_starts(N, 8)
    lo, _ = vdist.map_block(rank, world, 8 * world)

    def col(t, code):
        c = vb.rdd._Col(t)
        c.code = code
        return c
    maps = [(lo + m, col(keys[int(starts[m]):int(starts[m + 1])], L.VB_U64),
             tuple(col(t[int(starts[m]):int(starts[m + 1])], code) for t, code in ((v0, L.VB_U64), (v1, L.VB_I64), (v2, L.VB_F64))))
            for m in range(8)]

    def run():
        st = {}
        sh = vdist.run_combine_shuffle(ceng, maps, 8 * world, R, L.VB_U64, spec, rank, world, hint=D, stats=st)
        nk = cnt = 0
        for r in vdist.owned_partitions(rank, world, R):
            k, outs = sh.reduce_cols(r, [np.uint64, np.int64, np.int64, np.float64, np.uint64])
            nk += len(k)
            cnt += int(outs[4].sum(dtype=np.uint64))
        sh.free()
        return nk, cnt, st

    dt, (nk, cnt, st) = timed(run)
    emit({"op": "combine_by_key 5 aggs", "n_gpus": world, "rows_total": N * world, "partitions": R, "s": dt,
          "rows_per_s": N * world / dt, "distinct_keys_out": int(allsum(float(nk))),
          "counts_match_input": int(allsum(float(cnt))) == N * world, "exchange_ms": st.get("exchange_ms"),
          "sent_rows": st.get("sent_rows"), "bytes_sent_per_rank": 48 * st.get("sent_rows", 0),
          "note": "a sent row is the key and 5 partials (48 B); time includes the D2H read-back of every owned partition"})
    del keys, v0, v1, v2, maps
    torch.cuda.empty_cache()

if "group" in ops:
    n = N // 2            # raw rows cross the fabric and are sorted: keep 2 row buffers + sort scratch within HBM
    rows = torch.empty((n, 2), dtype=torch.int64, device=dev)
    sc.gen_pairs(out_rows=rows, first=rank * n, n=n, mode="uniform", n_distinct=D, seed_k=1, seed_v=2)
    R = max(8, world)

    def run():
        st = {}
        sh = shuffle(rows, 8, R, L.VB_AGG_GROUP, st)
        nk = nv = 0
        for r in vdist.owned_partitions(rank, world, R):
            a, b = sh.reduce_size(r)
            nk += a; nv += b
        sh.free()
        return nk, nv, st

    dt, (nk, nv, st) = timed(run)
    sent = 16 * st.get("sent_rows", 0)
    xms = st.get("exchange_ms") or 0.0
    emit({"op": "group_by_key uniform" + (" [p2p fused exchange]" if args.p2p else " [NCCL all-to-all-v]"), "n_gpus": world, "rows_total": n * world, "partitions": R, "s": dt, "rows_per_s": n * world / dt,
          "groups_out": int(allsum(float(nk))), "values_out": int(allsum(float(nv))), "values_match_input": int(allsum(float(nv))) == n * world,
          "exchange_ms": xms, "bytes_sent_per_rank": sent,
          "nvlink_all_to_all_GBps_per_rank": (sent / (xms * 1e-3) / 1e9) if xms else None})
    del rows
    torch.cuda.empty_cache()

if "join" in ops:
    n = int(min(N, 5e8 / max(world, 1))) if world > 1 else int(min(N, 6.25e7))
    shared_total = (n * world) // 50
    a = torch.empty((n, 2), dtype=torch.int64, device=dev)
    b = torch.empty((n, 2), dtype=torch.int64, device=dev)
    sc.gen_pairs(out_rows=a, first=rank * n, n=n, mode="unique", rank_base=0)
    sc.gen_pairs(out_rows=b, first=rank * n, n=n, mode="unique", rank_base=n * world - shared_total)
    R = max(8, world)

    def run():
        st = {}
        sa = shuffle(a, 1, R, L.VB_AGG_COGROUP, st)
        sb = shuffle(b, 1, R, L.VB_AGG_COGROUP, st)
        tot = 0
        samp = {}
        for r in vdist.owned_partitions(rank, world, R):
            nn = ctypes.c_uint64()
            L.check(sc._lib.vb_join_size(sa._h, sb._h, r, ctypes.byref(nn)))
            k, v, w = (torch.empty(nn.value, dtype=torch.int64, device=dev) for _ in range(3))
            p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
            L.check(sc._lib.vb_join(sa._h, sb._h, r, p(k), p(v), p(w), L.VB_DEVICE))
            tot += nn.value
            msk = sample_mask(k, JB)
            samp[r] = tuple(x[msk].cpu().numpy().view(np.uint64) for x in (k, v, w))
        sa.free(); sb.free()
        return tot, st, samp

    JB = 6                                       # 1/64 of the keys of both sides
    while JB < 20 and int(sample_mask(a[:, 0], JB).sum().item()) > 2_000_000:
        JB += 1
    dt, (tot, st, samp) = timed(run)
    out_rows = int(allsum(float(tot)))
    sent = 16 * st.get("sent_rows", 0)
    # oracle-sampled parity: the sampled rows of both sides from every rank -> O.join on rank 0 -> every (k, v, w) row
    sa_, sb_ = gather_objs(gather_sample(a, JB)), gather_objs(gather_sample(b, JB))
    gots = gather_objs(samp)
    n_cmp, ok = 0, None
    if rank == 0 and all(x is not None for x in sa_ + sb_):
        from oracle import oracle as O
        fa, fb = np.concatenate(sa_), np.concatenate(sb_)
        want = O.join(np.ascontiguousarray(fa[:, 0]), np.ascontiguousarray(fa[:, 1]), world, np.ascontiguousarray(fb[:, 0]),
                      np.ascontiguousarray(fb[:, 1]), world, R, threads=8)
        got = {}
        for g in gots:
            got.update(g)
        ok = True
        for r in range(R):
            g = got.get(r, (np.zeros(0, np.uint64),) * 3)
            ok = ok and sorted(zip(*[x.tolist() for x in g])) == sorted(zip(*[x.tolist() for x in want[r]]))
            n_cmp += len(want[r][0])
    emit({"op": "join unique keys [configs[3]]" + (" [p2p]" if args.p2p else " [NCCL]"), "n_gpus": world, "rows_per_side_total": n * world, "partitions": R, "s": dt,
          "input_rows_per_s": 2 * n * world / dt, "join_rows": out_rows, "join_rows_expected": shared_total,
          "parity": "oracle-sampled", "parity_rows_compared": n_cmp, "parity_ok": ok, "parity_sample": f"keys with low {JB} bits zero on both sides: all their rows -> oracle join on rank 0 -> every (k,v,w) output row per reduce partition must be equal",
          "exchange_ms_both_sides": st.get("exchange_ms"), "bytes_sent_per_rank_last_side": sent})
if "sort" in ops:
    # sort_by_key of N u64 keys per GPU (absent from the reference: F2), R = 8 partitions per GPU; property checks:
    # every owned partition ascending, partition ranges ordered across ranks, total row count preserved
    n = N
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    sc.gen_pairs(out_keys=keys, first=rank * n, n=n, mode="unique", rank_base=3)
    R = 8 * world

    def run_sort():
        st = {}
        starts = vb.slice_starts(n, 8)
        lo, _ = vdist.map_block(rank, world, 8 * world)
        maps = [(lo + m, keys[int(starts[m]):int(starts[m + 1])], None) for m in range(8)]
        sh = vdist.run_shuffle(eng, maps, 8 * world, R, L.VB_U64, L.VB_U64, L.VB_AGG_SORT, rank, world, stats=st)
        sh.has_payload = False
        return sh, st

    def run():                                   # timed: map tasks + local sort + exact cuts + exchange + owner re-sort (sealed result in HBM)
        sh, st = run_sort()
        sh.free()
        return st

    dt, st = timed(run)
    # property checks on one more (untimed) run
    sh, _ = run_sort()
    tot, ok, lo_k, hi_k = 0, True, [], []
    for r in vdist.owned_partitions(rank, world, R):
        nk, _ = sh.reduce_size(r)
        tot += nk
        if nk:
            out = torch.empty(nk, dtype=torch.int64, device=dev)
            sh.reduce_device(r, out_keys=out)
            sgn = out ^ torch.tensor(-(1 << 63), dtype=torch.int64, device=dev)      # unsigned order through the sign-flipped view
            ok = ok and bool((sgn[1:] >= sgn[:-1]).all().item())
            lo_k.append((r, int(sgn[0].item()))); hi_k.append((r, int(sgn[-1].item())))
            del out, sgn
    sh.free()
    alls = gather_objs((lo_k, hi_k))
    ranges_ok = None
    if rank == 0:
        lo_all = dict(x for a, _ in alls for x in a); hi_all = dict(x for _, b in alls for x in b)
        parts = sorted(lo_all)
        ranges_ok = all(hi_all[parts[i]] <= lo_all[parts[i + 1]] for i in range(len(parts) - 1))
    emit({"op": "sort_by_key u64 keys (multi-rank: local sort, exact cut keys, one grouped send/recv, owner re-sort; checks outside the timed region)", "n_gpus": world,
          "rows_total": n * world, "partitions": R, "s": dt, "rows_per_s": n * world / dt, "rows_out": int(allsum(float(tot))),
          "rows_match_input": int(allsum(float(tot))) == n * world, "partitions_sorted": bool(allsum(float(ok)) == world),
          "partition_ranges_ordered": ranges_ok, "exchange_ms": st.get("exchange_ms"), "bytes_sent_per_rank": 8 * st.get("sent_rows", 0)})
    del keys
    torch.cuda.empty_cache()
sc.close()
if world > 1:
    tdist.destroy_process_group()
