"""N>1 path on the GPU: two ranks (three in one fused-exchange case) run the real CudaEngine (export multisplit by
destination rank, import, seal) and must reproduce the single-process oracle.  With >= 2 GPUs the exchange is the
library's own (vb_ctx_comm_init + vb_shuffle_exchange: NCCL grouped send/recv or the fused P2P scatter,
one rank per GPU); on a 1-GPU box both ranks share GPU 0 (NCCL refuses duplicate devices) and the
all-to-all-v is staged through gloo — the pack/unpack/seal code under test is the same."""
import os
import pickle
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_ROWS, N_KEYS = 200_000, 30_000


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dataset(values="u64"):
    """values: "u64" (below 2^40), or a full-range set: "u64_full" (per-key sums wrap), "i64_full", "f64_special"
    (NaNs of both signs, +-0.0, +-inf, subnormals; see tests/util.py:rand_pairs)."""
    rng = np.random.default_rng(2024)
    if values != "u64":
        from tests.util import rand_pairs
        vdt, mode = values.split("_")
        return rand_pairs(rng, N_ROWS, N_KEYS, vdt, values=mode)
    keys = rng.integers(0, N_KEYS, N_ROWS).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(7)
    vals = rng.integers(0, 1 << 40, N_ROWS).astype(np.uint64)
    return keys, vals


VCODE = {"u64": 0, "i64": 1, "f64": 2}


def _worker(rank, world, port, agg, M, R, nccl, outdir, p2p=False, values="u64"):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if nccl else 0
    torch.cuda.set_device(dev)
    if nccl:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{dev}"))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    import vega_b200 as vb
    from vega_b200 import dist as vdist
    keys, vals = _dataset(values)
    starts = vb.slice_starts(N_ROWS, M)
    lo, hi = vdist.map_block(rank, world, M)
    sc = vb.Context(dev)
    if nccl:
        sc.comm_init(rank, world)      # >= 2 GPUs: the exchange runs inside libvega_b200 (vb_shuffle_exchange)
    eng = vdist.CudaEngine(sc)
    maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
    stats = {}
    sh = vdist.run_shuffle(eng, maps, M, R, 0, VCODE[values.split("_")[0]], agg, rank, world, stats=stats,
                           exchange_device=None if nccl else "cpu", p2p=p2p)
    if p2p and agg == 0:
        assert stats.get("exchange_kind") == "p2p"
        # a second shuffle through the same (cached) arena and peer mappings
        sh.free()
        stats = {}
        sh = vdist.run_shuffle(eng, maps, M, R, 0, 0, agg, rank, world, stats=stats, p2p=True)
    res = {}
    for r in range(R):
        out = sh.reduce(r)
        if r % world != rank:
            assert len(out[0]) == 0
        res[r] = [np.asarray(x) for x in out]
    with open(os.path.join(outdir, f"r{rank}.pkl"), "wb") as f:
        pickle.dump((res, stats), f)
    sh.free()
    sc.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("agg,M,R,p2p", [(1, 4, 4, False), (0, 4, 6, False), (4, 6, 3, False), (2, 2, 8, False), (0, 5, 2, False),
                                         (0, 4, 6, True), (0, 3, 2, True)])
def test_two_rank_cuda_shuffle_matches_oracle(agg, M, R, p2p):
    """p2p=True: the fused exchange — rows are stored by the partition kernel directly into the other rank's
    arena through a CUDA IPC mapping (same GPU on a 1-GPU box, NVLink peer on a multi-GPU box)."""
    from oracle import oracle as O
    world = 2
    nccl = torch.cuda.device_count() >= 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), agg, M, R, nccl, d, p2p), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, vals = _dataset()
    op = {0: "group", 1: "sum", 2: "min", 3: "max", 4: "count"}[agg]
    want = O.shuffle(op, keys, vals, M, R)
    for r in range(R):
        got = per_rank[r % world][0][r]
        w = want[r]
        if op == "group":
            gd = {int(k): got[2][int(got[1][i]):int(got[1][i + 1])].tolist() for i, k in enumerate(got[0])}
            wd = {int(k): w["vals"][int(w["offsets"][i]):int(w["offsets"][i + 1])].tolist() for i, k in enumerate(w["keys"])}
            assert gd == wd
        else:
            assert dict(zip(got[0].tolist(), got[1].tolist())) == dict(zip(w["keys"].tolist(), w["combined"].tolist()))
    assert sum(s["sent_rows"] for _, s in per_rank) == sum(s["recv_rows"] for _, s in per_rank) > 0


def test_three_rank_p2p_group_matches_oracle():
    """The fused exchange with two foreign sources per destination: every rank writes its block at its own offset
    (source-rank major) into the arena of each of the other two.  One rank per GPU with >= 3 GPUs, else all on GPU 0."""
    from oracle import oracle as O
    world, M, R = 3, 5, 7
    nccl = torch.cuda.device_count() >= world
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), 0, M, R, nccl, d, True), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, vals = _dataset()
    want = O.shuffle("group", keys, vals, M, R)
    for r in range(R):
        got, w = per_rank[r % world][0][r], want[r]
        gd = {int(k): got[2][int(got[1][i]):int(got[1][i + 1])].tolist() for i, k in enumerate(got[0])}
        wd = {int(k): w["vals"][int(w["offsets"][i]):int(w["offsets"][i + 1])].tolist() for i, k in enumerate(w["keys"])}
        assert gd == wd, f"partition {r}"
    assert all(s["exchange_kind"] == "p2p" for _, s in per_rank)
    assert sum(s["sent_rows"] for _, s in per_rank) == sum(s["recv_rows"] for _, s in per_rank) > 0


@pytest.mark.parametrize("agg,values", [(2, "i64_full"), (3, "i64_full"), (2, "f64_special"), (3, "f64_special"),
                                         (1, "u64_full")])
def test_two_rank_reduce_value_dtypes_match_oracle(agg, values):
    """MIN/MAX across ranks: the export packs order-transformed accumulators and the import merges them untransformed;
    the result must still be signed / f64::min-max order (NaN ignored, -0.0 < +0.0).  u64 SUM with wrapping sums."""
    from oracle import oracle as O
    from tests.util import bits_dict
    world, M, R = 2, 4, 5
    nccl = torch.cuda.device_count() >= 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, _free_port(), agg, M, R, nccl, d, False, values), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"r{r}.pkl"), "rb")) for r in range(world)]
    keys, vals = _dataset(values)
    op = {1: "sum", 2: "min", 3: "max"}[agg]
    want = O.shuffle(op, keys, vals, M, R, vdtype=values.split("_")[0])
    for r in range(R):
        got = per_rank[r % world][0][r]
        assert bits_dict(got[0], got[1]) == bits_dict(want[r]["keys"], want[r]["combined"]), f"partition {r}"
    assert sum(s["sent_rows"] for _, s in per_rank) == sum(s["recv_rows"] for _, s in per_rank) > 0


# ---------------------------------------------------------------------------------------------
# multi-rank join / cogroup (CoGroupedRdd::compute co_grouped_rdd.rs:206-249 + pair_rdd.rs:104-121)
# ---------------------------------------------------------------------------------------------
def _join_dataset():
    rng = np.random.default_rng(77)
    ka = rng.integers(0, 4000, 60_000).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)
    kb = rng.integers(2000, 7000, 45_000).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)
    va = rng.integers(0, 1 << 50, len(ka)).astype(np.uint64)
    vb_ = rng.integers(0, 1 << 50, len(kb)).astype(np.uint64)
    return ka, va, kb, vb_


def _join_worker(rank, world, port, Ma, Mb, R, nccl, outdir, p2p):
    import ctypes
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if nccl else 0
    torch.cuda.set_device(dev)
    if nccl:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{dev}"))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    import vega_b200 as vb
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    ka, va, kb, vb_ = _join_dataset()
    sc = vb.Context(dev)
    if nccl:
        sc.comm_init(rank, world)
    eng = vdist.CudaEngine(sc)
    shs = []
    for keys, vals, M in ((ka, va, Ma), (kb, vb_, Mb)):
        starts = vb.slice_starts(len(keys), M)
        lo, hi = vdist.map_block(rank, world, M)
        maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
        shs.append(vdist.run_shuffle(eng, maps, M, R, 0, 0, L.VB_AGG_COGROUP, rank, world,
                                     exchange_device=None if (nccl or p2p) else "cpu", p2p=p2p))
    sa, sb = shs
    res, cg = {}, {}
    for r in range(R):
        n = ctypes.c_uint64()
        L.check(sc._lib.vb_join_size(sa._h, sb._h, r, ctypes.byref(n)))
        k, v, w = (np.empty(n.value, dtype=np.uint64) for _ in range(3))
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
        L.check(sc._lib.vb_join(sa._h, sb._h, r, p(k), p(v), p(w), L.VB_HOST))
        if r % world != rank:
            assert n.value == 0
        res[r] = (k, v, w)
        cg[r] = ([np.asarray(x) for x in sa.reduce(r)], [np.asarray(x) for x in sb.reduce(r)])   # the cogroup sides
    with open(os.path.join(outdir, f"j{rank}.pkl"), "wb") as f:
        pickle.dump((res, cg), f)
    sa.free(); sb.free()
    sc.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("Ma,Mb,R,p2p", [(4, 2, 4, False), (3, 5, 6, True), (2, 2, 3, False)])
def test_two_rank_join_and_cogroup_match_oracle(Ma, Mb, R, p2p):
    """Full oracle diff of a 2-rank join (every output row, per reduce partition) and of both cogroup sides
    (ordered value lists per key), over the NCCL / gloo-staged all-to-all-v and the fused P2P exchange."""
    from oracle import oracle as O
    world = 2
    nccl = torch.cuda.device_count() >= 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_join_worker, args=(world, _free_port(), Ma, Mb, R, nccl, d, p2p), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"j{r}.pkl"), "rb")) for r in range(world)]
    ka, va, kb, vb_ = _join_dataset()
    want = O.join(ka, va, Ma, kb, vb_, Mb, R)
    wa, wb = O.shuffle("group", ka, va, Ma, R), O.shuffle("group", kb, vb_, Mb, R)
    total = 0
    for r in range(R):
        got = per_rank[r % world][0][r]
        assert sorted(zip(*[x.tolist() for x in got])) == sorted(zip(*[x.tolist() for x in want[r]])), f"join partition {r}"
        total += len(got[0])
        for side, w in ((0, wa[r]), (1, wb[r])):
            g = per_rank[r % world][1][r][side]
            gd = {int(k): g[2][int(g[1][i]):int(g[1][i + 1])].tolist() for i, k in enumerate(g[0])}
            wd = {int(k): w["vals"][int(w["offsets"][i]):int(w["offsets"][i + 1])].tolist() for i, k in enumerate(w["keys"])}
            assert gd == wd, f"cogroup side {side} partition {r}"
    assert total == sum(len(w[0]) for w in want) > 0


# ---------------------------------------------------------------------------------------------
# multi-rank sort_by_key (absent from the reference, SURVEY.md F2: parity against the oracle's stable sort)
# ---------------------------------------------------------------------------------------------
def _sort_dataset(kdtype):
    rng = np.random.default_rng(5)
    if kdtype == "tiny":          # 3 rows, more partitions than rows: one rank holds a single row, most partitions are empty
        return np.array([7, 7, 2], dtype=np.uint64), np.arange(3, dtype=np.uint64)
    n = 150_000
    if kdtype == "u64":
        keys = rng.integers(0, 3000, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)     # many duplicates
    elif kdtype == "i64":
        keys = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
    else:
        keys = rng.standard_normal(n)
    vals = np.arange(n, dtype=np.uint64)          # payload = input position: checks stability
    return keys, vals


def _sort_worker(rank, world, port, kdtype, M, R, payload, outdir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    import vega_b200 as vb
    from vega_b200 import _lib as L
    from vega_b200 import dist as vdist
    keys, vals = _sort_dataset(kdtype)
    sc = vb.Context(rank)
    sc.comm_init(rank, world)
    eng = vdist.CudaEngine(sc)
    starts = vb.slice_starts(len(keys), M)
    lo, hi = vdist.map_block(rank, world, M)
    maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]] if payload else None) for m in range(lo, hi)]
    kcode = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64, "tiny": L.VB_U64}[kdtype]
    sh = vdist.run_shuffle(eng, maps, M, R, kcode, L.VB_U64, L.VB_AGG_SORT, rank, world)
    sh.has_payload = payload
    res = {r: [None if x is None else np.asarray(x) for x in sh.reduce(r)] for r in range(R)}
    with open(os.path.join(outdir, f"s{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    sh.free()
    sc.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("kdtype,M,R,payload", [("u64", 4, 4, True), ("i64", 5, 6, True), ("f64", 2, 3, False), ("u64", 3, 2, False),
                                               ("tiny", 2, 5, True)])
def test_two_rank_sort_by_key_matches_oracle(kdtype, M, R, payload):
    if torch.cuda.device_count() < 2:
        pytest.skip("multi-rank sort_by_key runs through the library's NCCL communicator: needs >= 2 GPUs")
    from oracle import oracle as O
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_sort_worker, args=(world, _free_port(), kdtype, M, R, payload, d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"s{r}.pkl"), "rb")) for r in range(world)]
    keys, vals = _sort_dataset(kdtype)
    ok, ov, ps = O.sort_by_key(keys, vals if payload else None, R, "u64" if kdtype == "tiny" else kdtype)
    for r in range(R):
        gk, gv = per_rank[r % world][r]
        a, b = int(ps[r]), int(ps[r + 1])
        assert np.array_equal(gk.view(np.uint64), ok[a:b].view(np.uint64)), f"partition {r} keys"
        if payload:
            assert np.array_equal(gv.view(np.uint64), ov[a:b]), f"partition {r} payload (stability)"
        other = per_rank[(r + 1) % world][r]
        assert len(other[0]) == 0
