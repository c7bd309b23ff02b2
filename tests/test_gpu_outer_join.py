"""GPU outer joins (vb_join_outer, PairRdd.left_outer_join / right_outer_join / full_outer_join) against the reference
definitions in tests/outer_join_ref.py.  Every output row is checked per reduce partition: its value, its validity
bytes, that a key's rows are contiguous, and that they come in the nesting order (for v in vs { for w in ws })."""
import ctypes
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import vega_b200 as vb
from oracle import oracle as O
from tests import outer_join_ref as OJ
from tests.util import assert_parts_equal, rand_pairs
from vega_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["left", "right", "full"]
CODE = {"left": L.VB_JOIN_LEFT, "right": L.VB_JOIN_RIGHT, "full": L.VB_JOIN_FULL}
METHOD = {k: f"{k}_outer_join" for k in KINDS}


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def _u64(x):
    x = np.ascontiguousarray(x)
    return x.view(np.uint64) if x.dtype.itemsize == 8 else x.astype(np.int64).view(np.uint64)


def _side(x, nullable):
    """(u64 bits, validity) of one output side; a side that can be None is a MaskedArray whose None slots hold 0."""
    if nullable:
        assert isinstance(x, np.ma.MaskedArray)
        data, valid = _u64(np.ma.getdata(x)), ~np.ma.getmaskarray(x)
        assert (data[~valid] == 0).all(), "a None slot does not hold 0"
    else:
        assert not isinstance(x, np.ma.MaskedArray)
        data, valid = _u64(x), np.ones(len(x), dtype=bool)
    return data, valid.astype(np.uint8)


def by_key(k, v, w, vv, wv):
    """{key: [(v, w, v_valid, w_valid), ...]} in output order; a key's rows must be contiguous."""
    d, prev = {}, None
    for row in zip(_u64(k).tolist(), _u64(v).tolist(), _u64(w).tolist(), np.asarray(vv).tolist(), np.asarray(wv).tolist()):
        if row[0] != prev:
            assert row[0] not in d, f"the rows of key {row[0]:#x} are not contiguous"
            d[row[0]], prev = [], row[0]
        d[row[0]].append(row[1:])
    return d


def gpu_parts(j):
    """Per-partition by_key dicts of a JoinedRdd with an outer kind."""
    out = []
    for r in range(j.num_slices):
        k, v, w = j.compute(r)
        (vd, vv), (wd, wv) = _side(v, j.kind != "left"), _side(w, j.kind != "right")
        out.append(by_key(k, vd, wd, vv, wv))
    return out


def check(sc, kind, ka, va, Ma, kb, vb_, Mb, R, key_width=8):
    a, b = sc.parallelize((ka, va), Ma), sc.parallelize((kb, vb_), Mb)
    got = gpu_parts(getattr(a, METHOD[kind])(b, R))
    want = OJ.outer_join_parts(kind, ka, va, Ma, kb, vb_, Mb, R, key_width=key_width)
    assert_parts_equal(got, want)
    return got


def abi_rows(sc, sa, sb, r, kind, dst=L.VB_HOST):
    """One partition through the C ABI: (k, v, w, v_valid, w_valid) as host arrays; kind None is vb_join."""
    lib = sc._lib
    n = ctypes.c_uint64()
    if kind is None:
        L.check(lib.vb_join_size(sa._h, sb._h, r, ctypes.byref(n)))
    else:
        L.check(lib.vb_join_outer_size(sa._h, sb._h, r, CODE[kind], ctypes.byref(n)))
    n = n.value
    if dst == L.VB_HOST:
        bufs = [np.zeros(n, dtype=np.uint64) for _ in range(3)] + [np.full(n, 7, dtype=np.uint8) for _ in range(2)]
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    else:
        import torch
        bufs = [torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(3)] + \
               [torch.full((n,), 7, dtype=torch.uint8, device="cuda") for _ in range(2)]
        p = lambda x: ctypes.c_void_p(x.data_ptr()) if x.numel() else None
        torch.cuda.synchronize()
    if kind is None:
        L.check(lib.vb_join(sa._h, sb._h, r, p(bufs[0]), p(bufs[1]), p(bufs[2]), dst))
        bufs[3][:], bufs[4][:] = 1, 1
    else:
        L.check(lib.vb_join_outer(sa._h, sb._h, r, CODE[kind], *[p(x) for x in bufs], dst))
    if dst != L.VB_HOST:
        bufs = [x.cpu().numpy() for x in bufs]
    return tuple(bufs)


def _pair(sc, ka, va, Ma, kb, vb_, Mb, R):
    """Two sealed COGROUP shuffles (left, right), as a join builds them."""
    j = sc.parallelize((ka, va), Ma).join(sc.parallelize((kb, vb_), Mb), R)
    return j._run()


# ---- 1. random duplicates on both sides (keys include 0 and 2^64-1) -----------------------------
@pytest.mark.parametrize("na,nb,nkeys,R", [(20_000, 30_000, 3000, 4), (5000, 10, 50, 3)])
@pytest.mark.parametrize("kind", KINDS)
def test_random_duplicates(sc, kind, na, nb, nkeys, R):
    rng = np.random.default_rng(na + nb)
    ka, va = rand_pairs(rng, na, nkeys, values="full")
    kb, vb_ = rand_pairs(rng, nb, int(nkeys * 1.5), values="full")
    keep = kb % np.uint64(7) != 0                    # about 1/7 of the keys only on the left, whatever the row counts
    kb, vb_ = kb[keep], vb_[keep]
    assert {0, 2 ** 64 - 1} <= set(ka.tolist())
    got = check(sc, kind, ka, va, 3, kb, vb_, 5, R)
    valid = [(x[2], x[3]) for d in got for rows in d.values() for x in rows]
    assert (1, 1) in valid and ((1, 0) in valid) == (kind != "right") and ((0, 1) in valid) == (kind != "left")


# ---- 2. no shared key, every key shared, one side empty, both empty ------------------------------
@pytest.mark.parametrize("case", ["disjoint", "all_shared", "left_empty", "right_empty", "both_empty"])
@pytest.mark.parametrize("kind", KINDS)
def test_edge_cases(sc, kind, case):
    rng = np.random.default_rng(5)
    ka, va = rand_pairs(rng, 3000, 400)
    kb, vb_ = rand_pairs(rng, 2000, 400)
    e = np.empty(0, dtype=np.uint64)
    if case == "disjoint":
        kb = kb + np.uint64(1)                       # the keys are ranks * odd + 12345: +1 never hits another key
        assert not np.isin(kb, ka).any()
    elif case == "all_shared":
        kb = rng.permutation(np.unique(ka))
        vb_ = rng.integers(0, 1 << 40, len(kb)).astype(np.uint64)
    elif case == "left_empty":
        ka, va = e, e
    elif case == "right_empty":
        kb, vb_ = e, e
    else:
        ka, va, kb, vb_ = e, e, e, e
    got = check(sc, kind, ka, va, 2, kb, vb_, 3, 5)
    n = sum(len(rows) for d in got for rows in d.values())
    if case == "all_shared":
        assert n == len(ka)
    if case == "both_empty" or (case == "left_empty" and kind == "left") or (case == "right_empty" and kind == "right"):
        assert n == 0


# ---- 3. self-join: every key matches ------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_self_join(sc, kind):
    rng = np.random.default_rng(3)
    k, v = rand_pairs(rng, 4000, 300, values="full")
    rdd = sc.parallelize((k, v), 3)
    got = gpu_parts(getattr(rdd, METHOD[kind])(rdd, 4))
    assert_parts_equal(got, OJ.outer_join_parts(kind, k, v, 3, k, v, 3, 4))
    # the same shuffle on both sides: the inner join's rows, every validity byte 1
    sa, _ = _pair(sc, k, v, 3, k, v, 3, 4)
    for r in range(4):
        inner = by_key(*abi_rows(sc, sa, sa, r, None))
        outer = by_key(*abi_rows(sc, sa, sa, r, kind))
        assert outer == inner and all(x[2:] == (1, 1) for rows in outer.values() for x in rows)


# ---- 4. 4-byte keys -----------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_int32_keys(sc, kind):
    rng = np.random.default_rng(4)
    ka = rng.integers(-2000, 1000, 20_000).astype(np.int32)
    kb = rng.integers(0, 3000, 15_000).astype(np.int32)
    ka[:3] = [-1, -(1 << 31), (1 << 31) - 1]
    kb[:2] = [(1 << 31) - 1, -(1 << 31)]
    va = rng.integers(0, 1 << 40, len(ka)).astype(np.uint64)
    vb_ = rng.integers(0, 1 << 40, len(kb)).astype(np.uint64)
    check(sc, kind, ka, va, 3, kb, vb_, 2, 6, key_width=4)


# ---- 5. R = 1, and more partitions than keys ----------------------------------------------------
@pytest.mark.parametrize("R,nkeys", [(1, 500), (300, 100)])
@pytest.mark.parametrize("kind", KINDS)
def test_partition_counts(sc, kind, R, nkeys):
    rng = np.random.default_rng(R)
    ka, va = rand_pairs(rng, 2000, nkeys)
    kb, vb_ = rand_pairs(rng, 1500, nkeys + nkeys // 2)
    got = check(sc, kind, ka, va, 2, kb, vb_, 3, R)
    if R == 300:
        assert sum(1 for d in got if not d) >= 300 - 150


# ---- 6. the reference's examples/join.rs data ---------------------------------------------------
COL1 = [(1, ("A", "B")), (2, ("C", "D")), (3, ("E", "F")), (4, ("G", "H"))]
COL2 = [(1, "A1"), (1, "A2"), (2, "B1"), (2, "B2"), (3, "C1"), (3, "C2")]


@pytest.mark.parametrize("kind", KINDS)
def test_join_rs_data(sc, kind):
    r1 = sc.parallelize((np.array([k for k, _ in COL1], dtype=np.int32), np.arange(4, dtype=np.uint64)), 4)
    r2 = sc.parallelize((np.array([k for k, _ in COL2], dtype=np.int32), np.arange(6, dtype=np.uint64)), 4)
    k, v, w = getattr(r1, METHOD[kind])(r2, 4).collect()
    vs = [None if x is np.ma.masked else COL1[int(x)][1] for x in v] if kind != "left" else [COL1[int(x)][1] for x in v]
    ws = [None if x is np.ma.masked else COL2[int(x)][1] for x in w] if kind != "right" else [COL2[int(x)][1] for x in w]
    got = sorted(zip(k.tolist(), zip(vs, ws)), key=str)
    assert got == sorted(OJ.outer_join(kind, COL1, 4, COL2, 4, 4, int_width=4), key=str)
    if kind != "right":
        assert (4, (("G", "H"), None)) in got


def test_cpp_outer_join_example_runs():
    """examples/outer_join.cpp: r1.left_outer_join(r2) keeps key 4 ("G","H") with None; exit 0 only on the expected
    result of all three joins."""
    path = os.path.join(ROOT, "examples", "_build", "outer_join")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    out = subprocess.run([path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "(4, ((G,H), None))" in out.stdout and "(4, (None, (G,H)))" in out.stdout, out.stdout


# ---- 7. VB_DEVICE output equals VB_HOST output --------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_device_output_equals_host(sc, kind):
    rng = np.random.default_rng(7)
    ka, va = rand_pairs(rng, 8000, 900)
    kb, vb_ = rand_pairs(rng, 6000, 1200)
    sa, sb = _pair(sc, ka, va, 3, kb, vb_, 2, 4)
    for r in range(4):
        host = abi_rows(sc, sa, sb, r, kind, L.VB_HOST)
        dev = abi_rows(sc, sa, sb, r, kind, L.VB_DEVICE)
        for h, d in zip(host, dev):
            assert np.array_equal(_u64(h) if h.dtype.itemsize == 8 else h, _u64(d) if d.dtype.itemsize == 8 else d)
        assert set(np.concatenate([host[3], host[4]]).tolist()) <= {0, 1}
    # NULL validity arrays are skipped
    n = ctypes.c_uint64()
    L.check(sc._lib.vb_join_outer_size(sa._h, sb._h, 0, CODE[kind], ctypes.byref(n)))
    k, v, w = (np.zeros(n.value, dtype=np.uint64) for _ in range(3))
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    L.check(sc._lib.vb_join_outer(sa._h, sb._h, 0, CODE[kind], p(k), p(v), p(w), None, None, L.VB_HOST))
    assert np.array_equal(k, abi_rows(sc, sa, sb, 0, kind)[0])


def test_rejected_calls(sc):
    rng = np.random.default_rng(8)
    ka, va = rand_pairs(rng, 500, 50)
    sa, sb = _pair(sc, ka, va, 2, ka, va, 2, 3)
    lib, n = sc._lib, ctypes.c_uint64()
    for bad in (0, 4, -1):
        assert lib.vb_join_outer_size(sa._h, sb._h, 0, bad, ctypes.byref(n)) == L.VB_ERR_INVALID
        assert lib.vb_join_outer(sa._h, sb._h, 0, bad, None, None, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_join_outer_size(sa._h, sb._h, 3, L.VB_JOIN_LEFT, ctypes.byref(n)) == L.VB_ERR_INVALID
    L.check(lib.vb_join_outer_size(sa._h, sb._h, 0, L.VB_JOIN_FULL, ctypes.byref(n)))
    assert n.value > 0
    assert lib.vb_join_outer(sa._h, sb._h, 0, L.VB_JOIN_FULL, None, None, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    k = np.zeros(n.value, dtype=np.uint64)
    p = k.ctypes.data_as(ctypes.c_void_p)
    assert lib.vb_join_outer(sa._h, sb._h, 0, L.VB_JOIN_FULL, p, p, p, None, None, 5) == L.VB_ERR_INVALID
    other = vb.Shuffle(sc, 1, 4, L.VB_U64, L.VB_U64, L.VB_AGG_COGROUP)     # different n_reduce
    assert lib.vb_join_outer_size(sa._h, other._h, 0, L.VB_JOIN_LEFT, ctypes.byref(n)) == L.VB_ERR_INVALID
    other.free()


# ---- 8. inner and outer joins of the same two shuffles -----------------------------------------
@pytest.mark.parametrize("order", [("inner", "left", "right", "full", "inner"), ("full", "right", "left", "inner", "full"),
                                   ("group", "left", "right", "full", "inner")])
def test_inner_and_outer_on_the_same_shuffles(sc, order):
    """The lazy path caches the filtered sides per (right side, kind): each join must give what it gives alone.
    "group" reads every partition of both sides first (Shuffle.reduce), so the joins start from grouped sides: the
    outer joins must then give exactly the rows of two lazy sides."""
    rng = np.random.default_rng(len(order[0]))
    values = "full" if order[0] == "group" else "default"     # "full" keys include 0 and 2^64-1
    ka, va = rand_pairs(rng, 12_000, 1500, values=values)
    kb, vb_ = rand_pairs(rng, 9000, 2500, values=values)
    R = 4
    sa, sb = _pair(sc, ka, va, 3, kb, vb_, 2, R)
    lazy = _pair(sc, ka, va, 3, kb, vb_, 2, R) if order[0] == "group" else None
    inner = O.join(ka, va, 3, kb, vb_, 2, R)
    for kind in order:
        if kind == "group":
            for s_ in (sa, sb):
                for r in range(R):
                    s_.reduce(r)
            continue
        if kind == "inner":
            want = []
            for k, v, w in inner:
                d = {}
                for row in zip(k.tolist(), v.tolist(), w.tolist()):
                    d.setdefault(row[0], []).append((row[1], row[2], 1, 1))
                want.append(d)
        else:
            want = OJ.outer_join_parts(kind, ka, va, 3, kb, vb_, 2, R)
        got = [by_key(*abi_rows(sc, sa, sb, r, None if kind == "inner" else kind)) for r in range(R)]
        assert_parts_equal(got, want)
        if lazy and kind != "inner":
            assert got == [by_key(*abi_rows(sc, *lazy, r, kind)) for r in range(R)]


# ---- 9. two ranks: only the owned partitions have rows -----------------------------------------
def _dist_data():
    rng = np.random.default_rng(10)
    ka = rng.integers(0, 4000, 60_000).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)
    kb = rng.integers(2000, 7000, 45_000).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)
    va = rng.integers(0, 1 << 50, len(ka)).astype(np.uint64)
    vb_ = rng.integers(0, 1 << 50, len(kb)).astype(np.uint64)
    return ka, va, kb, vb_


def _dist_worker(rank, world, port, Ma, Mb, R, nccl, outdir, p2p):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if nccl else 0
    torch.cuda.set_device(dev)
    if nccl:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{dev}"))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    from vega_b200 import dist as vdist
    ka, va, kb, vb_ = _dist_data()
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
    res = {kind: [by_key(*abi_rows(sc, sa, sb, r, kind)) for r in range(R)] for kind in KINDS}
    with open(os.path.join(outdir, f"o{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    sa.free(); sb.free()
    sc.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("Ma,Mb,R,p2p", [(4, 2, 4, False), (3, 5, 6, True)])
def test_two_ranks(Ma, Mb, R, p2p):
    import socket
    import torch
    import torch.multiprocessing as mp
    world = 2
    nccl = torch.cuda.device_count() >= 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_dist_worker, args=(world, port, Ma, Mb, R, nccl, d, p2p), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"o{r}.pkl"), "rb")) for r in range(world)]
    ka, va, kb, vb_ = _dist_data()
    for kind in KINDS:
        want = OJ.outer_join_parts(kind, ka, va, Ma, kb, vb_, Mb, R)
        for r in range(R):
            owner = r % world
            assert per_rank[owner][kind][r] == want[r], f"{kind} partition {r}"
            assert per_rank[1 - owner][kind][r] == {}, f"{kind} partition {r} has rows on a rank that does not own it"


# ---- 10. configs[3] shape, scaled: unique keys, 2 % shared -----------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_config3_shape_scaled(sc, kind):
    import torch
    n, shared, R = 2_000_000, 40_000, 8
    a = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    b = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=a, first=0, n=n, mode="unique", rank_base=0)
    sc.gen_pairs(out_rows=b, first=0, n=n, mode="unique", rank_base=n - shared)
    ha, hb = a.cpu().numpy().view(np.uint64), b.cpu().numpy().view(np.uint64)
    j = getattr(sc.make_rdd(a, 8), METHOD[kind])(sc.make_rdd(b, 8), R)
    want_n = {"left": n, "right": n, "full": 2 * n - shared}[kind]
    lut_a = dict(zip(ha[:, 0].tolist(), ha[:, 1].tolist()))
    lut_b = dict(zip(hb[:, 0].tolist(), hb[:, 1].tolist()))
    inner = O.join(ha[:, 0].copy(), ha[:, 1].copy(), 8, hb[:, 0].copy(), hb[:, 1].copy(), 8, R)
    total = n_only_l = n_only_r = 0
    for r in range(R):
        k, v, w = j.compute(r)
        (vd, vv), (wd, wv) = _side(v, kind != "left"), _side(w, kind != "right")
        k = _u64(k)
        total += len(k)
        assert len(np.unique(k)) == len(k)                               # unique keys: one row per key
        both = (vv == 1) & (wv == 1)
        # the matched rows are exactly the oracle's inner join of this partition
        assert sorted(zip(k[both].tolist(), vd[both].tolist(), wd[both].tolist())) == \
            sorted(zip(*[x.tolist() for x in inner[r]]))
        # every unmatched row: validity 0 on the missing side, the key really is missing there
        only_l, only_r = (vv == 1) & (wv == 0), (vv == 0) & (wv == 1)
        assert not ((vv == 0) & (wv == 0)).any()
        n_only_l += int(only_l.sum())
        n_only_r += int(only_r.sum())
        # oracle-sampled subset: values and placement of every 997th unmatched row
        for i in np.flatnonzero(only_l | only_r)[::997].tolist():
            key = int(k[i])
            assert O.get_partition(key, R) == r
            if only_l[i]:
                assert key not in lut_b and lut_a[key] == int(vd[i]) and int(wd[i]) == 0
            else:
                assert key not in lut_a and lut_b[key] == int(wd[i]) and int(vd[i]) == 0
    assert total == want_n
    assert n_only_l == (n - shared if kind != "right" else 0) and n_only_r == (n - shared if kind != "left" else 0)
    del a, b
    torch.cuda.empty_cache()


# ---- 11. the right side freed after a size call, and a new shuffle at its address ------------------------------
def _grouped(sc, k, v, R):
    """A sealed COGROUP shuffle of (k, v) in one map task, grouped by reading every partition."""
    s = vb.Shuffle(sc, 1, R, L.VB_U64, L.VB_U64, L.VB_AGG_COGROUP)
    s.map(0, vb.rdd._Col(k), vb.rdd._Col(v), 0, len(k))
    s.seal()
    for r in range(R):
        s.reduce(r)
    return s


def test_right_side_address_reused(sc):
    """A size call with no write, then the right side freed: a later join with another shuffle that the allocator
    places at the freed side's address gets that shuffle's sizes and rows.  The sizes are checked before any write."""
    R = 3
    rng = np.random.default_rng(11)
    ka, va = rand_pairs(rng, 6000, 800)
    k1, v1 = rand_pairs(rng, 4000, 1000)
    k2, v2 = rand_pairs(rng, 9000, 3000)                # other rows: every partition's sizes differ from r1's
    lib, n = sc._lib, ctypes.c_uint64()
    mask = {"left": 0b01, "right": 0b10, "full": 0}
    want = {kind: OJ.outer_join_parts(kind, ka, va, 1, k2, v2, 1, R) for kind in KINDS}
    sa, r1 = _grouped(sc, ka, va, R), _grouped(sc, k1, v1, R)
    old = {}
    for kind in KINDS:
        for r in range(R):
            L.check(lib.vb_join_outer_size(sa._h, r1._h, r, CODE[kind], ctypes.byref(n)))
            old[kind, r] = n.value
    addr = r1._h.value
    r1.free()
    others = []
    try:
        for _ in range(64):
            r2 = _grouped(sc, k2, v2, R)
            if r2._h.value == addr:
                break
            others.append(r2)
        else:
            pytest.skip("the allocator never placed a new shuffle at the freed right side's address")
        nn = ctypes.c_uint64()
        for kind in KINDS:
            for r in range(R):
                L.check(lib.vb_join_outer_size(sa._h, r2._h, r, CODE[kind], ctypes.byref(n)))
                L.check(lib.vb_join_n_outer_size((ctypes.c_void_p * 2)(sa._h.value, r2._h.value), 2, r, mask[kind],
                                                 ctypes.byref(nn)))
                rows = sum(len(x) for x in want[kind][r].values())
                assert rows != old[kind, r]
                assert (n.value, nn.value) == (rows, rows), (kind, r, old[kind, r])
        for kind in KINDS:
            assert_parts_equal([by_key(*abi_rows(sc, sa, r2, r, kind)) for r in range(R)], want[kind])
    finally:
        for s_ in others:
            s_.free()
