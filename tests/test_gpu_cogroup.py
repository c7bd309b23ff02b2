"""GPU cogroup (vb_cogroup, JoinedRdd.cogroup_compute / cogroup_collect, PairRddT::cogroup) against the C oracle's group
shuffle of each side.  Every partition is checked: each key appears once and hashes to the partition, both value lists
equal the reference element for element and in order, the offsets start at 0, are monotone and match the value
counts, and no key has two empty lists."""
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
from oracle import pyref as P
from tests.test_gpu_outer_join import abi_rows, by_key
from tests.outer_join_ref import outer_join_parts
from tests.util import EMPTY_KEY, assert_parts_equal, rand_pairs
from vega_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def _u64(x):
    x = np.ascontiguousarray(x)
    return x.view(np.uint64) if x.dtype.itemsize == 8 else x.astype(np.int64).view(np.uint64)


def _group(keys, vals, M, R, key_width):
    """{key: [values]} per partition (u64 bits) from the C oracle's group shuffle."""
    if len(keys) == 0:
        return [{} for _ in range(R)]
    out = []
    for p in O.shuffle("group", _u64(keys), _u64(vals), M, R, key_width=key_width):
        o, v = p["offsets"].tolist(), _u64(p["vals"]).tolist()
        out.append({int(k): v[o[i]:o[i + 1]] for i, k in enumerate(p["keys"].tolist())})
    return out


def ref_parts(ka, va, Ma, kb, vb_, Mb, R, key_width=8):
    """Per partition {key: (left list, right list)}: the union of both sides' keys, [] for a side that lacks one."""
    ga, gb = _group(ka, va, Ma, R, key_width), _group(kb, vb_, Mb, R, key_width)
    return [{k: (a.get(k, []), b.get(k, [])) for k in a.keys() | b.keys()} for a, b in zip(ga, gb)]


def part_dict(keys, lo, lv, ro, rv, r, R, key_width=8):
    """Check one partition's structure and return it as {key: (left list, right list)}."""
    keys, lo, ro, lv, rv = _u64(keys).tolist(), _u64(lo), _u64(ro), _u64(lv).tolist(), _u64(rv).tolist()
    n = len(keys)
    assert len(lo) == n + 1 and len(ro) == n + 1
    for o, vals in ((lo, lv), (ro, rv)):
        assert o[0] == 0 and o[-1] == len(vals)
        assert (np.diff(o.astype(np.int64)) >= 0).all(), "offsets are not monotone"
    assert len(set(keys)) == n, "a key appears twice in one partition"
    lo, ro = lo.tolist(), ro.tolist()
    d = {}
    for i, k in enumerate(keys):
        assert O.get_partition(k, R, key_width) == r, f"key {k:#x} is not in partition {r}"
        assert lo[i + 1] > lo[i] or ro[i + 1] > ro[i], f"key {k:#x} has two empty lists"
        d[k] = (lv[lo[i]:lo[i + 1]], rv[ro[i]:ro[i + 1]])
    return d


def gpu_parts(j, key_width=8):
    """Per-partition dicts of a JoinedRdd's cogroup through the Python mirror."""
    out = []
    for r in range(j.num_slices):
        keys, (lo, lv), (ro, rv) = j.cogroup_compute(r)
        out.append(part_dict(keys, lo, lv, ro, rv, r, j.num_slices, key_width))
    return out


def abi_cogroup(sc, sa, sb, r, dst=L.VB_HOST):
    """One partition through the C ABI: (keys, left_offsets, left_vals, right_offsets, right_vals) as u64 host arrays."""
    lib = sc._lib
    nk, nl, nr = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    L.check(lib.vb_cogroup_size(sa._h, sb._h, r, ctypes.byref(nk), ctypes.byref(nl), ctypes.byref(nr)))
    sizes = (nk.value, nk.value + 1, nl.value, nk.value + 1, nr.value)
    if dst == L.VB_HOST:
        bufs = [np.full(s, 7, dtype=np.uint64) for s in sizes]
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    else:
        import torch
        bufs = [torch.full((s,), 7, dtype=torch.int64, device="cuda") for s in sizes]
        p = lambda x: ctypes.c_void_p(x.data_ptr()) if x.numel() else None
        torch.cuda.synchronize()
    L.check(lib.vb_cogroup(sa._h, sb._h, r, *[p(x) for x in bufs], dst))
    if dst != L.VB_HOST:
        bufs = [x.cpu().numpy().view(np.uint64) for x in bufs]
    return tuple(bufs)


def abi_parts(sc, sa, sb, R, key_width=8):
    return [part_dict(*abi_cogroup(sc, sa, sb, r), r, R, key_width) for r in range(R)]


def _pair(sc, ka, va, Ma, kb, vb_, Mb, R):
    """Two sealed COGROUP shuffles (left, right), as cogroup builds them."""
    return sc.parallelize((ka, va), Ma).cogroup(sc.parallelize((kb, vb_), Mb), R)._run()


def check(sc, ka, va, Ma, kb, vb_, Mb, R, key_width=8):
    a, b = sc.parallelize((ka, va), Ma), sc.parallelize((kb, vb_), Mb)
    got = gpu_parts(a.cogroup(b, R), key_width)
    assert_parts_equal(got, ref_parts(ka, va, Ma, kb, vb_, Mb, R, key_width))
    return got


# ---- 1. random duplicates on both sides; keys 0 and 2^64-1 on one side only, or on both -----------
@pytest.mark.parametrize("na,nb,nkeys,R", [(20_000, 30_000, 3000, 4), (5000, 10, 50, 3)])
@pytest.mark.parametrize("extremes", ["split", "both"])
def test_random_duplicates(sc, na, nb, nkeys, R, extremes):
    rng = np.random.default_rng(na + nb)
    ka, va = rand_pairs(rng, na, nkeys, values="full")
    kb, vb_ = rand_pairs(rng, nb, int(nkeys * 1.5), values="full")
    kb, vb_ = kb[kb % np.uint64(7) != 0], vb_[kb % np.uint64(7) != 0]     # some keys only on the left
    if extremes == "split":            # 0 only on the left, 2^64-1 only on the right
        ka[ka == np.uint64(EMPTY_KEY)] = np.uint64(0)
        kb = np.concatenate([np.full(2, EMPTY_KEY, dtype=np.uint64), kb])
        assert 0 in set(ka.tolist()) and EMPTY_KEY not in set(ka.tolist())
        assert EMPTY_KEY in set(kb.tolist()) and 0 not in set(kb.tolist())
    else:
        kb = np.concatenate([np.array([0, EMPTY_KEY], dtype=np.uint64), kb])
        assert {0, EMPTY_KEY} <= set(ka.tolist()) & set(kb.tolist())
    vb_ = np.concatenate([np.array([5, 2 ** 64 - 1], dtype=np.uint64), vb_])
    got = check(sc, ka, va, 3, kb, vb_, 5, R)
    lists = [x for d in got for x in d.values()]
    assert any(x and y for x, y in lists) and any(x and not y for x, y in lists)
    if len(kb) > 100:
        assert any(y and not x for x, y in lists)


# ---- 2. disjoint, identical, one side empty, both empty -----------------------------------------
@pytest.mark.parametrize("case", ["disjoint", "identical", "left_empty", "right_empty", "both_empty"])
def test_edge_cases(sc, case):
    rng = np.random.default_rng(5)
    ka, va = rand_pairs(rng, 3000, 400)
    kb, vb_ = rand_pairs(rng, 2000, 400)
    e = np.empty(0, dtype=np.uint64)
    if case == "disjoint":
        kb = kb + np.uint64(1)                       # the keys are ranks * odd + 12345: +1 never hits another key
        assert not np.isin(kb, ka).any()
    elif case == "identical":
        kb, vb_ = ka.copy(), va.copy()
    elif case == "left_empty":
        ka, va = e, e
    elif case == "right_empty":
        kb, vb_ = e, e
    else:
        ka, va, kb, vb_ = e, e, e, e
    got = check(sc, ka, va, 2, kb, vb_, 3, 5)
    n = sum(len(d) for d in got)
    assert n == len(set(ka.tolist()) | set(kb.tolist()))
    if case == "identical":
        assert all(x == y for d in got for x, y in d.values())


# ---- 3. self-cogroup: left == right --------------------------------------------------------------
def test_self_cogroup(sc):
    rng = np.random.default_rng(3)
    k, v = rand_pairs(rng, 4000, 300, values="full")
    R = 4
    sa, _ = _pair(sc, k, v, 3, k, v, 3, R)
    g = _group(k, v, 3, R, 8)
    want = [{kk: (vs, vs) for kk, vs in d.items()} for d in g]
    assert_parts_equal(abi_parts(sc, sa, sa, R), want)
    rdd = sc.parallelize((k, v), 3)
    assert_parts_equal(gpu_parts(rdd.cogroup(rdd, R)), want)


# ---- 4. 4-byte keys -----------------------------------------------------------------------------
def test_int32_keys(sc):
    rng = np.random.default_rng(4)
    ka = rng.integers(-2000, 1000, 20_000).astype(np.int32)
    kb = rng.integers(0, 3000, 15_000).astype(np.int32)
    ka[:3] = [-1, -(1 << 31), (1 << 31) - 1]
    kb[:2] = [(1 << 31) - 1, -(1 << 31)]
    va = rng.integers(0, 1 << 40, len(ka)).astype(np.uint64)
    vb_ = rng.integers(0, 1 << 40, len(kb)).astype(np.uint64)
    check(sc, ka, va, 3, kb, vb_, 2, 6, key_width=4)


# ---- 5. i64 and f64 values, bit for bit ---------------------------------------------------------
@pytest.mark.parametrize("vdtype,values", [("i64", "full"), ("f64", "special")])
def test_value_dtypes(sc, vdtype, values):
    rng = np.random.default_rng(11)
    ka, va = rand_pairs(rng, 12_000, 1500, vdtype=vdtype, values=values)
    kb, vb_ = rand_pairs(rng, 9000, 2500, vdtype=vdtype, values=values)
    j = sc.parallelize((ka, va), 3).cogroup(sc.parallelize((kb, vb_), 2), 5)
    keys, (lo, lv), (ro, rv) = j.cogroup_compute(0)
    assert lv.dtype == va.dtype and rv.dtype == vb_.dtype
    assert_parts_equal(gpu_parts(j), ref_parts(ka, va, 3, kb, vb_, 2, 5))
    # cogroup_collect keeps its return value: (k, (vs, ws)) with numpy arrays of the value dtype
    got = {int(_u64(np.array([k]))[0]): (_u64(x).tolist(), _u64(y).tolist()) for k, (x, y) in j.cogroup_collect()}
    want = {k: x for d in ref_parts(ka, va, 3, kb, vb_, 2, 5) for k, x in d.items()}
    assert got == want


# ---- 6. R = 1, and more partitions than keys ----------------------------------------------------
@pytest.mark.parametrize("R,nkeys", [(1, 500), (300, 100)])
def test_partition_counts(sc, R, nkeys):
    rng = np.random.default_rng(R)
    ka, va = rand_pairs(rng, 2000, nkeys)
    kb, vb_ = rand_pairs(rng, 1500, nkeys + nkeys // 2)
    got = check(sc, ka, va, 2, kb, vb_, 3, R)
    if R == 300:
        assert sum(1 for d in got if not d) >= 300 - 150


# ---- 7. one key with 10^6 right values, matched by a left key -----------------------------------
def test_skewed_key(sc):
    rng = np.random.default_rng(12)
    hot = np.uint64(0xDEADBEEF12345)
    ka, va = rand_pairs(rng, 20_000, 4000)
    kb, vb_ = rand_pairs(rng, 50_000, 6000)
    ka = np.concatenate([ka, np.full(3, hot, dtype=np.uint64)])
    va = np.concatenate([va, np.array([1, 2, 3], dtype=np.uint64)])
    kb = np.concatenate([np.full(1_000_000, hot, dtype=np.uint64), kb])
    vb_ = np.concatenate([np.arange(1_000_000, dtype=np.uint64) * np.uint64(3) + np.uint64(1), vb_])
    perm = rng.permutation(len(kb))                   # the hot key's values spread over every map task
    kb, vb_ = kb[perm], vb_[perm]
    R = 4
    got = check(sc, ka, va, 3, kb, vb_, 4, R)
    hot_lists = [d[int(hot)] for d in got if int(hot) in d]
    assert len(hot_lists) == 1 and hot_lists[0][0] == [1, 2, 3] and len(hot_lists[0][1]) == 1_000_000


# ---- 8. the reference's tests/test_rdd.rs data ----------------------------------------------------
def test_test_rdd_cogroup_golden(sc):
    # tests/test_rdd.rs:434-456: (1,"A"), (2,"B"), (3,"C"), (4,"D") cogrouped with itself, 2 slices, 2 partitions
    names = ["A", "B", "C", "D"]
    k = np.array([1, 2, 3, 4], dtype=np.int32)
    v = np.arange(4, dtype=np.uint64)
    cg = sc.parallelize((k, v), 2).cogroup(sc.parallelize((k, v), 2), 2).cogroup_collect()
    got = sorted((a, ([names[i] for i in x.tolist()], [names[i] for i in y.tolist()])) for a, (x, y) in cg)
    rows = list(zip(k.tolist(), names))
    want = sorted((a, (vs, ws)) for a, (vs, ws) in P.cogroup(rows, 2, rows, 2, 2, int_width=4))
    assert got == want == [(1, (["A"], ["A"])), (2, (["B"], ["B"])), (3, (["C"], ["C"])), (4, (["D"], ["D"]))]


@pytest.mark.parametrize("nparts", [3, 2])
def test_intersection_and_subtract_goldens(sc, nparts):
    # tests/test_rdd.rs:484-521 (intersection → [3,4,5,13]) and :675-699 (subtract → [0,1,2,10,12,19]), both read
    # off the device cogroup: keys with values on both sides, and keys with an empty right list
    c1 = np.array([1, 2, 3, 4, 5, 10, 12, 13, 19, 0], dtype=np.int32)
    c2 = np.array([3, 4, 5, 6, 7, 8, 11, 13], dtype=np.int32)
    j = sc.parallelize((c1, np.zeros(10, np.uint64)), 2).cogroup(sc.parallelize((c2, np.zeros(8, np.uint64)), 4), nparts)
    parts = gpu_parts(j, key_width=4)
    lists = {k: x for d in parts for k, x in d.items()}
    assert sorted(k for k, (x, y) in lists.items() if x and y) == [3, 4, 5, 13]
    assert sorted(k for k, (x, y) in lists.items() if x and not y) == [0, 1, 2, 10, 12, 19]
    assert len(lists) == 14


def test_cpp_cogroup_example_runs():
    """examples/cogroup.cpp: the test_rdd.rs cogroup, intersection and subtract data; exit 0 only on the expected
    result."""
    path = os.path.join(ROOT, "examples", "_build", "cogroup")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    out = subprocess.run([path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "(1, ([A], [A]))" in out.stdout and "intersection: [3, 4, 5, 13]" in out.stdout, out.stdout
    assert "subtract: [0, 1, 2, 10, 12, 19]" in out.stdout, out.stdout


# ---- 9. VB_DEVICE output equals VB_HOST output; NULL outputs are skipped ---------------------------
def test_device_output_equals_host(sc):
    rng = np.random.default_rng(7)
    ka, va = rand_pairs(rng, 8000, 900)
    kb, vb_ = rand_pairs(rng, 6000, 1200)
    sa, sb = _pair(sc, ka, va, 3, kb, vb_, 2, 4)
    for r in range(4):
        host = abi_cogroup(sc, sa, sb, r, L.VB_HOST)
        dev = abi_cogroup(sc, sa, sb, r, L.VB_DEVICE)
        for h, d in zip(host, dev):
            assert np.array_equal(h, d)
    lib, nk = sc._lib, ctypes.c_uint64()
    L.check(lib.vb_cogroup_size(sa._h, sb._h, 1, ctypes.byref(nk), None, None))
    ro = np.zeros(nk.value + 1, dtype=np.uint64)
    L.check(lib.vb_cogroup(sa._h, sb._h, 1, None, None, None, ro.ctypes.data_as(ctypes.c_void_p), None, L.VB_HOST))
    assert np.array_equal(ro, abi_cogroup(sc, sa, sb, 1)[3])


def test_rejected_calls(sc):
    rng = np.random.default_rng(8)
    ka, va = rand_pairs(rng, 500, 50)
    sa, sb = _pair(sc, ka, va, 2, ka, va, 2, 3)
    lib, n = sc._lib, ctypes.c_uint64()
    size = lambda x, y, r=0: lib.vb_cogroup_size(x, y, r, ctypes.byref(n), ctypes.byref(n), ctypes.byref(n))
    rows = lambda x, y, r=0, dst=L.VB_HOST: lib.vb_cogroup(x, y, r, None, None, None, None, None, dst)
    assert size(None, sb._h) == L.VB_ERR_INVALID and rows(sa._h, None) == L.VB_ERR_INVALID
    assert size(sa._h, sb._h, 3) == L.VB_ERR_INVALID and rows(sa._h, sb._h, 3) == L.VB_ERR_INVALID
    assert rows(sa._h, sb._h, 0, 5) == L.VB_ERR_INVALID and rows(sa._h, sb._h, 0, -1) == L.VB_ERR_INVALID
    others = {
        "n_reduce": _pair(sc, ka, va, 2, ka, va, 2, 4)[0],
        "key width": _pair(sc, ka.astype(np.int32), va, 2, ka.astype(np.int32), va, 2, 3)[0],
        "SUM": sc.parallelize((ka, va), 2).reduce_by_key("sum", 3)._run(),
        "combine_by_key": sc.parallelize(ka, 2, values=(va,)).combine_by_key({"n": ("count", None)}, 3)._run(),
    }
    for what, o in others.items():
        for x, y in ((sa._h, o._h), (o._h, sa._h)):
            assert size(x, y) == L.VB_ERR_INVALID, what
            assert rows(x, y) == L.VB_ERR_INVALID, what
    # the valid call still works after the rejections
    L.check(size(sa._h, sb._h))


# ---- 10. cogroup, inner join and full outer join of the same two shuffles ---------------------------
@pytest.mark.parametrize("order", [("cogroup", "inner", "full", "cogroup"), ("full", "inner", "cogroup", "cogroup"),
                                   ("group", "cogroup", "inner", "full")])
def test_cogroup_and_joins_on_the_same_shuffles(sc, order):
    """cogroup shares the FULL filtered pair with full_outer_join; each call must give what it gives alone, and the
    originals must still group as they did.  "group" reads every partition of both sides first (Shuffle.reduce), so
    the later calls start from grouped sides: the cogroup must then equal the one of two lazy sides."""
    rng = np.random.default_rng(len(order[0]))
    values = "full" if order[0] == "group" else "default"     # "full" keys include 0 and 2^64-1
    ka, va = rand_pairs(rng, 12_000, 1500, values=values)
    kb, vb_ = rand_pairs(rng, 9000, 2500, values=values)
    R = 4
    sa, sb = _pair(sc, ka, va, 3, kb, vb_, 2, R)
    lazy = _pair(sc, ka, va, 3, kb, vb_, 2, R) if order[0] == "group" else None
    want_cg = ref_parts(ka, va, 3, kb, vb_, 2, R)
    for op in order:
        if op == "group":
            for s_ in (sa, sb):
                for r in range(R):
                    s_.reduce(r)
        elif op == "cogroup":
            got = abi_parts(sc, sa, sb, R)
            assert_parts_equal(got, want_cg)
            if lazy:
                assert got == abi_parts(sc, *lazy, R)
        elif op == "inner":
            want = []
            for k, v, w in O.join(ka, va, 3, kb, vb_, 2, R):
                d = {}
                for row in zip(k.tolist(), v.tolist(), w.tolist()):
                    d.setdefault(row[0], []).append((row[1], row[2], 1, 1))
                want.append(d)
            assert_parts_equal([by_key(*abi_rows(sc, sa, sb, r, None)) for r in range(R)], want)
        else:
            assert_parts_equal([by_key(*abi_rows(sc, sa, sb, r, "full")) for r in range(R)],
                               outer_join_parts("full", ka, va, 3, kb, vb_, 2, R))
    for s_, k, v, M in ((sa, ka, va, 3), (sb, kb, vb_, 2)):
        got = []
        for r in range(R):
            keys, offs, vals = s_.reduce(r)
            o, vals = offs.tolist(), _u64(vals).tolist()
            got.append({int(x): vals[o[i]:o[i + 1]] for i, x in enumerate(_u64(keys).tolist())})
        assert_parts_equal(got, _group(k, v, M, R, 8))
    assert_parts_equal(abi_parts(sc, sa, sb, R), want_cg)


# ---- 11. two ranks: only the owned partitions have keys ------------------------------------------
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
    res = abi_parts(sc, sa, sb, R)
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
    want = ref_parts(ka, va, Ma, kb, vb_, Mb, R)
    for r in range(R):
        owner = r % world
        assert per_rank[owner][r] == want[r], f"partition {r}"
        assert per_rank[1 - owner][r] == {}, f"partition {r} has keys on a rank that does not own it"


# ---- 12. the benchmark's shape, scaled: unique keys, 2 % shared ------------------------------------
def test_bench_shape_scaled(sc):
    import torch
    n, shared, R = 2_000_000, 40_000, 8
    a = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    b = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=a, first=0, n=n, mode="unique", rank_base=0)
    sc.gen_pairs(out_rows=b, first=0, n=n, mode="unique", rank_base=n - shared)
    ha, hb = a.cpu().numpy().view(np.uint64), b.cpu().numpy().view(np.uint64)
    j = sc.make_rdd(a, 8).cogroup(sc.make_rdd(b, 8), R)
    sides = []
    for h in (ha, hb):
        order = np.argsort(h[:, 0], kind="stable")
        sides.append((h[order, 0], h[order, 1]))
    total = n_both = 0
    for r in range(R):
        keys, (lo, lv), (ro, rv) = j.cogroup_compute(r)
        keys = _u64(keys)
        total += len(keys)
        assert len(np.unique(keys)) == len(keys)
        for (sk, sv), o, vals in zip(sides, (lo, ro), (_u64(lv), _u64(rv))):
            cnt = np.diff(o.astype(np.int64))
            assert o[0] == 0 and o[-1] == len(vals) and set(np.unique(cnt).tolist()) <= {0, 1}
            at = np.searchsorted(sk, keys)
            present = (at < len(sk)) & (sk[np.minimum(at, len(sk) - 1)] == keys)
            assert np.array_equal(present, cnt == 1), "a key's list is empty on a side that has it, or the reverse"
            assert np.array_equal(sv[at[present]], vals)
        n_both += int(((np.diff(lo.astype(np.int64)) == 1) & (np.diff(ro.astype(np.int64)) == 1)).sum())
        for i in range(0, len(keys), 9973):
            assert O.get_partition(int(keys[i]), R) == r
    assert total == 2 * n - shared and n_both == shared
    del a, b
    torch.cuda.empty_cache()
