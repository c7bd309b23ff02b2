"""GPU cogroup and inner join of any number of shuffles (vb_cogroup_n / vb_join_n, CoGroupedRdd, PairRddT::cogroup_n /
join_n) against each side's C-oracle group shuffle joined by key union (tests/cogroup_n_ref.py), and against
vb_shuffle_reduce, vb_cogroup and vb_join where they apply.  Every partition is checked: each key appears once and
hashes to the partition, every side's list equals the reference element for element and in order, the offsets start
at 0, are monotone and match the value counts, and no key has every list empty.  Join rows are compared per key in
output order."""
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
from tests import cogroup_n_ref as CN
from tests.test_gpu_cogroup import _group, abi_parts
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


def shuffles(sc, sides, R):
    """One sealed COGROUP shuffle per side [(keys, vals, num_slices), ...], as CoGroupedRdd builds them."""
    return vb.CoGroupedRdd([sc.parallelize((k, v), M) for k, v, M in sides], R)._run()


def group_all(shs, R):
    """Read every partition of every shuffle with vb_shuffle_reduce: a lazy COGROUP shuffle is grouped by it."""
    for s in shs:
        for r in range(R):
            s.reduce(r)


def _arr(shs):
    return (ctypes.c_void_p * len(shs))(*[s._h.value if s is not None else None for s in shs])


def _bufs(sizes, dst, fill=7):
    if dst == L.VB_HOST:
        return [np.full(s, fill, dtype=np.uint64) for s in sizes], lambda x: x.ctypes.data
    import torch
    torch.cuda.synchronize()
    return [torch.full((s,), fill, dtype=torch.int64, device="cuda") for s in sizes], \
        lambda x: x.data_ptr() if x.numel() else None


def _host(xs):
    return [x if isinstance(x, np.ndarray) else x.cpu().numpy().view(np.uint64) for x in xs]


def abi_cogroup_n(sc, shs, r, dst=L.VB_HOST):
    """One partition through the C ABI: (keys, [offsets per side], [values per side]) as u64 host arrays."""
    lib, n = sc._lib, len(shs)
    nk, nv = ctypes.c_uint64(), (ctypes.c_uint64 * n)()
    L.check(lib.vb_cogroup_n_size(_arr(shs), n, r, ctypes.byref(nk), nv))
    bufs, p = _bufs([nk.value] + [nk.value + 1] * n + list(nv), dst)
    ptrs = lambda xs: (ctypes.c_void_p * n)(*[p(x) for x in xs])
    L.check(lib.vb_cogroup_n(_arr(shs), n, r, p(bufs[0]), ptrs(bufs[1:1 + n]), ptrs(bufs[1 + n:]), dst))
    bufs = _host(bufs)
    return bufs[0], bufs[1:1 + n], bufs[1 + n:]


def part_dict_n(keys, offs, vals, r, R, key_width=8):
    """Check one partition's structure and return it as {key: (list of side 0, list of side 1, ...)}."""
    keys = _u64(keys).tolist()
    n = len(keys)
    lists = []
    for o, v in zip(offs, vals):
        o = _u64(o)
        assert len(o) == n + 1 and o[0] == 0 and o[-1] == len(v), "offsets do not start at 0 or end at the value count"
        assert (np.diff(o.astype(np.int64)) >= 0).all(), "offsets are not monotone"
        lists.append((o.tolist(), _u64(v).tolist()))
    assert len(set(keys)) == n, "a key appears twice in one partition"
    d = {}
    for i, k in enumerate(keys):
        assert O.get_partition(k, R, key_width) == r, f"key {k:#x} is not in partition {r}"
        d[k] = tuple(v[o[i]:o[i + 1]] for o, v in lists)
        assert any(d[k]), f"key {k:#x} has every list empty"
    return d


def abi_parts_n(sc, shs, R, key_width=8):
    return [part_dict_n(*abi_cogroup_n(sc, shs, r), r, R, key_width) for r in range(R)]


def abi_join_n(sc, shs, r, dst=L.VB_HOST):
    """One partition of vb_join_n: (k, [v per side]) as u64 host arrays."""
    lib, n = sc._lib, len(shs)
    rows = ctypes.c_uint64()
    L.check(lib.vb_join_n_size(_arr(shs), n, r, ctypes.byref(rows)))
    bufs, p = _bufs([rows.value] * (n + 1), dst)
    L.check(lib.vb_join_n(_arr(shs), n, r, p(bufs[0]), (ctypes.c_void_p * n)(*[p(x) for x in bufs[1:]]), dst))
    bufs = _host(bufs)
    return bufs[0], bufs[1:]


def join_by_key(k, vs):
    """{key: [row tuples in output order]}; a key's rows must be contiguous."""
    d, prev = {}, None
    for row in zip(_u64(k).tolist(), *[_u64(v).tolist() for v in vs]):
        if row[0] != prev:
            assert row[0] not in d, f"the rows of key {row[0]:#x} are not contiguous"
            d[row[0]], prev = [], row[0]
        d[row[0]].append(row[1:])
    return d


def join_parts_n(sc, shs, R, key_width=8):
    out = []
    for r in range(R):
        d = join_by_key(*abi_join_n(sc, shs, r))
        assert all(O.get_partition(k, R, key_width) == r for k in d)
        out.append(d)
    return out


def check(sc, sides, R, key_width=8, join=True):
    """Cogroup (and join) of fresh shuffles of the sides against the array reference; returns the cogroup parts."""
    want = CN.ref_parts_n(sides, R, key_width)
    shs = shuffles(sc, sides, R)
    got = abi_parts_n(sc, shs, R, key_width)
    assert_parts_equal(got, want)
    if join:
        assert_parts_equal(join_parts_n(sc, shs, R, key_width), CN.join_of_parts(want))
    return got


# ---- 1. three sides, random duplicates; keys 0 and 2^64-1 on some sides only -------------------------------------
@pytest.mark.parametrize("R", [4, 7])
def test_three_sides_random_duplicates(sc, R):
    rng = np.random.default_rng(R)
    ka, va = rand_pairs(rng, 20_000, 3000, values="full")          # 0 and 2^64-1 among the keys
    kb, vb_ = rand_pairs(rng, 15_000, 4000, values="full")
    kc, vc = rand_pairs(rng, 8000, 2500)
    kb[kb == np.uint64(EMPTY_KEY)] = np.uint64(0)                   # side 1: 0 only; side 2: 2^64-1 only
    kc = np.concatenate([np.full(3, EMPTY_KEY, dtype=np.uint64), kc])
    vc = np.concatenate([np.array([1, 2, 3], dtype=np.uint64), vc])
    assert EMPTY_KEY not in set(kb.tolist()) and 0 not in set(kc.tolist())
    got = check(sc, [(ka, va, 3), (kb, vb_, 5), (kc, vc, 2)], R)
    lists = [x for d in got for x in d.values()]
    for j in range(3):
        assert any(not x[j] for x in lists) and any(x[j] for x in lists)
    assert any(all(x) for x in lists) and any(sum(1 for y in x if y) == 1 for x in lists)


# ---- 2. one side: vb_shuffle_reduce of that side, key by key ----------------------------------------------------------
@pytest.mark.parametrize("grouped", [False, True])
def test_one_side_is_the_shuffle_reduce(sc, grouped):
    rng = np.random.default_rng(2)
    k, v = rand_pairs(rng, 12_000, 1500, values="full")
    R = 5
    (s,) = shuffles(sc, [(k, v, 3)], R)
    ref = [{kk: tuple([x]) for kk, x in d.items()} for d in _group(k, v, 3, R, 8)]
    if grouped:
        group_all([s], R)
    got = abi_parts_n(sc, [s], R)
    for r in range(R):
        keys, offs, vals = s.reduce(r)
        o, vals = offs.tolist(), _u64(vals).tolist()
        assert {int(x): (vals[o[i]:o[i + 1]],) for i, x in enumerate(_u64(keys).tolist())} == got[r]
    assert_parts_equal(got, ref)
    want_j = [{kk: [(x,) for x in vs[0]] for kk, vs in d.items()} for d in ref]
    assert_parts_equal(join_parts_n(sc, [s], R), want_j)


# ---- 3. two sides: vb_cogroup and vb_join of the same data, lazy and grouped sides ------------------------------------
@pytest.mark.parametrize("grouped", [False, True])
def test_two_sides_match_cogroup_and_join(sc, grouped):
    rng = np.random.default_rng(3)
    ka, va = rand_pairs(rng, 15_000, 2000, values="full")
    kb, vb_ = rand_pairs(rng, 10_000, 3000, values="full")
    R = 4
    sides = [(ka, va, 3), (kb, vb_, 2)]
    fresh = lambda: shuffles(sc, sides, R)
    pair, pair_j = fresh(), fresh()
    n_way, n_way_j = (fresh(), fresh()) if not grouped else (pair, pair_j)
    if grouped:
        group_all(pair + pair_j, R)
    want_cg = abi_parts(sc, *pair, R)
    want_j = [{k: [x[:2] for x in rows] for k, rows in by_key(*abi_rows(sc, *pair_j, r, None)).items()} for r in range(R)]
    got_cg = abi_parts_n(sc, n_way, R)
    assert got_cg == want_cg
    assert join_parts_n(sc, n_way_j, R) == want_j
    assert_parts_equal(got_cg, CN.ref_parts_n(sides, R))


# ---- 4. sixteen sides; seventeen are rejected ---------------------------------------------------------------------------
def test_sixteen_sides_and_seventeen_rejected(sc):
    rng = np.random.default_rng(4)
    sides = []
    for j in range(16):
        k, v = rand_pairs(rng, 600 + 50 * j, 120)
        sides.append((k, v, 1 + j % 4))
    R = 3
    got = check(sc, sides, R, join=False)
    assert any(all(x) for d in got for x in d.values())
    # the join of these sides has about 10^15 rows: its size only, the sum over keys of the product of the list lengths
    shs = shuffles(sc, sides, R)
    n = ctypes.c_uint64()
    for r in range(R):
        L.check(sc._lib.vb_join_n_size(_arr(shs), 16, r, ctypes.byref(n)))
        assert n.value == sum(int(np.prod([len(x) for x in lists], dtype=object)) for lists in got[r].values())
    # rows of a small 16-way join: key 1 once on every side, key 2 twice on sides 0 and 15 and once elsewhere
    small = [(np.array([1, 2, 2, 100 + j] if j in (0, 15) else [1, 2, 100 + j], dtype=np.uint64), None, 1 + j % 3)
             for j in range(16)]
    small = [(k, np.arange(len(k), dtype=np.uint64) + np.uint64(1000 * j), M) for j, (k, _, M) in enumerate(small)]
    check(sc, small, R)
    rows = {k: x for d in join_parts_n(sc, shuffles(sc, small, R), R) for k, x in d.items()}
    assert sorted(rows) == [1, 2] and len(rows[1]) == 1 and len(rows[2]) == 4
    shs = shuffles(sc, sides[:1], 3) * 17
    assert sc._lib.vb_cogroup_n_size(_arr(shs), 17, 0, ctypes.byref(n), None) == L.VB_ERR_INVALID
    assert sc._lib.vb_join_n_size(_arr(shs), 17, 0, ctypes.byref(n)) == L.VB_ERR_INVALID
    assert sc._lib.vb_cogroup_n(_arr(shs), 17, 0, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    assert sc._lib.vb_join_n(_arr(shs), 17, 0, None, None, L.VB_HOST) == L.VB_ERR_INVALID


# ---- 5. the same shuffle twice: [a, b, a] -------------------------------------------------------------------------------
def test_same_shuffle_twice(sc):
    rng = np.random.default_rng(5)
    ka, va = rand_pairs(rng, 6000, 800, values="full")
    kb, vb_ = rand_pairs(rng, 5000, 1200)
    R = 4
    sa, sb = shuffles(sc, [(ka, va, 3), (kb, vb_, 2)], R)
    want = CN.ref_parts_n([(ka, va, 3), (kb, vb_, 2), (ka, va, 3)], R)
    got = abi_parts_n(sc, [sa, sb, sa], R)
    assert_parts_equal(got, want)
    assert all(x[0] == x[2] for d in got for x in d.values())
    assert_parts_equal(join_parts_n(sc, [sa, sb, sa], R), CN.join_of_parts(want))


# ---- 6. an empty side first, in the middle, last; every side empty ------------------------------------------------------
@pytest.mark.parametrize("empty", [(0,), (1,), (2,), (0, 1, 2)])
def test_empty_sides(sc, empty):
    rng = np.random.default_rng(6)
    e = np.empty(0, dtype=np.uint64)
    sides = []
    for j in range(3):
        k, v = rand_pairs(rng, 3000, 500)
        sides.append((e, e, 2) if j in empty else (k, v, 2 + j))
    got = check(sc, sides, 5)
    assert sum(len(d) for d in got) == len(set().union(*(set(k.tolist()) for k, _, _ in sides)))
    assert all(not x[j] for d in got for x in d.values() for j in empty)


# ---- 7. disjoint and identical sides ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["disjoint", "identical"])
def test_disjoint_and_identical(sc, case):
    rng = np.random.default_rng(7)
    k, v = rand_pairs(rng, 4000, 600)
    if case == "disjoint":      # the keys are ranks * odd + 12345: +1 / +2 never hit another key
        sides = [(k, v, 2), (k + np.uint64(1), v, 3), (k + np.uint64(2), v, 1)]
    else:
        sides = [(k, v, 2), (k.copy(), v.copy(), 3), (k.copy(), v.copy(), 1)]
    got = check(sc, sides, 4)
    lists = [x for d in got for x in d.values()]
    if case == "disjoint":
        assert all(sum(1 for y in x if y) == 1 for x in lists)
        assert all(not d for d in join_parts_n(sc, shuffles(sc, sides, 4), 4))
    else:
        assert all(x[0] == x[1] == x[2] for x in lists)


# ---- 8. 4-byte keys ---------------------------------------------------------------------------------------------------------
def test_int32_keys(sc):
    rng = np.random.default_rng(8)
    ks = [rng.integers(-2000, 1000, 20_000).astype(np.int32), rng.integers(0, 3000, 15_000).astype(np.int32),
          rng.integers(-500, 2500, 9000).astype(np.int32)]
    ks[0][:3] = [-1, -(1 << 31), (1 << 31) - 1]
    ks[2][:2] = [(1 << 31) - 1, -(1 << 31)]
    sides = [(k, rng.integers(0, 1 << 40, len(k)).astype(np.uint64), M) for k, M in zip(ks, (3, 2, 4))]
    check(sc, sides, 6, key_width=4)


# ---- 9. u64 / i64 / f64 values on different sides, bit for bit, through the mirror -------------------------------------------
def test_mixed_value_dtypes(sc):
    rng = np.random.default_rng(9)
    ka, va = rand_pairs(rng, 9000, 1500, vdtype="u64", values="full")
    kb, vb_ = rand_pairs(rng, 8000, 2000, vdtype="i64", values="full")
    kc, vc = rand_pairs(rng, 7000, 1800, vdtype="f64", values="special")
    R = 5
    cg = vb.CoGroupedRdd([sc.parallelize((ka, va), 3), sc.parallelize((kb, vb_), 2), sc.parallelize((kc, vc), 4)], R)
    want = CN.ref_parts_n([(ka, va, 3), (kb, vb_, 2), (kc, vc, 4)], R)
    got = []
    for r in range(R):
        keys, lists = cg.compute(r)
        assert [v.dtype for _, v in lists] == [np.uint64, np.int64, np.float64] and keys.dtype == np.uint64
        got.append(part_dict_n(keys, [o for o, _ in lists], [v for _, v in lists], r, R))
    assert_parts_equal(got, want)
    k, vs = cg.join_collect()
    assert [v.dtype for v in vs] == [np.uint64, np.int64, np.float64]
    got_j = join_by_key(k, vs)
    want_j = {kk: rows for d in CN.join_of_parts(want) for kk, rows in d.items()}
    assert got_j == want_j


# ---- 10. R = 1, and more partitions than keys ------------------------------------------------------------------------------
@pytest.mark.parametrize("R,nkeys", [(1, 500), (300, 100)])
def test_partition_counts(sc, R, nkeys):
    rng = np.random.default_rng(R)
    sides = [(*rand_pairs(rng, n, nkeys + 50 * j), M) for j, (n, M) in enumerate(((2000, 2), (1500, 3), (1000, 1)))]
    got = check(sc, sides, R)
    if R == 300:
        assert sum(1 for d in got if not d) >= 100


# ---- 11. one key with 10^6 values on the middle side ------------------------------------------------------------------------
def test_skewed_middle_side(sc):
    rng = np.random.default_rng(11)
    hot = np.uint64(0xDEADBEEF12345)
    ka, va = rand_pairs(rng, 20_000, 4000)
    kb, vb_ = rand_pairs(rng, 50_000, 6000)
    kc, vc = rand_pairs(rng, 10_000, 3000)
    ka = np.concatenate([ka, np.full(2, hot, dtype=np.uint64)])
    va = np.concatenate([va, np.array([1, 2], dtype=np.uint64)])
    kb = np.concatenate([np.full(1_000_000, hot, dtype=np.uint64), kb])
    vb_ = np.concatenate([np.arange(1_000_000, dtype=np.uint64) * np.uint64(3) + np.uint64(1), vb_])
    perm = rng.permutation(len(kb))
    kb, vb_ = kb[perm], vb_[perm]
    kc = np.concatenate([kc, np.full(3, hot, dtype=np.uint64)])
    vc = np.concatenate([vc, np.array([7, 8, 9], dtype=np.uint64)])
    R = 4
    got = check(sc, [(ka, va, 3), (kb, vb_, 4), (kc, vc, 2)], R)
    hot_lists = [d[int(hot)] for d in got if int(hot) in d]
    assert len(hot_lists) == 1 and hot_lists[0][0] == [1, 2] and len(hot_lists[0][1]) == 1_000_000
    assert hot_lists[0][2] == [7, 8, 9]


# ---- 12. three sides of 5e6 rows against numpy triples ----------------------------------------------------------------------
def test_large_three_sides(sc):
    n, R = 5_000_000, 8
    rng = np.random.default_rng(12)
    sides, ranks = [], []
    for nk in (2_000_000, 3_000_000, 1_000_000):       # overlapping key ranges: keys on one, two or three sides
        rk = rng.integers(0, nk, n)
        ranks.append(rk)
        sides.append((rk.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15), rng.integers(0, 1 << 63, n, dtype=np.uint64)))
    cg = vb.CoGroupedRdd([sc.parallelize((k, v), 8) for k, v in sides], R)
    CN.assert_cogroup_n_equal([cg.compute(r) for r in range(R)], sides, R)
    # the join has a row count of sum over keys of the product of the three counts (the keys of rank < 1e6)
    counts = [np.bincount(rk, minlength=3_000_000)[:1_000_000] for rk in ranks]
    want_rows = int((counts[0] * counts[1] * counts[2]).sum())
    rows = ctypes.c_uint64()
    shs = cg._run()
    got_rows = 0
    for r in range(R):
        L.check(sc._lib.vb_join_n_size(_arr(shs), 3, r, ctypes.byref(rows)))
        got_rows += rows.value
    assert got_rows == want_rows


# ---- 13. VB_DEVICE output equals VB_HOST output; NULL outputs are skipped ----------------------------------------------------
def test_device_output_equals_host_and_null_outputs(sc):
    rng = np.random.default_rng(13)
    sides = [(*rand_pairs(rng, n, nk), M) for n, nk, M in ((8000, 900, 3), (6000, 1200, 2), (4000, 700, 1))]
    R = 4
    shs = shuffles(sc, sides, R)
    lib = sc._lib
    for r in range(R):
        host, dev = abi_cogroup_n(sc, shs, r, L.VB_HOST), abi_cogroup_n(sc, shs, r, L.VB_DEVICE)
        assert np.array_equal(host[0], dev[0])
        for h, d in zip(host[1] + host[2], dev[1] + dev[2]):
            assert np.array_equal(h, d)
        hk, hv = abi_join_n(sc, shs, r, L.VB_HOST)
        dk, dv = abi_join_n(sc, shs, r, L.VB_DEVICE)
        assert np.array_equal(hk, dk) and all(np.array_equal(a, b) for a, b in zip(hv, dv))
    full = abi_cogroup_n(sc, shs, 1)
    nk = ctypes.c_uint64()
    L.check(lib.vb_cogroup_n_size(_arr(shs), 3, 1, ctypes.byref(nk), None))
    assert nk.value == len(full[0])
    # only side 2's offsets and side 1's values; then keys alone with both arrays NULL
    o2 = np.zeros(nk.value + 1, dtype=np.uint64)
    v1 = np.zeros(len(full[2][1]), dtype=np.uint64)
    offs = (ctypes.c_void_p * 3)(None, None, o2.ctypes.data)
    vals = (ctypes.c_void_p * 3)(None, v1.ctypes.data, None)
    L.check(lib.vb_cogroup_n(_arr(shs), 3, 1, None, offs, vals, L.VB_HOST))
    assert np.array_equal(o2, full[1][2]) and np.array_equal(v1, full[2][1])
    keys = np.zeros(nk.value, dtype=np.uint64)
    L.check(lib.vb_cogroup_n_size(_arr(shs), 3, 1, None, None))
    L.check(lib.vb_cogroup_n(_arr(shs), 3, 1, keys.ctypes.data, None, None, L.VB_HOST))
    assert np.array_equal(keys, full[0])


# ---- 14. the N-way calls, then vb_cogroup / vb_join / vb_join_outer on the same shuffles -------------------------------------
def test_then_binary_calls_on_the_same_shuffles(sc):
    rng = np.random.default_rng(14)
    ka, va = rand_pairs(rng, 12_000, 1500, values="full")
    kb, vb_ = rand_pairs(rng, 9000, 2500, values="full")
    kc, vc = rand_pairs(rng, 5000, 1000)
    R = 4
    sa, sb, s_c = shuffles(sc, [(ka, va, 3), (kb, vb_, 2), (kc, vc, 2)], R)
    assert_parts_equal(abi_parts_n(sc, [sa, sb, s_c], R), CN.ref_parts_n([(ka, va, 3), (kb, vb_, 2), (kc, vc, 2)], R))
    join_parts_n(sc, [sa, sb, s_c], R)
    fa, fb = shuffles(sc, [(ka, va, 3), (kb, vb_, 2)], R)
    assert abi_parts(sc, sa, sb, R) == abi_parts(sc, fa, fb, R)
    fa, fb = shuffles(sc, [(ka, va, 3), (kb, vb_, 2)], R)
    assert [by_key(*abi_rows(sc, sa, sb, r, None)) for r in range(R)] == [by_key(*abi_rows(sc, fa, fb, r, None)) for r in range(R)]
    got_full = [by_key(*abi_rows(sc, sa, sb, r, "full")) for r in range(R)]
    assert_parts_equal(got_full, outer_join_parts("full", ka, va, 3, kb, vb_, 2, R))
    for s_, k, v, M in ((sa, ka, va, 3), (sb, kb, vb_, 2), (s_c, kc, vc, 2)):
        got = []
        for r in range(R):
            keys, offs, vals = s_.reduce(r)
            o, vals = offs.tolist(), _u64(vals).tolist()
            got.append({int(x): vals[o[i]:o[i + 1]] for i, x in enumerate(_u64(keys).tolist())})
        assert_parts_equal(got, _group(k, v, M, R, 8))


# ---- 15. joins: partial keys give no rows; 2^63 rows are VB_ERR_TOO_LARGE -----------------------------------------------------
def test_join_partial_keys_give_no_rows(sc):
    u = lambda *x: np.array(x, dtype=np.uint64)
    sides = [(u(1, 2, 3, 1), u(10, 20, 30, 11), 2), (u(1, 2, 4), u(100, 200, 400), 1), (u(1, 3, 4, 1), u(1000, 3000, 4000, 1001), 2)]
    R = 2
    shs = shuffles(sc, sides, R)
    rows = {k: r for d in join_parts_n(sc, shs, R) for k, r in d.items()}
    assert rows == {1: [(10, 100, 1000), (10, 100, 1001), (11, 100, 1000), (11, 100, 1001)]}
    assert sorted(k for k, _ in vb.CoGroupedRdd([sc.parallelize((k, v), M) for k, v, M in sides], R).collect()) == [1, 2, 3, 4]


@pytest.mark.parametrize("shape", ["one_key", "partition_total"])
def test_join_too_large(sc, shape):
    """One key with 2^21 values on each of three sides: 2^63 rows.  Or two keys of one partition with 2^21, 2^21 and
    2^20 values: 2^62 rows each, 2^63 in total.  Both are refused by the size call, and the shuffles still work."""
    R = 1                                   # (key, values) per side; every key in the one partition
    if shape == "one_key":
        per_side = [[(5, 1 << 21)]] * 3
    else:
        per_side = [[(5, 1 << 21), (6, 1 << 21)], [(5, 1 << 21), (6, 1 << 21)], [(5, 1 << 20), (6, 1 << 20)]]
    sides = []
    for pairs in per_side:
        k = np.concatenate([np.full(m, key, dtype=np.uint64) for key, m in pairs])
        sides.append((k, np.arange(len(k), dtype=np.uint64), 2))
    shs = shuffles(sc, sides, R)
    n = ctypes.c_uint64(12345)
    assert sc._lib.vb_join_n_size(_arr(shs), 3, 0, ctypes.byref(n)) == L.VB_ERR_TOO_LARGE
    assert n.value == 12345
    assert "2^63" in sc._lib.vb_last_error().decode()
    # the first two sides still give a join size (2^42 rows per key), and the cogroup of all three works
    L.check(sc._lib.vb_join_n_size(_arr(shs[:2]), 2, 0, ctypes.byref(n)))
    assert n.value == sum(m * m for _, m in per_side[0])
    keys, offs, vals = abi_cogroup_n(sc, shs, 0)
    assert sorted(keys.tolist()) == [key for key, _ in per_side[0]]
    assert [len(v) for v in vals] == [len(k) for k, _, _ in sides]


# ---- 16. rejected calls; the shuffles still work afterwards --------------------------------------------------------------------
def test_rejected_calls(sc):
    rng = np.random.default_rng(16)
    ka, va = rand_pairs(rng, 500, 50)
    sa, sb = shuffles(sc, [(ka, va, 2), (ka, va, 2)], 3)
    lib, n = sc._lib, ctypes.c_uint64()
    size = lambda shs, r=0, m=None: lib.vb_cogroup_n_size(_arr(shs) if shs is not None else None,
                                                          len(shs) if m is None else m, r, ctypes.byref(n), None)
    write = lambda shs, r=0, dst=L.VB_HOST, m=None: lib.vb_cogroup_n(_arr(shs) if shs is not None else None,
                                                                     len(shs) if m is None else m, r, None, None, None, dst)
    jsize = lambda shs, r=0, m=None: lib.vb_join_n_size(_arr(shs) if shs is not None else None,
                                                        len(shs) if m is None else m, r, ctypes.byref(n))
    jwrite = lambda shs, r=0, dst=L.VB_HOST, m=None: lib.vb_join_n(_arr(shs) if shs is not None else None,
                                                                   len(shs) if m is None else m, r, None, None, dst)
    calls = (size, write, jsize, jwrite)
    for f in calls:
        assert f(None, m=2) == L.VB_ERR_INVALID                         # NULL sides array
        assert f([sa, None]) == L.VB_ERR_INVALID                        # NULL entry
        assert f([None, sa]) == L.VB_ERR_INVALID
        assert f([sa, sb], m=0) == L.VB_ERR_INVALID                     # no side
        assert f([sa, sb], r=3) == L.VB_ERR_INVALID                     # reduce_id >= n_reduce
    for f in (write, jwrite):
        assert f([sa, sb], dst=5) == L.VB_ERR_INVALID and f([sa, sb], dst=-1) == L.VB_ERR_INVALID
    assert lib.vb_join_n_size(_arr([sa, sb]), 2, 0, None) == L.VB_ERR_INVALID
    other_ctx = vb.Context(0)
    try:
        others = {
            "n_reduce": shuffles(sc, [(ka, va, 2)], 4)[0],
            "key width": shuffles(sc, [(ka.astype(np.int32), va, 2)], 3)[0],
            "SUM": sc.parallelize((ka, va), 2).reduce_by_key("sum", 3)._run(),
            "combine_by_key": sc.parallelize(ka, 2, values=(va,)).combine_by_key({"n": ("count", None)}, 3)._run(),
            "string": sc.parallelize([str(x) for x in range(50)], 2, values=np.arange(50, dtype=np.uint64)).group_by_key(3)._run(),
            "context": shuffles(other_ctx, [(ka, va, 2)], 3)[0],
        }
        for what, o in others.items():
            for shs in ([sa, o], [o, sa], [sa, sb, o]):
                for f in calls:
                    assert f(shs) == L.VB_ERR_INVALID, what
        # a join partition with rows needs every output
        rows = ctypes.c_uint64()
        L.check(lib.vb_join_n_size(_arr([sa, sb]), 2, 0, ctypes.byref(rows)))
        assert rows.value > 0
        k = np.zeros(rows.value, dtype=np.uint64)
        assert lib.vb_join_n(_arr([sa, sb]), 2, 0, k.ctypes.data, (ctypes.c_void_p * 2)(k.ctypes.data, None), L.VB_HOST) == L.VB_ERR_INVALID
        assert lib.vb_join_n(_arr([sa, sb]), 2, 0, None, (ctypes.c_void_p * 2)(k.ctypes.data, k.ctypes.data), L.VB_HOST) == L.VB_ERR_INVALID
        for s_ in others.values():
            s_.free()
    finally:
        other_ctx.close()
    # the valid calls still work after the rejections
    want = CN.ref_parts_n([(ka, va, 2), (ka, va, 2)], 3)
    assert_parts_equal(abi_parts_n(sc, [sa, sb], 3), want)
    assert_parts_equal(join_parts_n(sc, [sa, sb], 3), CN.join_of_parts(want))


# ---- 17. the mirror: collect / join_collect on the reference's tests/test_rdd.rs data with a third parent ----------------------
def test_mirror_collect_and_join_collect(sc):
    names = ["A", "B", "C", "D", "X", "Y", "Z"]
    k = np.array([1, 2, 3, 4], dtype=np.int32)
    v = np.arange(4, dtype=np.uint64)
    k3, v3 = np.array([4, 5, 4], dtype=np.int32), np.array([4, 5, 6], dtype=np.uint64)
    cg = vb.CoGroupedRdd([sc.parallelize((k, v), 2), sc.parallelize((k, v), 2), sc.parallelize((k3, v3), 2)], 2)
    got = sorted((a, [[names[i] for i in x.tolist()] for x in ls]) for a, ls in cg.collect())
    rows = [(1, "A"), (2, "B"), (3, "C"), (4, "D")]
    want = sorted(CN.cogroup_n([(rows, 2), (rows, 2), ([(4, "X"), (5, "Y"), (4, "Z")], 2)], 2, int_width=4))
    assert got == want
    jk, jv = cg.join_collect()
    got_j = [(a, [names[x[i]] for x in jv]) for i, a in enumerate(jk.tolist())]
    assert got_j == CN.join_n([(rows, 2), (rows, 2), ([(4, "X"), (5, "Y"), (4, "Z")], 2)], 2, int_width=4)


def test_cpp_cogroup_n_example_runs():
    """examples/cogroup_n.cpp: three parents on hand-written data, cogroup and join; exit 0 only on the expected result."""
    path = os.path.join(ROOT, "examples", "_build", "cogroup_n")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    out = subprocess.run([path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "(1, [[10, 11], [100, 101], [1000]])" in out.stdout, out.stdout
    assert "join: [(1, [10, 100, 1000]), (1, [10, 101, 1000]), (1, [11, 100, 1000]), (1, [11, 101, 1000])]" in out.stdout, out.stdout


# ---- 18. two ranks: only the owned partitions have keys --------------------------------------------------------------------------
def _dist_data():
    rng = np.random.default_rng(18)
    out = []
    for lo, hi, n in ((0, 4000, 60_000), (2000, 7000, 45_000), (3000, 5000, 30_000)):
        k = rng.integers(lo, hi, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)
        out.append((k, rng.integers(0, 1 << 50, n).astype(np.uint64)))
    return out


def _dist_worker(rank, world, port, Ms, R, outdir):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    from vega_b200 import dist as vdist
    sc = vb.Context(rank)
    sc.comm_init(rank, world)
    eng = vdist.CudaEngine(sc)
    shs = []
    for (keys, vals), M in zip(_dist_data(), Ms):
        starts = vb.slice_starts(len(keys), M)
        lo, hi = vdist.map_block(rank, world, M)
        maps = [(m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]]) for m in range(lo, hi)]
        shs.append(vdist.run_shuffle(eng, maps, M, R, 0, 0, L.VB_AGG_COGROUP, rank, world))
    res = (abi_parts_n(sc, shs, R), join_parts_n(sc, shs, R))
    with open(os.path.join(outdir, f"o{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    for s in shs:
        s.free()
    sc.close()
    dist.destroy_process_group()


def test_two_ranks():
    import socket
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    world, Ms, R = 2, (4, 2, 3), 6
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_dist_worker, args=(world, port, Ms, R, d), nprocs=world, join=True)
        per_rank = [pickle.load(open(os.path.join(d, f"o{r}.pkl"), "rb")) for r in range(world)]
    want = CN.ref_parts_n([(k, v, M) for (k, v), M in zip(_dist_data(), Ms)], R)
    want_j = CN.join_of_parts(want)
    for r in range(R):
        owner = r % world
        assert per_rank[owner][0][r] == want[r] and per_rank[owner][1][r] == want_j[r], f"partition {r}"
        assert per_rank[1 - owner][0][r] == {} and per_rank[1 - owner][1][r] == {}, f"partition {r} on a rank that does not own it"
