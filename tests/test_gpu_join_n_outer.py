"""GPU outer join of any number of shuffles (vb_join_n_outer, CoGroupedRdd.outer_join_compute / outer_join_collect,
PairRddT::join_n_outer) against the restatement over each side's C-oracle group shuffle (tests/join_n_outer_ref.py), and
against vb_join and vb_join_outer at two sides.  Every partition is checked row by row: each key's rows are contiguous,
in nested order, with the values and validity bytes of the reference, and every key is in its own partition."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import vega_b200 as vb
from oracle import oracle as O
from tests import cogroup_n_ref as CN
from tests import join_n_outer_ref as JO
from tests import outer_join_ref as OJ
from tests.test_gpu_outer_join import abi_rows, by_key
from tests.util import assert_parts_equal, rand_pairs
from vega_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = 0x9E3779B97F4A7C15


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
    for s in shs:
        for r in range(R):
            s.reduce(r)


def _arr(shs):
    return (ctypes.c_void_p * len(shs))(*[s._h.value if s is not None else None for s in shs])


def _buf(n, dtype, dst, fill):
    if dst == L.VB_HOST:
        return np.full(n, fill, dtype=dtype)
    import torch
    return torch.full((n,), fill, dtype=torch.int64 if dtype == np.uint64 else torch.uint8, device="cuda")


def _ptr(x):
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    return x.data_ptr() if x.numel() else None


def _host(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def abi_outer(sc, shs, r, required, dst=L.VB_HOST, valid=None):
    """One partition of vb_join_n_outer: (k, [v per side], [validity per side]) as host arrays.  valid: the sides whose
    validity array is passed (default every side); None entries come back for the others."""
    lib, n = sc._lib, len(shs)
    rows = ctypes.c_uint64()
    L.check(lib.vb_join_n_outer_size(_arr(shs), n, r, required, ctypes.byref(rows)))
    want_valid = range(n) if valid is None else valid
    if dst != L.VB_HOST:
        import torch
        torch.cuda.synchronize()
    k = _buf(rows.value, np.uint64, dst, 7)
    vs = [_buf(rows.value, np.uint64, dst, 7) for _ in range(n)]
    oks = [_buf(rows.value, np.uint8, dst, 7) if j in want_valid else None for j in range(n)]
    L.check(lib.vb_join_n_outer(_arr(shs), n, r, required, _ptr(k), (ctypes.c_void_p * n)(*[_ptr(v) for v in vs]),
                                (ctypes.c_void_p * n)(*[_ptr(x) for x in oks]), dst))
    return _u64(_host(k)), [_u64(_host(v)) for v in vs], [None if x is None else _host(x) for x in oks]


def rows_by_key(k, vs, oks):
    """{key: [(v_0, ..., v_{n-1}, valid_0, ..., valid_{n-1}), ...]} in output order; a key's rows must be contiguous."""
    d, prev = {}, None
    for row in zip(_u64(k).tolist(), *[v.tolist() for v in vs], *[np.asarray(x).tolist() for x in oks]):
        if row[0] != prev:
            assert row[0] not in d, f"the rows of key {row[0]:#x} are not contiguous"
            d[row[0]], prev = [], row[0]
        d[row[0]].append(row[1:])
    return d


def outer_parts(sc, shs, R, required, key_width=8):
    out = []
    for r in range(R):
        d = rows_by_key(*abi_outer(sc, shs, r, required))
        assert all(O.get_partition(k, R, key_width) == r for k in d), f"a key outside partition {r}"
        out.append(d)
    return out


def check(sc, sides, R, masks, key_width=8, shs=None):
    """Every mask on one set of shuffles of the sides against the reference; returns {mask: parts}."""
    ref = CN.ref_parts_n(sides, R, key_width)
    shs = shs if shs is not None else shuffles(sc, sides, R)
    got = {}
    for m in masks:
        got[m] = outer_parts(sc, shs, R, m, key_width)
        assert_parts_equal(got[m], JO.outer_of_parts(ref, m))
    return got


# ---- 1. one, two and three sides, every mask ------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3])
def test_every_mask(sc, n):
    rng = np.random.default_rng(n)
    sides = []
    for j, (rows, nkeys, M) in enumerate(((12_000, 1500, 3), (9000, 2000, 2), (6000, 1200, 4))[:n]):
        k, v = rand_pairs(rng, rows, nkeys, values="full")      # keys 0 and 2^64-1 among them
        keep = (k >> np.uint64(7)) % np.uint64(4) != np.uint64(j)   # a quarter of the keys lack side j
        sides.append((k[keep], v[keep], M))
    got = check(sc, sides, 4, range(1 << n))
    oks = {row[n:] for rows in (r for d in got[0] for r in d.values()) for row in rows}
    assert (1,) * n in oks and (n == 1 or len(oks) > 2)


# ---- 2. five and sixteen sides ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,masks", [(5, [0, 1, 0b10101, 0b11111, 0b10000]), (16, [0, 1, 0x8000, 0xFFFF, 0x0F0F])])
def test_many_sides(sc, n, masks):
    rng = np.random.default_rng(n)
    sides = []
    for j in range(n):                        # about one value per key and side, so 16-way products stay small
        k, v = rand_pairs(rng, 30 + 3 * j, 60)
        sides.append((k, v, 1 + j % 3))
    got = check(sc, sides, 3, masks)
    assert sum(len(d) for d in got[0]) > sum(len(d) for d in got[masks[1]])


# ---- 3. two sides: vb_join and vb_join_outer LEFT / RIGHT / FULL, on lazy and on grouped sides --------------------------
@pytest.mark.parametrize("grouped", [False, True])
def test_two_sides_match_the_two_side_joins(sc, grouped):
    rng = np.random.default_rng(3)
    ka, va = rand_pairs(rng, 15_000, 2000, values="full")
    kb, vb_ = rand_pairs(rng, 10_000, 3000, values="full")
    keep = kb % np.uint64(5) != 0                             # keys only on the left as well as only on the right
    kb, vb_ = kb[keep], vb_[keep]
    R = 4
    sides = [(ka, va, 3), (kb, vb_, 2)]
    if grouped:
        shs = shuffles(sc, sides, R)
        group_all(shs, R)
        pair = lambda: shs
    else:
        pair = lambda: shuffles(sc, sides, R)                 # fresh lazy shuffles for every call
    for mask, kind in ((0b11, None), (0b01, "left"), (0b10, "right"), (0b00, "full")):
        sa, sb = pair()
        want = [by_key(*abi_rows(sc, sa, sb, r, kind)) for r in range(R)]
        got = outer_parts(sc, pair(), R, mask)
        assert got == want, kind
        assert_parts_equal(got, JO.outer_of_parts(CN.ref_parts_n(sides, R), mask))


# ---- 4. empty sides; disjoint and identical key sets; the same shuffle twice; 4-byte keys --------------------------------
@pytest.mark.parametrize("empty", [(0,), (1,), (2,), (0, 1, 2)])
def test_empty_sides(sc, empty):
    rng = np.random.default_rng(4)
    e = np.empty(0, dtype=np.uint64)
    sides = [(e, e, 2) if j in empty else (*rand_pairs(rng, 3000, 500), 2 + j) for j in range(3)]
    got = check(sc, sides, 5, range(8))
    for m in range(8):
        n_rows = sum(len(rows) for d in got[m] for rows in d.values())
        assert (n_rows == 0) == (len(empty) == 3 or any(m >> j & 1 for j in empty))


@pytest.mark.parametrize("case", ["disjoint", "identical"])
def test_disjoint_and_identical(sc, case):
    rng = np.random.default_rng(5)
    k, v = rand_pairs(rng, 4000, 600)
    if case == "disjoint":      # the keys are ranks * odd + 12345: +1 / +2 never hit another key
        sides = [(k, v, 2), (k + np.uint64(1), v, 3), (k + np.uint64(2), v, 1)]
    else:
        sides = [(k, v, 2), (k.copy(), v.copy(), 3), (k.copy(), v.copy(), 1)]
    got = check(sc, sides, 4, range(8))
    all_rows = lambda m: [row for d in got[m] for rows in d.values() for row in rows]
    if case == "disjoint":      # a key gives rows only with at most one required side; each row has one valid side
        assert all(not all_rows(m) for m in (3, 5, 6, 7))
        assert all(sum(row[3:]) == 1 for row in all_rows(0)) and len(all_rows(0)) == 3 * len(k)
    else:                       # every mask is the inner join
        assert all(all_rows(m) == all_rows(7) for m in range(7))


def test_same_shuffle_twice(sc):
    rng = np.random.default_rng(6)
    ka, va = rand_pairs(rng, 6000, 800, values="full")
    kb, vb_ = rand_pairs(rng, 5000, 1200)
    R = 4
    sa, sb = shuffles(sc, [(ka, va, 3), (kb, vb_, 2)], R)
    check(sc, [(ka, va, 3), (kb, vb_, 2), (ka, va, 3)], R, range(8), shs=[sa, sb, sa])


def test_int32_keys(sc):
    rng = np.random.default_rng(7)
    ks = [rng.integers(-2000, 1000, 20_000).astype(np.int32), rng.integers(0, 3000, 15_000).astype(np.int32),
          rng.integers(-500, 2500, 9000).astype(np.int32)]
    ks[0][:3] = [-1, -(1 << 31), (1 << 31) - 1]
    ks[2][:2] = [(1 << 31) - 1, -(1 << 31)]
    sides = [(k, rng.integers(0, 1 << 40, len(k)).astype(np.uint64), M) for k, M in zip(ks, (3, 2, 4))]
    check(sc, sides, 6, range(8), key_width=4)


# ---- 5. about 10^7 rows with a skewed key, checked with numpy -------------------------------------------------------------
def test_large_skewed(sc):
    """Three sides over overlapping key ranges; one hot key with 3000 values on side 0 and 1000 on side 1 (absent on
    side 2).  Values are row indices, so a value names its row: every valid slot must hold a row of its key, each key
    must give prod max(count, 1) rows, contiguous and strictly increasing (the nested order of the increasing lists)."""
    rng = np.random.default_rng(8)
    hot, R = 5_000_000, 8
    ranks = []
    for lo, hi, n, extra in ((0, 1_500_000, 3_000_000, 3000), (1_000_000, 2_500_000, 2_000_000, 1000),
                             (2_000_000, 3_000_000, 1_000_000, 0)):
        rk = np.concatenate([rng.integers(lo, hi, n), np.full(extra, hot)])
        ranks.append(rng.permutation(rk))
    keys = [rk.astype(np.uint64) * np.uint64(GOLD) + np.uint64(12345) for rk in ranks]
    cg = vb.CoGroupedRdd([sc.parallelize((k, np.arange(len(k), dtype=np.uint64)), 4) for k in keys], R)
    shs = cg._run()
    inv = np.uint64(pow(GOLD, -1, 1 << 64))
    cnt = [np.bincount(rk, minlength=hot + 1) for rk in ranks]
    for mask in (0b001, 0):
        parts = [abi_outer(sc, shs, r, mask) for r in range(R)]
        k = np.concatenate([p[0] for p in parts])
        vs = [np.concatenate([p[1][j] for p in parts]) for j in range(3)]
        oks = [np.concatenate([p[2][j] for p in parts]) for j in range(3)]
        kept = np.ones(hot + 1, dtype=bool) if mask == 0 else cnt[0] > 0
        kept &= (cnt[0] > 0) | (cnt[1] > 0) | (cnt[2] > 0)
        want = np.where(kept, np.maximum(cnt[0], 1) * np.maximum(cnt[1], 1) * np.maximum(cnt[2], 1), 0)
        assert len(k) == int(want.sum()) and len(k) > 5_000_000
        rk = ((k - np.uint64(12345)) * inv).astype(np.int64)
        assert (rk <= hot).all()
        assert np.array_equal(np.bincount(rk, minlength=hot + 1), want)
        for j in range(3):
            ok = oks[j].astype(bool)
            assert set(np.unique(oks[j]).tolist()) <= {0, 1}
            assert np.array_equal(ok, cnt[j][rk] > 0), f"side {j}: validity"
            assert (vs[j][~ok] == 0).all(), f"side {j}: a None slot does not hold 0"
            assert np.array_equal(keys[j][vs[j][ok].astype(np.int64)], k[ok]), f"side {j}: a value of another key"
        starts = np.flatnonzero(np.r_[True, rk[1:] != rk[:-1]])
        assert len(starts) == int((want > 0).sum()), "a key's rows are not contiguous"
        same = rk[1:] == rk[:-1]
        gt, eq = np.zeros(len(k) - 1, dtype=bool), np.ones(len(k) - 1, dtype=bool)
        for j in range(3):
            a, b = vs[j][:-1], vs[j][1:]
            gt |= eq & (b > a)
            eq &= b == a
        assert gt[same].all(), "a key's rows are not in nested order"
        for r, p in enumerate(parts):
            u = np.unique(p[0])
            assert len(u) and (OJ.key_partitions(u, R) == r).all(), f"a key outside partition {r}"
        if mask == 0b001:
            assert want[hot] == 3_000_000


# ---- 6. VB_DEVICE output equals VB_HOST output; NULL validity entries -------------------------------------------------------
def test_device_output_equals_host_and_null_validity(sc):
    rng = np.random.default_rng(9)
    sides = [(*rand_pairs(rng, n, nk), M) for n, nk, M in ((8000, 900, 3), (6000, 1200, 2), (4000, 700, 1))]
    R = 4
    shs = shuffles(sc, sides, R)
    for m in (0, 0b010, 0b111):
        for r in range(R):
            hk, hv, ho = abi_outer(sc, shs, r, m, L.VB_HOST)
            dk, dv, do = abi_outer(sc, shs, r, m, L.VB_DEVICE)
            assert np.array_equal(hk, dk)
            assert all(np.array_equal(a, b) for a, b in zip(hv + ho, dv + do))
            for dst in (L.VB_HOST, L.VB_DEVICE):        # only side 1's validity; then no validity array at all
                k1, v1, o1 = abi_outer(sc, shs, r, m, dst, valid=[1])
                assert np.array_equal(k1, hk) and all(np.array_equal(a, b) for a, b in zip(v1, hv))
                assert o1[0] is None and o1[2] is None and np.array_equal(o1[1], ho[1])
            rows = ctypes.c_uint64()
            L.check(sc._lib.vb_join_n_outer_size(_arr(shs), 3, r, m, ctypes.byref(rows)))
            k = np.zeros(rows.value, dtype=np.uint64)
            vs = [np.zeros(rows.value, dtype=np.uint64) for _ in range(3)]
            L.check(sc._lib.vb_join_n_outer(_arr(shs), 3, r, m, k.ctypes.data, (ctypes.c_void_p * 3)(*[v.ctypes.data for v in vs]),
                                            None, L.VB_HOST))
            assert np.array_equal(k, hk) and all(np.array_equal(a, b) for a, b in zip(vs, hv))


# ---- 7. size and write calls of different joins of the same shuffles, interleaved -------------------------------------------
def test_interleaved_plans(sc):
    """The plan kept between the size and the write call is keyed by the mask: the inner join's plan, the all-required
    outer join's and the full outer join's never stand in for each other."""
    rng = np.random.default_rng(10)
    sides = [(*rand_pairs(rng, n, nk), M) for n, nk, M in ((5000, 900, 3), (4000, 1200, 2))]
    R = 3
    shs = shuffles(sc, sides, R)
    want = {m: JO.outer_of_parts(CN.ref_parts_n(sides, R), m) for m in (0, 3)}
    lib = sc._lib
    for r in range(R):
        sizes = {}
        for m in (0, 3):
            n = ctypes.c_uint64()
            L.check(lib.vb_join_n_outer_size(_arr(shs), 2, r, m, ctypes.byref(n)))
            sizes[m] = n.value
        n = ctypes.c_uint64()
        L.check(lib.vb_join_n_size(_arr(shs), 2, r, ctypes.byref(n)))
        assert n.value == sizes[3] and sizes[0] >= sizes[3]
        inner = [np.zeros(n.value, dtype=np.uint64) for _ in range(3)]
        out = {m: ([np.zeros(sizes[m], dtype=np.uint64) for _ in range(3)], [np.zeros(sizes[m], dtype=np.uint8) for _ in range(2)])
               for m in (0, 3)}
        p2 = lambda xs: (ctypes.c_void_p * 2)(*[x.ctypes.data if len(x) else None for x in xs])
        for m in (0, 3):
            u, ok = out[m]
            L.check(lib.vb_join_n_outer(_arr(shs), 2, r, m, u[0].ctypes.data if len(u[0]) else None, p2(u[1:]), p2(ok), L.VB_HOST))
        L.check(lib.vb_join_n(_arr(shs), 2, r, inner[0].ctypes.data if len(inner[0]) else None, p2(inner[1:]), L.VB_HOST))
        for m in (0, 3):
            u, ok = out[m]
            assert rows_by_key(u[0], u[1:], ok) == want[m][r]
        assert rows_by_key(inner[0], inner[1:], [np.ones(n.value, np.uint8)] * 2) == want[3][r]


# ---- 8. 2^63 rows for one key or one partition are VB_ERR_TOO_LARGE ---------------------------------------------------------
@pytest.mark.parametrize("shape", ["one_key", "partition_total"])
def test_too_large(sc, shape):
    """One key with 2^21 values on each of three sides: 2^63 rows.  Or two keys with 2^21, 2^21 and 2^20 values: 2^62
    rows each, 2^63 in total.  A fourth, empty side adds a None slot (a factor of 1) when it is optional."""
    if shape == "one_key":
        per_side = [[(5, 1 << 21)]] * 3
    else:
        per_side = [[(5, 1 << 21), (6, 1 << 21)], [(5, 1 << 21), (6, 1 << 21)], [(5, 1 << 20), (6, 1 << 20)]]
    sides = []
    for pairs in per_side:
        k = np.concatenate([np.full(m, key, dtype=np.uint64) for key, m in pairs])
        sides.append((k, np.arange(len(k), dtype=np.uint64), 2))
    e = np.empty(0, dtype=np.uint64)
    shs = shuffles(sc, sides + [(e, e, 1)], 1)
    n = ctypes.c_uint64(12345)
    for sub, masks in ((shs[:3], (0, 0b001, 0b111)), (shs, (0, 0b0111))):
        for m in masks:
            assert sc._lib.vb_join_n_outer_size(_arr(sub), len(sub), 0, m, ctypes.byref(n)) == L.VB_ERR_TOO_LARGE, m
            assert n.value == 12345 and "2^63" in sc._lib.vb_last_error().decode()
    L.check(sc._lib.vb_join_n_outer_size(_arr(shs), 4, 0, 0b1000, ctypes.byref(n)))       # the empty side required
    assert n.value == 0
    L.check(sc._lib.vb_join_n_outer_size(_arr([shs[0], shs[3]]), 2, 0, 0, ctypes.byref(n)))
    assert n.value == sum(m for _, m in per_side[0])


# ---- 9. rejected calls; the shuffles still work afterwards ------------------------------------------------------------------
def test_rejected_calls(sc):
    rng = np.random.default_rng(11)
    ka, va = rand_pairs(rng, 500, 50)
    sa, sb = shuffles(sc, [(ka, va, 2), (ka, va, 2)], 3)
    lib, n = sc._lib, ctypes.c_uint64()
    size = lambda shs, r=0, m=0, cnt=None: lib.vb_join_n_outer_size(_arr(shs) if shs is not None else None,
                                                                   len(shs) if cnt is None else cnt, r, m, ctypes.byref(n))
    write = lambda shs, r=0, m=0, cnt=None, dst=L.VB_HOST: lib.vb_join_n_outer(
        _arr(shs) if shs is not None else None, len(shs) if cnt is None else cnt, r, m, None, None, None, dst)
    for f in (size, write):
        for bad in (4, 8, 1 << 16, 0x80000000, 0xFFFFFFFF):                       # a bit at n_sides or above
            assert f([sa, sb], m=bad) == L.VB_ERR_INVALID, bad
        assert f([sa] * 16, m=1 << 16) == L.VB_ERR_INVALID
        assert f(None, cnt=2) == L.VB_ERR_INVALID
        assert f([sa, None]) == L.VB_ERR_INVALID
        assert f([sa, sb], cnt=0) == L.VB_ERR_INVALID
        assert f([sa] * 17) == L.VB_ERR_INVALID
        assert f([sa, sb], r=3) == L.VB_ERR_INVALID
    assert write([sa, sb], dst=5) == L.VB_ERR_INVALID
    assert lib.vb_join_n_outer_size(_arr([sa, sb]), 2, 0, 0, None) == L.VB_ERR_INVALID
    others = {
        "SUM": sc.parallelize((ka, va), 2).reduce_by_key("sum", 3)._run(),
        "string": sc.parallelize([str(x) for x in range(50)], 2, values=np.arange(50, dtype=np.uint64)).group_by_key(3)._run(),
        "n_reduce": shuffles(sc, [(ka, va, 2)], 4)[0],
    }
    for what, o in others.items():
        for shs in ([sa, o], [o, sa]):
            assert size(shs) == L.VB_ERR_INVALID and write(shs) == L.VB_ERR_INVALID, what
    for s_ in others.values():
        s_.free()
    # a partition with rows needs out_k, out_vals and every entry of it
    L.check(lib.vb_join_n_outer_size(_arr([sa, sb]), 2, 0, 0, ctypes.byref(n)))
    assert n.value > 0
    k = np.zeros(n.value, dtype=np.uint64)
    two = lambda a, b: (ctypes.c_void_p * 2)(a, b)
    for out_k, out_vals in ((None, two(k.ctypes.data, k.ctypes.data)), (k.ctypes.data, None),
                            (k.ctypes.data, two(k.ctypes.data, None)), (k.ctypes.data, two(None, k.ctypes.data))):
        L.check(lib.vb_join_n_outer_size(_arr([sa, sb]), 2, 0, 0, ctypes.byref(n)))
        assert lib.vb_join_n_outer(_arr([sa, sb]), 2, 0, 0, out_k, out_vals, None, L.VB_HOST) == L.VB_ERR_INVALID
    want = CN.ref_parts_n([(ka, va, 2), (ka, va, 2)], 3)
    for m in range(4):
        assert_parts_equal(outer_parts(sc, [sa, sb], 3, m), JO.outer_of_parts(want, m))


# ---- 10. the mirror: masked arrays for the optional parents, each parent's dtype ----------------------------------------------
def test_mirror_outer_join_collect(sc):
    rng = np.random.default_rng(12)
    ka, va = rand_pairs(rng, 9000, 1500, vdtype="u64", values="full")
    kb, vb_ = rand_pairs(rng, 8000, 2000, vdtype="i64", values="full")
    kc, vc = rand_pairs(rng, 7000, 1800, vdtype="f64", values="special")
    R = 5
    sides = [(ka, va, 3), (kb, vb_, 2), (kc, vc, 4)]
    cg = vb.CoGroupedRdd([sc.parallelize((k, v), M) for k, v, M in sides], R)
    ref = CN.ref_parts_n(sides, R)
    for required, mask in (([0], 0b001), ((2, 1), 0b110), (0, 0), (range(3), 0b111)):
        k, vs = cg.outer_join_collect(required)
        assert [v.dtype for v in vs] == [np.uint64, np.int64, np.float64] and k.dtype == np.uint64
        assert [isinstance(v, np.ma.MaskedArray) for v in vs] == [not mask >> j & 1 for j in range(3)]
        data = [_u64(np.ma.getdata(v)) for v in vs]
        oks = [(~np.ma.getmaskarray(v)).astype(np.uint8) for v in vs]
        got = rows_by_key(k, data, oks)
        assert got == {kk: rows for d in JO.outer_of_parts(ref, mask) for kk, rows in d.items()}, required
        k1, vs1 = cg.outer_join_compute(1, required)
        assert rows_by_key(k1, [_u64(np.ma.getdata(v)) for v in vs1],
                           [(~np.ma.getmaskarray(v)).astype(np.uint8) for v in vs1]) == JO.outer_of_parts(ref, mask)[1]


def test_cpp_join_n_outer_example_runs():
    """examples/join_n_outer.cpp: a LEFT JOIN b LEFT JOIN c and the full outer join of three parents; exit 0 only on the
    expected rows."""
    path = os.path.join(ROOT, "examples", "_build", "join_n_outer")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    out = subprocess.run([path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "(2, [20, None, 2000]), (5, [50, None, None])]" in out.stdout, out.stdout
    assert "(3, [None, 300, 3000])" in out.stdout, out.stdout
