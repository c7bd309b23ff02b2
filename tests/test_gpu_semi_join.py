"""GPU semi and anti joins of any number of shuffles (vb_semi_join_n / vb_semi_join_n_str, PairRdd.subtract_by_key /
semi_join, CoGroupedRdd.semi_join_compute) against the restatement over each side's C-oracle group shuffle
(tests/semi_join_ref.py), partition by partition: each kept key's rows contiguous and in its side-0 list order, every key
in its own partition, and nothing else.  Also: vb_join_n_outer at two sides, lazy filter sides left ungrouped, a hot key,
String and Vec<u8> keys with crafted MetroHash collisions, several ranks in one process, and every refusal."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import vega_b200 as vb
from oracle import oracle as O
from tests import cogroup_n_ref as CN
from tests import metro_collide_ref as MC
from tests import semi_join_ref as SJ
from tests import slot_hash_ref as SH
from tests.multirank import maps_by_rank, run_ranks
from tests.test_gpu_join_n_outer import _arr, _host, _ptr, _u64, abi_outer, group_all, shuffles
from tests.test_gpu_str_collisions import key_col
from tests.util import assert_parts_equal, rand_pairs
from vega_b200 import _lib as L
from vega_b200 import dist as vdist

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def masks(n):
    return [(req, exc) for req in range(0, 1 << n, 2) for exc in range(0, 1 << n, 2) if not req & exc]


def abi_semi(sc, shs, r, req, exc, dst=L.VB_HOST):
    """One partition of vb_semi_join_n: (keys, values) as u64 host arrays."""
    lib, n = sc._lib, len(shs)
    rows = ctypes.c_uint64()
    L.check(lib.vb_semi_join_n_size(_arr(shs), n, r, req, exc, ctypes.byref(rows)))
    if dst == L.VB_HOST:
        k, v = np.full(rows.value, 7, np.uint64), np.full(rows.value, 7, np.uint64)
    else:
        k, v = (torch.full((rows.value,), 7, dtype=torch.int64, device="cuda") for _ in range(2))
    L.check(lib.vb_semi_join_n(_arr(shs), n, r, req, exc, _ptr(k), _ptr(v), dst))
    return _u64(_host(k)), _u64(_host(v))


def rows_by_key(keys, vals):
    """{key: [values]} in output order; a key's rows must be contiguous"""
    d, prev = {}, None
    for k, v in zip(keys.tolist(), vals.tolist()):
        if k != prev:
            assert k not in d, f"the rows of key {k:#x} are not contiguous"
            d[k], prev = [], k
        d[k].append(v)
    return d


def semi_parts(sc, shs, R, req, exc, key_width=8, dst=L.VB_HOST):
    out = []
    for r in range(R):
        d = rows_by_key(*abi_semi(sc, shs, r, req, exc, dst))
        assert all(O.get_partition(k, R, key_width) == r for k in d), f"a key outside partition {r}"
        out.append(d)
    return out


def check(sc, sides, R, pairs, key_width=8, shs=None):
    ref = CN.ref_parts_n(sides, R, key_width)
    shs = shs if shs is not None else shuffles(sc, sides, R)
    got = {}
    for req, exc in pairs:
        got[req, exc] = semi_parts(sc, shs, R, req, exc, key_width)
        assert_parts_equal(got[req, exc], SJ.semi_of_parts(ref, req, exc))
    return got


def n_rows(parts):
    return sum(len(l) for d in parts for l in d.values())


def grouping_launches(sh):
    return sh.stats()["kernels"]["dict"]["launches"]


# ---- 1. one to four sides, every (required, excluded) pair; five and sixteen sides, random pairs ----------------------
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_every_mask_pair(sc, n):
    rng = np.random.default_rng(n)
    sides = []
    for j in range(n):
        k, v = rand_pairs(rng, 6000 - 1000 * j, 1200, values="full")    # keys 0 and 2^64-1 among them
        keep = (k >> np.uint64(7)) % np.uint64(4) != np.uint64(j)         # a quarter of the keys lack side j
        sides.append((k[keep], v[keep], 1 + j % 3))
    got = check(sc, sides, 4, masks(n))
    assert n == 1 or 0 < n_rows(got[0, 0b10]) < n_rows(got[0, 0]) and 0 < n_rows(got[0b10, 0]) < n_rows(got[0, 0])


@pytest.mark.parametrize("n", [5, 16])
def test_many_sides(sc, n):
    rng = np.random.default_rng(n)
    sides = []
    for j in range(n):
        k, v = rand_pairs(rng, 400 + 20 * j, 300)
        sides.append((k, v, 1 + j % 3))
    pairs = [(0, 0), (0b10, 0), (0, 0b10), ((1 << n) - 2, 0), (0, (1 << n) - 2)]
    while len(pairs) < 12:
        req, exc = int(rng.integers(0, 1 << n)) & ~1, int(rng.integers(0, 1 << n)) & ~1
        pairs.append((req & ~exc, exc))
    check(sc, sides, 3, pairs)


# ---- 2. side kinds: lazy, grouped by a cogroup call, GROUP, narrow views; a side twice; empty sides and partitions -----
def test_grouped_and_group_sides(sc):
    rng = np.random.default_rng(11)
    sides = [(*rand_pairs(rng, 8000, 1500, values="full"), 3), (*rand_pairs(rng, 5000, 2500), 2), (*rand_pairs(rng, 3000, 800), 4)]
    R = 5
    shs = shuffles(sc, sides, R)
    group_all(shs[:1], R)                                     # side 0 grouped by a reduce, the filters still lazy
    check(sc, sides, R, masks(3), shs=shs)
    shs2 = shuffles(sc, sides, R)
    L.check(sc._lib.vb_cogroup_n_size(_arr(shs2), 3, 0, ctypes.byref(ctypes.c_uint64()), (ctypes.c_uint64 * 3)()))
    check(sc, sides, R, masks(3), shs=shs2)                   # every side grouped by vb_cogroup_n
    grp = [sc.parallelize((k, v), M).group_by_key(R)._run() for k, v, M in sides]
    check(sc, sides, R, masks(3), shs=grp)                    # GROUP shuffles
    mixed = [grp[0], shuffles(sc, sides[1:2], R)[0], grp[2]]
    check(sc, sides, R, masks(3), shs=mixed)


@pytest.mark.parametrize("side0", ["pair", "sum", "count", "combine"])
def test_narrow_views(sc, side0):
    rng = np.random.default_rng(12)
    k, v = rand_pairs(rng, 20_000, 3000)
    ks, vs = rand_pairs(rng, 4000, 1500)
    R = 6
    pair = sc.parallelize((k, v), 3)
    stop = sc.parallelize((ks, vs), 2)
    if side0 == "pair":
        a, others = pair, [stop.reduce_by_key("sum", R), stop.count_by_key(R),
                           stop.combine_by_key({"n": ("count", None), "m": ("max", 0)}, R).aggregate("m")]
    else:
        a = {"sum": pair.reduce_by_key("sum", R), "count": pair.count_by_key(R),
             "combine": pair.combine_by_key({"n": ("count", None), "s": ("sum", 0)}, R).aggregate("s")}[side0]
        others = [stop, stop.count_by_key(R)]
    for b in others:
        for method, has in (("subtract_by_key", False), ("semi_join", True)):
            got_k, got_v = getattr(a, method)(b, R).collect()
            stop_keys = set(ks.tolist())
            if side0 == "pair":
                want = sorted((int(x), int(y)) for x, y in zip(k, v) if (int(x) in stop_keys) == has)
            else:
                sums = {}
                for x, y in zip(k.tolist(), v.tolist()):
                    c = sums.setdefault(x, [0, 0])
                    c[0] = (c[0] + y) % (1 << 64)
                    c[1] += 1
                col = 1 if side0 == "count" else 0
                want = sorted((x, c[col]) for x, c in sums.items() if (x in stop_keys) == has)
            got = sorted(zip(_u64(got_k).tolist(), _u64(got_v).tolist()))
            assert got == want, (side0, method)
            assert len(got_k) and len(got_k) < len(k)


def test_same_shuffle_twice_empty_sides_and_many_partitions(sc):
    rng = np.random.default_rng(13)
    e = np.empty(0, dtype=np.uint64)
    a = (*rand_pairs(rng, 3000, 400), 2)
    b = (*rand_pairs(rng, 2000, 600), 3)
    shs = shuffles(sc, [a, b], 300)                             # R > 256: most partitions empty or nearly
    sides = [a, b, b, a]
    pairs = [(0b0110, 0), (0, 0b0110), (0b1000, 0b0110), (0b0010, 0b0100)]
    got = check(sc, sides, 300, pairs, shs=[shs[0], shs[1], shs[1], shs[0]])
    assert n_rows(got[0b0010, 0b0100]) == 0                      # required and excluded the same shuffle: nothing
    check(sc, [a, (e, e, 2), b], 7, masks(3))                    # an empty filter side
    check(sc, [(e, e, 2), a, b], 7, masks(3))                    # an empty side 0


# ---- 3. keys: 4-byte keys with negatives; u64::MAX; slot-hash-colliding keys on a filter side ------------------------
def test_int32_keys(sc):
    rng = np.random.default_rng(14)
    ks = [rng.integers(-2000, 1000, 20_000).astype(np.int32), rng.integers(0, 3000, 9000).astype(np.int32),
          rng.integers(-500, 2500, 7000).astype(np.int32)]
    sides = [(k, rng.integers(0, 1 << 62, len(k)).astype(np.uint64), 2 + j) for j, k in enumerate(ks)]
    check(sc, sides, 6, masks(3), key_width=4)


def test_slot_hash_collisions_on_a_filter_side(sc):
    rng = np.random.default_rng(15)
    fam = SH.same_home(rng, 3000, 12345)
    wrap = SH.wrap(rng, 1000, exclude=fam)
    filt = np.concatenate([fam[::2], wrap[::2], np.array([0, 2 ** 64 - 1], np.uint64)]).astype(np.uint64)
    base = np.concatenate([fam, wrap, np.array([0, 2 ** 64 - 1, 5], np.uint64)]).astype(np.uint64)
    k0 = np.repeat(base, 3)
    rng.shuffle(k0)
    sides = [(k0, rng.integers(0, 1 << 63, len(k0)).astype(np.uint64), 3),
             (np.repeat(filt, 2), np.arange(2 * len(filt), dtype=np.uint64), 2)]
    got = check(sc, sides, 4, masks(2))
    assert n_rows(got[0, 0b10]) == 3 * (len(base) - len(filt))


# ---- 4. values: sorted lists and byte-string values on side 0 -------------------------------------------------------------
def test_sorted_values_on_side0(sc):
    rng = np.random.default_rng(16)
    k, v = rand_pairs(rng, 30_000, 500, "i64", values="full")
    ks, _ = rand_pairs(rng, 2000, 700)
    R = 4
    for method, has in (("subtract_by_key", False), ("semi_join", True)):
        sj = getattr(sc.parallelize((k, v), 3), method)(sc.parallelize((ks, ks), 2), R, sort_values=True)
        stop = set(_u64(ks).tolist())
        for r in range(R):
            gk, gv = sj.compute(r)
            d = rows_by_key(_u64(gk), gv.view(np.int64))
            for key, vals in d.items():
                assert vals == sorted(vals) and (key in stop) == has
        want = sorted((int(x), int(y)) for x, y in zip(_u64(k), v) if (int(x) in stop) == has)
        gk, gv = sj.collect()
        assert sorted(zip(_u64(gk).tolist(), gv.astype(np.int64).tolist())) == want


def test_byte_string_values_on_side0(sc):
    rng = np.random.default_rng(17)
    n = 5000
    k = rng.integers(0, 800, n).astype(np.uint64)
    vals = [bytes(rng.integers(0, 256, int(rng.integers(0, 40))).astype(np.uint8)) for _ in range(n)]
    ks = rng.integers(400, 1200, 600).astype(np.uint64)
    a = sc.parallelize(k, 3, values=vals)
    for method, has in (("subtract_by_key", False), ("semi_join", True)):
        gk, gv = getattr(a, method)(sc.parallelize((ks, ks), 2), 5).collect()
        stop = set(ks.tolist())
        want = {}
        for x, y in zip(k.tolist(), vals):
            if (x in stop) == has:
                want.setdefault(x, []).append(y)
        got = {}
        for x, y in zip(gk.tolist(), gv):
            got.setdefault(x, []).append(y)
        assert got == want, method


# ---- 5. cross-checks: vb_join_n_outer at two sides; lazy filter sides are not grouped; a hot key -----------------------
def test_subtract_is_the_left_outer_join_without_a_match(sc):
    rng = np.random.default_rng(18)
    a = (*rand_pairs(rng, 12_000, 2000, values="full"), 3)
    b = (*rand_pairs(rng, 4000, 3000), 2)
    R = 4
    shs = shuffles(sc, [a, b], R)
    for r in range(R):
        k, vs, oks = abi_outer(sc, shs, r, 0b01)
        miss = oks[1] == 0
        want = {}
        for x, y in zip(k[miss].tolist(), vs[0][miss].tolist()):
            want.setdefault(x, []).append(y)
        sub = rows_by_key(*abi_semi(sc, shs, r, 0, 0b10))
        assert sub == want, r


def test_lazy_filter_sides_are_not_grouped(sc):
    rng = np.random.default_rng(19)
    sides = [(*rand_pairs(rng, 20_000, 3000), 3), (*rand_pairs(rng, 10_000, 4000), 2), (*rand_pairs(rng, 5000, 2000), 2)]
    shs = shuffles(sc, sides, 4)
    before = [grouping_launches(s) for s in shs[1:]]
    check(sc, sides, 4, [(0b10, 0b100), (0, 0b110)], shs=shs)
    assert [grouping_launches(s) for s in shs[1:]] == before == [0, 0]


def test_hot_key(sc):
    n = 100_000
    hot = np.uint64(0xDEADBEEF)
    k0 = np.concatenate([np.full(n, hot), np.arange(1, 1001, dtype=np.uint64)])
    k1 = np.concatenate([np.full(n, hot), np.arange(2001, 2101, dtype=np.uint64)])
    sides = [(k0, np.arange(len(k0), dtype=np.uint64), 4), (k1, np.arange(len(k1), dtype=np.uint64), 3)]
    shs = shuffles(sc, sides, 4)
    got = semi_parts(sc, shs, 4, 0b10, 0)
    assert n_rows(got) == n and got[O.get_partition(int(hot), 4)][int(hot)] == list(range(n))
    assert n_rows(semi_parts(sc, shuffles(sc, sides, 4), 4, 0, 0b10)) == 1000


def test_device_output_equals_host(sc):
    rng = np.random.default_rng(20)
    sides = [(*rand_pairs(rng, 6000, 900), 2), (*rand_pairs(rng, 3000, 900), 3)]
    shs = shuffles(sc, sides, 3)
    for pair in ((0, 0b10), (0b10, 0)):
        assert semi_parts(sc, shs, 3, *pair, dst=L.VB_DEVICE) == semi_parts(sc, shs, 3, *pair)


# ---- 6. String and Vec<u8> keys, with MetroHash-colliding keys on side 0 and on a filter side ---------------------------
def str_semi(sc, shs, r, req, exc, dev=False):
    lib, n = sc._lib, len(shs)
    nr, nk, nb = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    L.check(lib.vb_semi_join_n_str_size(_arr(shs), n, r, req, exc, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)))
    if dev:
        ko, kb, ro, v = (torch.empty(nk.value + 1, dtype=torch.int64, device="cuda"), torch.empty(nb.value, dtype=torch.uint8, device="cuda"),
                         torch.empty(nk.value + 1, dtype=torch.int64, device="cuda"), torch.empty(nr.value, dtype=torch.int64, device="cuda"))
    else:
        ko, kb, ro, v = np.empty(nk.value + 1, np.uint64), np.empty(nb.value, np.uint8), np.empty(nk.value + 1, np.uint64), np.empty(nr.value, np.uint64)
    L.check(lib.vb_semi_join_n_str(_arr(shs), n, r, req, exc, _ptr(ko), _ptr(kb), _ptr(ro), _ptr(v), L.VB_DEVICE if dev else L.VB_HOST))
    ko, kb, ro, v = (_host(x) for x in (ko, kb, ro, v))
    ko, ro, v = ko.astype(np.int64), ro.astype(np.int64), _u64(v)
    assert ko[0] == 0 and ro[0] == 0 and ro[-1] == nr.value and (np.diff(ro) > 0).all()
    keys = [bytes(kb[ko[i]:ko[i + 1]]) for i in range(len(ko) - 1)]
    assert len(set(keys)) == len(keys), f"a key twice in partition {r}"
    return {key: v[ro[i]:ro[i + 1]].tolist() for i, key in enumerate(keys)}


def str_lists(keys, vals):
    d = {}
    for k, v in zip(keys, _u64(vals).tolist()):
        d.setdefault(k, []).append(v)
    return d


def str_check(sc, kind, data, R, pairs, shs=None, dev=False):
    """data [(keys as bytes, vals, M)] -> per mask pair the partitions, checked against the restatement"""
    hashes = {}
    for keys, _, _ in data:
        u = list(dict.fromkeys(keys))
        hashes.update(zip(u, MC.hashes(kind, u).tolist()) if u else [])
    if shs is None:
        shs = [sc.parallelize(key_col(kind, keys), M, values=vals).group_by_key(R)._run() for keys, vals, M in data]
    lists = [str_lists(keys, vals) for keys, vals, _ in data]
    got = {}
    for req, exc in pairs:
        parts = [str_semi(sc, shs, r, req, exc, dev) for r in range(R)]
        assert parts == SJ.semi_of_lists(lists, R, req, exc, lambda k, R: hashes[k] % R), (req, exc)
        got[req, exc] = parts
    return got, shs


def str_rows(rng, pool, n):
    return [pool[i] for i in rng.integers(0, len(pool), n)]


@pytest.mark.parametrize("kind", [MC.STR, MC.BYTES])
def test_string_keys_every_mask_pair(sc, kind):
    rng = np.random.default_rng(21)
    pool = [b"k%d" % i for i in range(1500)] + [b"", "é".encode(), b"x" * 70]
    data = []
    for j, (n, lo, hi) in enumerate(((8000, 0, 1000), (4000, 600, 1503), (3000, 200, 900))):
        keys = str_rows(rng, pool[lo:hi], n)
        data.append((keys, rng.integers(0, 1 << 63, n).astype(np.uint64), 2 + j))
    got, shs = str_check(sc, kind, data, 5, masks(3))
    assert 0 < sum(len(l) for d in got[0, 0b10] for l in d.values()) < len(data[0][0])
    str_check(sc, kind, data, 5, [(0b10, 0b100), (0, 0b110)], shs=shs, dev=True)


@pytest.mark.parametrize("kind", [MC.STR, MC.BYTES])
def test_string_metro_collisions(sc, kind):
    fam = MC.same_hash(kind, 400, seed=31)
    absent = MC.absent(fam, 100)
    rng = np.random.default_rng(22)
    k0 = [k for k in fam.keys for _ in range(2)] + absent[:50]
    filt = fam.keys[::3] + absent[50:]                         # colliding keys on both sides, most not shared
    data = [(k0, rng.integers(0, 1 << 63, len(k0)).astype(np.uint64), 3),
            (filt, np.arange(len(filt), dtype=np.uint64), 2)]
    got, _ = str_check(sc, kind, data, 4, masks(2))
    assert sum(len(d) for d in got[0b10, 0]) == len(fam.keys[::3])


@pytest.mark.parametrize("kind", [MC.STR, MC.BYTES])
def test_string_views_and_mirror(sc, kind):
    rng = np.random.default_rng(23)
    pool = [b"w%d" % i for i in range(600)]
    k = str_rows(rng, pool, 6000)
    stop = pool[::4]
    R = 4
    words = sc.parallelize(key_col(kind, k), 3, values=np.ones(len(k), np.uint64))
    stops = sc.parallelize(key_col(kind, stop), 2, values=np.zeros(len(stop), np.uint64))
    dec = (lambda b: b) if kind == MC.BYTES else (lambda b: b.decode())
    counts = {}
    for w in k:
        counts[dec(w)] = counts.get(dec(w), 0) + 1
    stop_set = {dec(w) for w in stop}
    gk, gv = words.count_by_key(R).subtract_by_key(stops, R).collect()    # word count minus stop words, through a view
    assert dict(zip(gk.tolist(), gv.tolist())) == {w: c for w, c in counts.items() if w not in stop_set}
    gk, gv = words.semi_join(stops.count_by_key(R), R).collect()
    assert sorted(gk.tolist()) == sorted(dec(w) for w in k if dec(w) in stop_set) and (gv == 1).all()


# ---- 7. several ranks in one process ----------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [2, 3, 8])
def test_ranks_in_one_process(sc, W):
    eng = vdist.CudaEngine(sc)
    rng = np.random.default_rng(24 + W)
    sides = [(*rand_pairs(rng, 9000, 1500), 4), (*rand_pairs(rng, 4000, 2000), 3), (*rand_pairs(rng, 3000, 800), 2)]
    R = 6
    per_side = []
    for k, v, M in sides:
        place = lambda m, lo, hi, k=k, v=v: (k[lo:hi], v[lo:hi])
        shs, _ = run_ranks(eng, W, L.VB_AGG_COGROUP, maps_by_rank(len(k), M, W, place), R, L.VB_U64, L.VB_U64, n_map=M)
        per_side.append(shs)
    single = shuffles(sc, sides, R)
    for req, exc in ((0, 0b10), (0b10, 0b100), (0b110, 0)):
        want = semi_parts(sc, single, R, req, exc)
        for d in range(W):
            got = semi_parts(sc, [s[d] for s in per_side], R, req, exc)
            for r in range(R):
                assert got[r] == (want[r] if r % W == d else {}), (W, d, r)


@pytest.mark.parametrize("W", [2, 3])
def test_string_ranks_in_one_process(sc, W):
    from tests.test_gpu_str_multirank import run_ranks as str_run_ranks
    rng = np.random.default_rng(40 + W)
    pool = ["s%d" % i for i in range(900)]
    data = [([pool[i] for i in rng.integers(0, 900, 5000)], rng.integers(0, 1 << 40, 5000).astype(np.uint64)),
            ([pool[i] for i in rng.integers(300, 900, 2000)], rng.integers(0, 1 << 40, 2000).astype(np.uint64))]
    R = 5
    per_side = [str_run_ranks(sc, W, "group", "u64", k, v, 3, R) for k, v in data]
    single = [str_run_ranks(sc, 1, "group", "u64", k, v, 3, R)[0] for k, v in data]
    for req, exc in ((0, 0b10), (0b10, 0)):
        want = [str_semi(sc, single, r, req, exc) for r in range(R)]
        for d in range(W):
            for r in range(R):
                got = str_semi(sc, [s[d] for s in per_side], r, req, exc)
                assert got == (want[r] if r % W == d else {}), (W, d, r)


# ---- 8. refusals, every side usable afterwards ------------------------------------------------------------------------
def test_rejected_calls(sc):
    rng = np.random.default_rng(25)
    sides = [(*rand_pairs(rng, 2000, 300), 2), (*rand_pairs(rng, 1000, 300), 2), (*rand_pairs(rng, 500, 300), 2)]
    shs = shuffles(sc, sides, 3)
    lib, arr = sc._lib, _arr(shs)
    n = ctypes.c_uint64()
    bad = [(0b1000, 0), (0, 0b1000), (1, 0), (0, 1), (0b10, 0b10), (0b110, 0b100), (1 << 31, 0)]
    for req, exc in bad:
        assert lib.vb_semi_join_n_size(arr, 3, 0, req, exc, ctypes.byref(n)) == L.VB_ERR_INVALID, (req, exc)
        assert lib.vb_semi_join_n(arr, 3, 0, req, exc, None, None, L.VB_HOST) == L.VB_ERR_INVALID, (req, exc)
    assert lib.vb_semi_join_n_size(arr, 3, 3, 0, 0b10, ctypes.byref(n)) == L.VB_ERR_INVALID       # reduce_id
    assert lib.vb_semi_join_n_size(arr, 0, 0, 0, 0, ctypes.byref(n)) == L.VB_ERR_INVALID           # n_sides
    assert lib.vb_semi_join_n_size(arr, 17, 0, 0, 0, ctypes.byref(n)) == L.VB_ERR_INVALID
    assert lib.vb_semi_join_n_size(arr, 3, 0, 0, 0b10, None) == L.VB_ERR_INVALID
    assert lib.vb_semi_join_n(arr, 3, 0, 0, 0b10, None, None, 7) == L.VB_ERR_INVALID              # dst_loc
    r_rows = next(r for r in range(3) if len(abi_semi(sc, shs, r, 0, 0)[0]))
    assert lib.vb_semi_join_n(arr, 3, r_rows, 0, 0, None, None, L.VB_HOST) == L.VB_ERR_INVALID     # NULL outputs
    other = sc.parallelize((np.arange(10, dtype=np.int32), np.arange(10, dtype=np.uint64)), 2).cogroup(
        sc.parallelize((np.arange(10, dtype=np.int32), np.arange(10, dtype=np.uint64)), 2), 3)._run()[0]
    assert lib.vb_semi_join_n_size(_arr([shs[0], other]), 2, 0, 0, 0b10, ctypes.byref(n)) == L.VB_ERR_INVALID  # key width
    red = sc.parallelize((sides[0][0], sides[0][1]), 2).reduce_by_key("sum", 3)._run()
    assert lib.vb_semi_join_n_size(_arr([shs[0], red]), 2, 0, 0, 0b10, ctypes.byref(n)) == L.VB_ERR_INVALID  # not a side
    s = sc.parallelize(key_col(MC.STR, [b"a", b"b"]), 1, values=np.arange(2, dtype=np.uint64)).group_by_key(3)._run()
    sb = sc.parallelize(key_col(MC.BYTES, [b"a", b"b"]), 1, values=np.arange(2, dtype=np.uint64)).group_by_key(3)._run()
    assert lib.vb_semi_join_n_size(_arr([shs[0], s]), 2, 0, 0, 0b10, ctypes.byref(n)) == L.VB_ERR_INVALID    # String side
    nr = ctypes.c_uint64()
    assert lib.vb_semi_join_n_str_size(_arr([s, shs[0]]), 2, 0, 0, 0b10, ctypes.byref(nr), None, None) == L.VB_ERR_INVALID
    assert lib.vb_semi_join_n_str_size(_arr([s, sb]), 2, 0, 0, 0b10, ctypes.byref(nr), None, None) == L.VB_ERR_INVALID
    for req, exc in bad:
        assert lib.vb_semi_join_n_str_size(_arr([s, s, s]), 3, 0, req, exc, ctypes.byref(nr), None, None) == L.VB_ERR_INVALID
    rs = next(r for r in range(3) if str_semi(sc, [s], r, 0, 0))
    assert lib.vb_semi_join_n_str(_arr([s]), 1, rs, 0, 0, None, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    check(sc, sides, 3, masks(3), shs=shs)                     # every side still usable
    str_semi(sc, [s, s], 0, 0b10, 0)


# ---- 9. the C++ example -----------------------------------------------------------------------------------------------
def test_cpp_subtract_by_key_example_runs():
    exe = os.path.join(ROOT, "examples", "_build", "subtract_by_key")
    if not os.path.exists(exe):
        pytest.skip("examples not built (run __graft_entry__.build())")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "subtract_by_key: [(1, 100), (1, 101), (3, 300)]" in r.stdout, r.stdout
