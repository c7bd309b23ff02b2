"""GPU parity: the CUDA path, called through the C ABI (vega_b200 → libvega_b200.so), against
the CPU oracle on the same inputs.  Bit-exact for keys, counts, integer reductions, grouped
membership AND order (tests/test_pair_rdd.rs:30-36 pins input order inside a group); f64 sums
within 1e-6 relative (north_star).  Golden vectors are the reference's own test data."""
import threading

import numpy as np
import pytest

import vega_b200 as vb
from oracle import oracle as O
from tests.util import (assert_f64_sums, bits_dict, gpu_group_parts, gpu_reduce_parts, oracle_group, oracle_reduce,
                        oracle_reduce_bits, rand_pairs)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


# ---- the reference's golden vectors through the GPU path ------------------------------------
def test_group_by_key_golden(sc):
    # tests/test_pair_rdd.rs:8-37 / examples/group_by.rs with "x"→10, "y"→20
    keys = np.array([10] * 7 + [20] * 8, dtype=np.uint64)
    vals = np.array(list(range(1, 8)) + list(range(1, 9)), dtype=np.int64)
    g = sc.make_rdd((keys, vals), 4).group_by_key(4)
    res = sorted((k, v.tolist()) for k, v in g.collect().to_list())
    assert res == [(10, [1, 2, 3, 4, 5, 6, 7]), (20, [1, 2, 3, 4, 5, 6, 7, 8])]


def test_join_golden(sc):
    # tests/test_pair_rdd.rs:39-82 / examples/join.rs; payload strings → table indices
    col1 = [(1, ("A", "B")), (2, ("C", "D")), (3, ("E", "F")), (4, ("G", "H"))]
    col2 = [(1, "A1"), (1, "A2"), (2, "B1"), (2, "B2"), (3, "C1"), (3, "C2")]
    r1 = sc.parallelize((np.array([k for k, _ in col1], dtype=np.int32), np.arange(4, dtype=np.uint64)), 4)
    r2 = sc.parallelize((np.array([k for k, _ in col2], dtype=np.int32), np.arange(6, dtype=np.uint64)), 4)
    k, v, w = r2.join(r1, 4).collect()
    res = sorted((int(a), (col2[int(b)][1], col1[int(c)][1])) for a, b, c in zip(k, v, w))
    assert res == [(1, ("A1", ("A", "B"))), (1, ("A2", ("A", "B"))), (2, ("B1", ("C", "D"))),
                   (2, ("B2", ("C", "D"))), (3, ("C1", ("E", "F"))), (3, ("C2", ("E", "F")))]


@pytest.mark.parametrize("slices", [4, 2])
def test_count_by_value_golden(sc, slices):
    # tests/test_pair_rdd.rs:84-109
    rdd = sc.parallelize(np.array([1, 2, 1, 3, 2, 3, 3, 2, 3], dtype=np.int32), slices)
    k, c = rdd.count_by_value().collect()
    assert sorted(zip(k.tolist(), c.tolist())) == [(1, 2), (2, 3), (3, 4)]


def test_group_by_golden(sc):
    # tests/test_pair_rdd.rs:111-135: group_by(sign) with neg→0, zero→1, pos→2
    xs = np.array([-3, -2, -1, 0, 1, 2, 3], dtype=np.int64)
    keys = np.where(xs < 0, 0, np.where(xs == 0, 1, 2)).astype(np.uint64)
    res = sorted((k, v.tolist()) for k, v in sc.make_rdd((keys, xs), 2).group_by_key(2).collect().to_list())
    assert res == [(0, [-3, -2, -1]), (1, [0]), (2, [1, 2, 3])]


@pytest.mark.parametrize("parts", [None, 2, 10])
def test_distinct_golden(sc, parts):
    # tests/test_rdd.rs:285-322
    rdd = sc.parallelize(np.array([1, 2, 2, 2, 3, 3, 3, 4, 4, 5], dtype=np.int32), 3)
    res = rdd.distinct(parts).collect()
    assert len(res) == 5 and set(res.tolist()) == {1, 2, 3, 4, 5}


def test_cogroup_and_intersection_golden(sc):
    # tests/test_rdd.rs:434-456 (cogroup → 4 keys) and :484-521 (intersection → [3,4,5,13])
    k = np.array([1, 2, 3, 4], dtype=np.int32)
    v = np.arange(4, dtype=np.uint64)
    cg = sc.parallelize((k, v), 2).cogroup(sc.parallelize((k, v), 2), 2).cogroup_collect()
    assert sorted((a, (x.tolist(), y.tolist())) for a, (x, y) in cg) == [(i + 1, ([i], [i])) for i in range(4)]
    c1 = np.array([1, 2, 3, 4, 5, 10, 12, 13, 19, 0], dtype=np.int32)
    c2 = np.array([3, 4, 5, 6, 7, 8, 11, 13], dtype=np.int32)
    for nparts in (3, 2):
        cg = sc.parallelize((c1, np.zeros(10, np.uint64)), 2).cogroup(sc.parallelize((c2, np.zeros(8, np.uint64)), 4), nparts)
        inter = sorted(a for a, (x, y) in cg.cogroup_collect() if len(x) >= 1 and len(y) >= 1)
        assert inter == [3, 4, 5, 13]


@pytest.mark.parametrize("nparts", [None, 3])
def test_intersection_api_golden(sc, nparts):
    # tests/test_rdd.rs:484-521 through the API (Rdd.intersection / intersection_with_num_partitions)
    first = sc.parallelize(np.array([1, 2, 3, 4, 5, 10, 12, 13, 19, 0], dtype=np.int32), 2)
    second = sc.parallelize(np.array([3, 4, 5, 6, 7, 8, 11, 13], dtype=np.int32), 4)
    inter = first.intersection(second, nparts)
    assert sorted(inter.collect().tolist()) == [3, 4, 5, 13]
    for r in range(inter.num_slices):         # placement: HashPartitioner over 4-byte keys
        assert all(O.get_partition(int(x), inter.num_slices, 4) == r for x in inter.compute(r))


def test_subtract_api_golden(sc):
    # tests/test_rdd.rs:675-699
    first = sc.parallelize(np.array([1, 2, 3, 4, 5, 10, 12, 13, 19, 0], dtype=np.int32), 4)
    second = sc.parallelize(np.array([3, 4, 5, 6, 7, 8, 11, 13], dtype=np.int32), 4)
    assert sorted(first.subtract(second).collect().tolist()) == [0, 1, 2, 10, 12, 19]


def test_set_ops_match_numpy_on_random_inputs(sc):
    rng = np.random.default_rng(9)
    a = rng.integers(0, 5000, 40_000).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    b = rng.integers(2500, 9000, 30_000).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    ra, rb = sc.parallelize(a, 5), sc.parallelize(b, 3)
    assert sorted(ra.intersection(rb, 7).collect().tolist()) == sorted(np.intersect1d(a, b).tolist())
    assert sorted(ra.subtract(rb).collect().tolist()) == sorted(np.setdiff1d(a, b).tolist())


def test_group_by_api_golden(sc):
    # tests/test_pair_rdd.rs:111-135 through Rdd.group_by(func): neg -> 0, zero -> 1, pos -> 2
    xs = np.array([-3, -2, -1, 0, 1, 2, 3], dtype=np.int64)
    g = sc.make_rdd(xs, 2).group_by(lambda x: (np.sign(x) + 1).astype(np.uint64))
    assert sorted((k, v.tolist()) for k, v in g.collect().to_list()) == [(0, [-3, -2, -1]), (1, [0]), (2, [1, 2, 3])]


# ---- randomized differential tests against the oracle -----------------------------------------
@pytest.mark.parametrize("op,vdtype", [("sum", "u64"), ("sum", "i64"), ("sum", "f64"), ("min", "u64"), ("max", "u64"),
                                       ("min", "i64"), ("max", "i64"), ("min", "f64"), ("max", "f64")])
@pytest.mark.parametrize("n,M,R,nkeys", [(50_000, 5, 7, 1000), (3, 8, 2, 3), (200_000, 8, 8, 150_000)])
def test_reduce_by_key_matches_oracle(sc, op, vdtype, n, M, R, nkeys):
    rng = np.random.default_rng(hash((op, vdtype, n)) % 2 ** 32)
    keys, vals = rand_pairs(rng, n, nkeys, vdtype)
    got = gpu_reduce_parts(sc.parallelize((keys, vals), M).reduce_by_key(op, R))
    if vdtype == "f64" and op == "sum":
        assert_f64_sums(got, keys, vals, R)                          # every key, its placement, the exact-sum bound
        return
    want = oracle_reduce(op, keys, vals, M, R, vdtype)
    assert [set(d) for d in got] == [set(d) for d in want]          # keys AND placement (hash % R)
    assert got == want


@pytest.mark.parametrize("layout", ["aos_host", "soa_device", "aos_device"])
def test_reduce_layouts_and_locations(sc, layout):
    import torch
    rng = np.random.default_rng(11)
    keys, vals = rand_pairs(rng, 100_000, 5000)
    want = oracle_reduce("sum", keys, vals, 6, 5)
    if layout == "aos_host":
        rdd = sc.parallelize(np.stack([keys, vals], axis=1), 6)
    elif layout == "soa_device":
        rdd = sc.parallelize((torch.from_numpy(keys.view(np.int64)).cuda(), torch.from_numpy(vals.view(np.int64)).cuda()), 6)
    else:
        rdd = sc.parallelize(torch.from_numpy(np.stack([keys, vals], axis=1).view(np.int64)).cuda(), 6)
    got = gpu_reduce_parts(rdd.reduce_by_key("sum", 5))
    if layout != "aos_host":       # int64 tensors: same bits
        got = [{k & (2 ** 64 - 1): v & (2 ** 64 - 1) for k, v in d.items()} for d in got]
    assert got == want


@pytest.mark.parametrize("n,M,R,nkeys", [(60_000, 4, 4, 500), (15, 4, 4, 2), (5, 32, 3, 4), (100_000, 7, 300, 40_000),
                                         (30_000, 3, 1, 30_000)])
def test_group_by_key_matches_oracle_in_order(sc, n, M, R, nkeys):
    rng = np.random.default_rng(n + R)
    keys, vals = rand_pairs(rng, n, nkeys)
    want = oracle_group(keys, vals, M, R)
    got = gpu_group_parts(sc.parallelize((keys, vals), M).group_by_key(R))
    assert got == want        # per partition: same keys, each value list in input order (F5)


def test_group_aos_device_borrowed(sc):
    import torch
    rng = np.random.default_rng(5)
    keys, vals = rand_pairs(rng, 300_000, 20_000)
    rows = torch.from_numpy(np.stack([keys, vals], axis=1).view(np.int64)).cuda()
    got = gpu_group_parts(sc.parallelize(rows, 8).group_by_key(8))
    got = [{k & (2 ** 64 - 1): [x & (2 ** 64 - 1) for x in v] for k, v in d.items()} for d in got]
    assert got == oracle_group(keys, vals, 8, 8)


def test_count_and_i32_key_width(sc):
    rng = np.random.default_rng(9)
    keys = rng.integers(-500, 500, 40_000).astype(np.int32)
    want = oracle_reduce("count", keys.astype(np.int64), None, 5, 6, key_width=4)
    got = gpu_reduce_parts(sc.parallelize(keys, 5).count_by_value().__class__(
        vb.PairRdd(sc, vb.rdd._Col(keys), None, 5), "count", 6))
    got = [{k & (2 ** 64 - 1): v for k, v in d.items()} for d in got]
    assert got == want


def test_sentinel_and_extreme_keys(sc):
    # 0xFFFF_FFFF_FFFF_FFFF is the table's empty marker internally — it must still work as a key
    keys = np.array([2 ** 64 - 1, 0, 2 ** 64 - 1, 1, 2 ** 63, 0, 2 ** 64 - 1, 2 ** 64 - 2], dtype=np.uint64)
    vals = np.arange(1, 9, dtype=np.uint64)
    for M, R in ((1, 1), (3, 4)):
        assert gpu_reduce_parts(sc.parallelize((keys, vals), M).reduce_by_key("sum", R)) == oracle_reduce("sum", keys, vals, M, R)
        assert gpu_group_parts(sc.parallelize((keys, vals), M).group_by_key(R)) == oracle_group(keys, vals, M, R)
        assert gpu_reduce_parts(sc.parallelize((keys, vals), M).reduce_by_key("min", R)) == oracle_reduce("min", keys, vals, M, R)


def test_empty_and_tiny_inputs(sc):
    e = np.empty(0, dtype=np.uint64)
    assert gpu_reduce_parts(sc.parallelize((e, e), 4).reduce_by_key("sum", 3)) == [{}, {}, {}]
    assert gpu_group_parts(sc.parallelize((e, e), 4).group_by_key(2)) == [{}, {}]
    k, v, w = sc.parallelize((e, e), 2).join(sc.parallelize((e, e), 2), 2).collect()
    assert len(k) == len(v) == len(w) == 0
    one = np.array([7], dtype=np.uint64)
    assert gpu_reduce_parts(sc.parallelize((one, one), 5).reduce_by_key("max", 2)) == oracle_reduce("max", one, one, 5, 2)


def test_table_growth_all_distinct(sc):
    # a (deliberately wrong) hint of 1000 distinct keys sizes the first table at 2^11 slots:
    # 3M distinct keys must overflow it and restart with larger tables until they fit
    n = 3_000_000
    keys = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
    vals = np.ones(n, dtype=np.uint64)
    rdd = sc.parallelize((keys, vals), 2).reduce_by_key("sum", 4, hint=1000)
    k, c = rdd.collect()
    assert len(k) == n and (c == 1).all() and len(np.unique(k)) == n
    assert rdd.stats()["table_restarts"] >= 1
    for r in (0, 3):
        kk, _ = rdd.compute(r)
        sample = kk[:: max(1, len(kk) // 50)]
        assert all(O.get_partition(int(x), 4) == r for x in sample)
    # same through the dictionary of group_by_key
    g = sc.parallelize((keys[:500_000], vals[:500_000]), 3).group_by_key(2).collect()
    assert len(g) == 500_000 and (np.diff(g.offsets.astype(np.int64)) == 1).all()


@pytest.mark.parametrize("na,nb,R,nkeys", [(20_000, 30_000, 4, 3000), (5000, 10, 3, 50), (1000, 1000, 300, 2000)])
def test_join_matches_oracle(sc, na, nb, R, nkeys):
    rng = np.random.default_rng(na + nb)
    ka, va = rand_pairs(rng, na, nkeys)
    kb, vb_ = rand_pairs(rng, nb, nkeys)
    want = sorted(zip(*[np.concatenate(x).tolist() for x in zip(*O.join(ka, va, 3, kb, vb_, 5, R))]))
    k, v, w = sc.parallelize((ka, va), 3).join(sc.parallelize((kb, vb_), 5), R).collect()
    assert sorted(zip(k.tolist(), v.tolist(), w.tolist())) == want
    # per-partition placement and the reference's nesting order (for v in vs { for w in ws })
    j = sc.parallelize((ka, va), 3).join(sc.parallelize((kb, vb_), 5), R)
    ora = O.join(ka, va, 3, kb, vb_, 5, R)
    for r in range(min(R, 4)):
        gk, gv, gw = j.compute(r)
        ok, ov, ow = ora[r]
        assert sorted(zip(gk.tolist(), gv.tolist(), gw.tolist())) == sorted(zip(ok.tolist(), ov.tolist(), ow.tolist()))
        # within one key, GPU rows keep (v outer, w inner) order like the oracle
        if len(gk):
            key = gk[0]
            assert list(zip(gv[gk == key].tolist(), gw[gk == key].tolist())) == list(zip(ov[ok == key].tolist(), ow[ok == key].tolist()))


@pytest.mark.parametrize("kdtype", ["u64", "i64", "f64"])
@pytest.mark.parametrize("payload", [True, False])
def test_sort_by_key_matches_oracle(sc, kdtype, payload):
    rng = np.random.default_rng(3)
    n = 70_000
    if kdtype == "u64":
        keys = rng.integers(0, 2 ** 63, n).astype(np.uint64) * np.uint64(2) + rng.integers(0, 2, n).astype(np.uint64)
    elif kdtype == "i64":
        keys = rng.integers(-2 ** 62, 2 ** 62, n).astype(np.int64)
    else:
        keys = rng.standard_normal(n) * 1e6
    keys[::7] = keys[3]          # long runs of equal keys: stability + cut rule
    vals = np.arange(n, dtype=np.uint64)
    ok, ov, ps = O.sort_by_key(keys, vals, 8, kdtype)
    src = sc.parallelize((keys, vals), 5) if payload else sc.parallelize(keys, 5)
    rdd = src.sort_by_key(8) if payload else src.sort(8)
    k, v = rdd.collect()
    assert (k == ok).all()
    if payload:
        assert (v == ov).all()      # stable: equal keys keep input order
    sizes = [len(rdd.compute(r)[0]) for r in range(8)]
    assert sizes == np.diff(ps.astype(np.int64)).tolist()


def test_partition_by_key(sc):
    keys = np.arange(1000, dtype=np.uint64)
    vals = keys * np.uint64(3)
    parts = sc.parallelize((keys, vals), 4).partition_by_key(100).glom()
    assert len(parts) == 100 and sum(len(p) for p in parts) == 1000
    for r in (0, 17, 99):
        assert all(O.get_partition(int(v) // 3, 100) == r for v in parts[r])


def test_device_generator_matches_oracle(sc):
    import torch
    n, D = 100_000, 977
    rows = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=12345, n=n, mode="uniform", n_distinct=D, seed_k=1, seed_v=2)
    k, v = O.gen_uniform(12345, n, D, 1, 2)
    got = rows.cpu().numpy().view(np.uint64)
    assert (got[:, 0] == k).all() and (got[:, 1] == v).all()


# ---- boundary behaviour ---------------------------------------------------------------------
def test_stage_resubmission_overwrites(sc):
    keys = np.array([1, 2, 3, 1], dtype=np.uint64)
    v1 = np.array([10, 20, 30, 40], dtype=np.uint64)
    sh = vb.Shuffle(sc, 2, 2, 0, 0, 1)
    ck, cv = vb.rdd._Col(keys), vb.rdd._Col(v1)
    sh.map(0, ck, cv, 0, 2)
    sh.map(1, ck, cv, 2, 4)
    sh.map(0, ck, cv, 0, 2)          # resubmitted map task must not double count
    sh.seal()
    got = {}
    for r in range(2):
        k, c = sh.reduce(r)
        got.update(zip(k.tolist(), c.tolist()))
    assert got == {1: 50, 2: 20, 3: 30}
    sh.free()


def test_reduce_blocks_until_sealed(sc):
    keys = np.arange(100, dtype=np.uint64)
    sh = vb.Shuffle(sc, 1, 1, 0, 0, 1)
    col = vb.rdd._Col(keys)
    sh.map(0, col, col, 0, 100)
    out = {}
    t = threading.Thread(target=lambda: out.setdefault("r", sh.reduce(0)))
    t.start()
    t.join(0.3)
    assert t.is_alive()              # blocked in vb_shuffle_reduce_size (condvar), like get_server_uris
    sh.seal()
    t.join(10)
    assert not t.is_alive() and sorted(out["r"][0].tolist()) == list(range(100))
    sh.free()


def test_error_conventions(sc):
    keys = np.arange(10, dtype=np.uint64)
    col = vb.rdd._Col(keys)
    sh = vb.Shuffle(sc, 2, 2, 0, 0, 1)
    sh.map(0, col, col, 0, 5)
    with pytest.raises(vb.VegaB200Error) as e:       # map 1 never submitted
        sh.seal()
    assert e.value.code == -4
    sh.free()
    sh = vb.Shuffle(sc, 1, 2, 0, 0, 1)
    sh.map(0, col, col, 0, 10)
    sh.seal()
    with pytest.raises(vb.VegaB200Error):            # map after seal
        sh.map(0, col, col, 0, 10)
    with pytest.raises(vb.VegaB200Error):            # bad reduce id
        sh.reduce(2)
    sh.free()
    with pytest.raises(vb.VegaB200Error):            # f64 keys are not Hash
        vb.Shuffle(sc, 1, 1, 2, 0, 1)


# ---- BASELINE.json configs as (scaled-down) parity cases -------------------------------------
def test_config1_group_by_1e6_pairs_4_partitions(sc):
    """configs[0]: examples/group_by.rs shape at 1e6 (u64,u64) pairs, 4 partitions — full size."""
    import torch
    n, D = 1_000_000, 10_000
    rows = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=0, n=n, mode="uniform", n_distinct=D, seed_k=1, seed_v=2)
    keys, vals = O.gen_uniform(0, n, D, 1, 2)
    got = gpu_group_parts(sc.make_rdd(rows, 4).group_by_key(4))
    got = [{k & (2 ** 64 - 1): [x & (2 ** 64 - 1) for x in v] for k, v in d.items()} for d in got]
    assert got == oracle_group(keys, vals, 4, 4)


def test_config5_zipf_skew_reduce_and_group(sc):
    """configs[4] scaled: Zipf(1.1) keys, 64 reduce partitions.  The hot-key cache path must give
    exactly the oracle's sums/counts, and group order must survive the skew."""
    import torch
    n, D = 2_000_000, 50_000
    rows = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=0, n=n, mode="zipf", n_distinct=D, seed_k=5, seed_v=2, zipf_s=1.1)
    host = rows.cpu().numpy().view(np.uint64)
    keys, vals = host[:, 0].copy(), host[:, 1].copy()
    top = np.bincount(np.unique(keys, return_inverse=True)[1]).max()
    assert top > 0.05 * n                      # the generator really is skewed
    for op in ("sum", "max"):
        got = gpu_reduce_parts(sc.make_rdd(rows, 8).reduce_by_key(op, 64))
        got = [{k & (2 ** 64 - 1): v & (2 ** 64 - 1) for k, v in d.items()} for d in got]
        assert got == oracle_reduce(op, keys, vals, 8, 64)
    got = gpu_reduce_parts(sc.make_rdd(rows, 8).count_by_key(64))
    got = [{k & (2 ** 64 - 1): v for k, v in d.items()} for d in got]
    assert got == oracle_reduce("count", keys, vals, 8, 64)
    fv = (vals.astype(np.float64) / 2 ** 20)
    gotf = gpu_reduce_parts(sc.make_rdd((keys, fv), 8).reduce_by_key("sum", 64))
    assert_f64_sums(gotf, keys, fv, 64, exact=True)        # 20-bit values / 2^20: every partial sum is exact
    sub = slice(0, 300_000)
    assert gpu_group_parts(sc.make_rdd((keys[sub], vals[sub]), 8).group_by_key(64)) == oracle_group(keys[sub], vals[sub], 8, 64)


def test_config4_join_unique_keys_scaled(sc):
    """configs[3] scaled: two RDDs whose keys occur once per side, a known number of shared keys, 8 partitions."""
    import torch
    n, shared = 400_000, 8_000
    a = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    b = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=a, first=0, n=n, mode="unique", rank_base=0)
    sc.gen_pairs(out_rows=b, first=0, n=n, mode="unique", rank_base=n - shared)
    k, v, w = sc.make_rdd(a, 8).join(sc.make_rdd(b, 8), 8).collect()
    assert len(k) == shared and len(np.unique(k)) == shared
    ha, hb = a.cpu().numpy().view(np.uint64), b.cpu().numpy().view(np.uint64)
    want = O.join(ha[:, 0].copy(), ha[:, 1].copy(), 8, hb[:, 0].copy(), hb[:, 1].copy(), 8, 8)
    want_rows = sorted(zip(*[np.concatenate(x).tolist() for x in zip(*want)]))
    assert sorted(zip(k.view(np.uint64).tolist(), v.view(np.uint64).tolist(), w.view(np.uint64).tolist())) == want_rows


def test_config2_full_size_properties(sc):
    """configs[1] at FULL size (1e9 pairs, 1e6 keys) through size-independent properties: every key of the
    universe appears exactly once over the 8 partitions, in the partition its hash names; the sums add up
    to the sum of all values; per-key sums of sampled keys equal a brute-force torch reduction."""
    import torch
    if torch.cuda.get_device_properties(0).total_memory < 60 * 2 ** 30:
        pytest.skip("needs ~20 GB of HBM")
    n, D = 1_000_000_000, 1_000_000
    rows = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=0, n=n, mode="uniform", n_distinct=D, seed_k=1, seed_v=2)
    rdd = sc.make_rdd(rows, 8).reduce_by_key("sum", 8)
    parts = [rdd.compute(r) for r in range(8)]
    allk = np.concatenate([p[0] for p in parts]).view(np.uint64)
    allc = np.concatenate([p[1] for p in parts]).view(np.uint64)
    assert len(allk) == D and len(np.unique(allk)) == D
    assert int(allc.sum(dtype=np.uint64)) == int(rows[:, 1].sum().item())
    universe = np.array([O.lib().vo_splitmix64(int(r) ^ 0xA5A5A5A5A5A5A5A5) for r in range(0, D, 9973)], dtype=np.uint64)
    assert np.isin(universe, allk).all()
    for r in (0, 5):
        kk = parts[r][0].view(np.uint64)
        assert all(O.get_partition(int(x), 8) == r for x in kk[:: len(kk) // 40])
    lut = dict(zip(allk.tolist(), allc.tolist()))
    for key in universe[:3]:
        brute = int(rows[:, 1][rows[:, 0] == int(np.int64(np.uint64(key).view(np.int64)))].sum().item())
        assert lut[int(key)] == brute
    del rows
    torch.cuda.empty_cache()


def test_cpp_host_mirror_examples_run():
    """examples/group_by.cpp and examples/join.cpp are the reference's examples/group_by.rs and
    examples/join.rs over include/vega_b200.hpp (same data); set_ops.cpp is tests/test_rdd.rs:484-521,675-699
    (intersection / subtract); they exit 0 only on the expected result."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for exe, needle in (("group_by", "[1, 2, 3, 4, 5, 6, 7, 8]"), ("join", "(3, (C2, (E,F)))"), ("set_ops", "subtract: 0 1 2 10 12 19")):
        path = os.path.join(root, "examples", "_build", exe)
        if not os.path.exists(path):
            pytest.skip("examples not built (run __graft_entry__.build())")
        out = subprocess.run([path], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        assert needle in out.stdout, out.stdout


# ---- SURVEY §8(f) N1: bincode blobs ------------------------------------------------------------
def test_bincode_blobs_encode_decode(sc):
    from oracle import bincode_ref as B
    rng = np.random.default_rng(77)
    keys, vals = rand_pairs(rng, 40_000, 900)
    # encode: reduce partition → Vec<(u64,u64)> bytes == oracle's encoding of the same rows
    rdd = sc.parallelize((keys, vals), 3).reduce_by_key("sum", 4)
    sh = rdd._run()
    for r in range(4):
        k, c = sh.reduce(r)
        blob = sh.reduce_blob(r)
        assert blob == B.encode_pairs(list(zip(k.tolist(), c.tolist())))
        assert dict(B.decode_pairs(blob)) == oracle_reduce("sum", keys, vals, 3, 4)[r]
    # encode: group partition → Vec<(u64,Vec<u64>)>
    g = sc.parallelize((keys, vals), 3).group_by_key(2)
    gsh = g._run()
    for r in range(2):
        k, o, v = gsh.reduce(r)
        want = [(int(k[i]), v[int(o[i]):int(o[i + 1])].tolist()) for i in range(len(k))]
        assert gsh.reduce_blob(r) == B.encode_groups(want)
    # decode: CPU-produced map-side-combined buckets (the oracle's map outputs) consumed as map tasks
    for op, agg in (("sum", 1), ("count", 4), ("max", 3)):
        sh2 = vb.Shuffle(sc, 3, 1, 0, 0, agg)
        starts = vb.slice_starts(len(keys), 3)
        for m in range(3):
            part = O.shuffle(op, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]], 1, 1)[0]
            sh2.map_blob(m, B.encode_pairs(list(zip(part["keys"].tolist(), part["combined"].tolist()))))
        sh2.seal()
        k, c = sh2.reduce(0)
        assert dict(zip(k.tolist(), c.tolist())) == oracle_reduce(op, keys, vals, 3, 1)[0]
        sh2.free()
    # combined blobs over i64 MAX (signed order, full range) and f64 MIN (NaN ignored, -0.0 < +0.0): a blob carries the
    # raw value bits, which the merge orders through the same transform as map inputs
    for op, agg, vdt, mode in (("max", 3, "i64", "full"), ("min", 2, "f64", "special")):
        k2, v2 = rand_pairs(rng, 40_000, 900, vdt, values=mode)
        sh2 = vb.Shuffle(sc, 3, 1, 0, {"i64": 1, "f64": 2}[vdt], agg)
        starts = vb.slice_starts(len(k2), 3)
        for m in range(3):
            part = O.shuffle(op, k2[starts[m]:starts[m + 1]], v2[starts[m]:starts[m + 1]], 1, 1, vdtype=vdt)[0]
            sh2.map_blob(m, B.encode_pairs(list(zip(part["keys"].tolist(), part["combined"].view(np.uint64).tolist()))))
        sh2.seal()
        assert [bits_dict(*sh2.reduce(0))] == oracle_reduce_bits(op, k2, v2, 3, 1, vdt), (op, vdt)
        sh2.free()
    sh3 = vb.Shuffle(sc, 2, 2, 0, 0, 0)
    half = len(keys) // 2
    for m, sl in enumerate((slice(0, half), slice(half, None))):
        part = oracle_group(keys[sl], vals[sl], 1, 1)[0]
        sh3.map_blob(m, B.encode_groups(list(part.items())))
    sh3.seal()
    got = {}
    for r in range(2):
        k, o, v = sh3.reduce(r)
        got.update({int(k[i]): v[int(o[i]):int(o[i + 1])].tolist() for i in range(len(k))})
    want = {}
    for d in oracle_group(keys, vals, 2, 2):
        want.update(d)
    # a blob lists each key's values in the map task's encounter order, so the reference's group order survives
    assert got == want
    sh3.free()
    # corrupted payloads are rejected, not crashed on (shuffle_fetcher.rs:168-185)
    bad = vb.Shuffle(sc, 1, 1, 0, 0, 1)
    for blob in (b"\x05" + b"\x00" * 7, b"\x01" + b"\x00" * 15, b"\x00" * 7):
        with pytest.raises(vb.VegaB200Error) as e:
            bad.map_blob(0, blob)
        assert e.value.code == -1
    bad.free()


def test_shared_table_of_borrowed_map_tasks(sc):
    """Map tasks with VB_DEVICE_BORROWED input combine into one shared table, launched without a host round
    trip; overflow and map-id resubmission are repaired at seal from the still-borrowed inputs."""
    import torch
    rng = np.random.default_rng(123)
    keys, vals = rand_pairs(rng, 400_000, 150_000)
    tk = torch.from_numpy(keys.view(np.int64)).cuda()
    tv = torch.from_numpy(vals.view(np.int64)).cuda()
    want = oracle_reduce("sum", keys, vals, 4, 3)
    # (a) plain
    got = gpu_reduce_parts(sc.parallelize((tk, tv), 4).reduce_by_key("sum", 3))
    assert [{k & (2 ** 64 - 1): v & (2 ** 64 - 1) for k, v in d.items()} for d in got] == want
    # (b) a wrong hint (100 keys) makes the shared table overflow: seal must rebuild it larger
    rdd = sc.parallelize((tk, tv), 4).reduce_by_key("sum", 3, hint=100)
    got = gpu_reduce_parts(rdd)
    assert [{k & (2 ** 64 - 1): v & (2 ** 64 - 1) for k, v in d.items()} for d in got] == want
    assert rdd.stats()["table_restarts"] >= 1
    # (c) resubmitting a map id must not double count; mixing borrowed and host-copied map tasks merges both
    starts = vb.slice_starts(len(keys), 4)
    sh = vb.Shuffle(sc, 4, 3, 0, 1, 1)
    ck, cv = vb.rdd._Col(tk), vb.rdd._Col(tv)
    hk, hv = vb.rdd._Col(keys), vb.rdd._Col(vals)
    for m in range(4):
        if m == 2:
            sh.map(m, hk, hv, int(starts[m]), int(starts[m + 1]))       # host input: per-map table
        else:
            sh.map(m, ck, cv, int(starts[m]), int(starts[m + 1]))
    sh.map(1, ck, cv, int(starts[1]), int(starts[2]))                   # resubmission of a borrowed task
    sh.seal()
    for r in range(3):
        k, c = sh.reduce(r)
        assert {int(a) & (2 ** 64 - 1): int(b) & (2 ** 64 - 1) for a, b in zip(k, c)} == want[r]
    sh.free()
    # (d) min over f64 through the shared table (order-preserving transform + hot-key cache flush)
    fv = torch.from_numpy(rng.standard_normal(len(keys))).cuda()
    gotf = gpu_reduce_parts(sc.parallelize((tk, fv), 4).reduce_by_key("min", 3))
    wantf = oracle_reduce("min", keys, fv.cpu().numpy(), 4, 3, "f64")
    assert [{k & (2 ** 64 - 1): v for k, v in d.items()} for d in gotf] == wantf


@pytest.mark.parametrize("kind", ["small_u64", "small_i64_neg", "all_equal", "f64_narrow", "high_bits_only"])
def test_sort_skips_constant_digits(sc, kind):
    """Radix digits on which every key agrees are skipped; the result must still equal the stable oracle sort."""
    rng = np.random.default_rng(17)
    n = 50_000
    kdt = "u64"
    if kind == "small_u64":
        keys = rng.integers(0, 1000, n).astype(np.uint64)
    elif kind == "small_i64_neg":
        keys = rng.integers(-300, 300, n).astype(np.int64); kdt = "i64"
    elif kind == "all_equal":
        keys = np.full(n, 12345, dtype=np.uint64)
    elif kind == "f64_narrow":
        keys = rng.integers(-50, 50, n).astype(np.float64) * 0.5; kdt = "f64"
    else:
        keys = rng.integers(0, 256, n).astype(np.uint64) << np.uint64(56)
    vals = np.arange(n, dtype=np.uint64)
    ok, ov, ps = O.sort_by_key(keys, vals, 4, kdt)
    rdd = sc.parallelize((keys, vals), 3).sort_by_key(4)
    k, v = rdd.collect()
    assert (k == ok).all() and (v == ov).all()
    launches = rdd.stats()["kernels"]["rp_scatter"]["launches"]
    assert launches <= {"small_u64": 2, "small_i64_neg": 8, "all_equal": 1, "f64_narrow": 8, "high_bits_only": 1}[kind]


def _big_gpu():
    import torch
    return torch.cuda.get_device_properties(0).total_memory >= 60 * 2 ** 30


def test_group_by_key_full_size_properties(sc):
    """group_by_key of 5e8 pairs (1e6 keys, 8 partitions: the largest size that leaves an 80 GB GPU room for the
    brute-force checks) through size-independent properties:
    all N values come back, every partition's CSR is consistent, and for sampled keys the value list equals
    the brute-force filter of the input IN INPUT ORDER."""
    import torch
    if not _big_gpu():
        pytest.skip("needs an 80 GB GPU")
    n, D, R = 500_000_000, 1_000_000, 8
    rows = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=0, n=n, mode="uniform", n_distinct=D, seed_k=1, seed_v=2)
    sh = sc.make_rdd(rows, 8).group_by_key(R)._run()
    tot_keys = tot_vals = 0
    checked = 0
    for r in range(R):
        nk, nv = sh.reduce_size(r)
        tot_keys += nk; tot_vals += nv
        if r in (0, 5):
            k = torch.empty(nk, dtype=torch.int64, device="cuda")
            o = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
            v = torch.empty(nv, dtype=torch.int64, device="cuda")
            sh.reduce_device(r, out_keys=k, out_offs=o, out_vals=v)
            assert int(o[0]) == 0 and int(o[-1]) == nv and bool((o[1:] >= o[:-1]).all())
            assert int(torch.unique(k).numel()) == nk
            for j in (0, nk // 2, nk - 1):
                key = int(k[j])
                assert O.get_partition(key & (2 ** 64 - 1), R) == r
                brute = rows[:, 1][rows[:, 0] == key]              # input order
                got = v[int(o[j]):int(o[j + 1])]
                assert got.numel() == brute.numel() and bool((got == brute).all())
                checked += 1
            del k, o, v
    assert tot_keys == D and tot_vals == n and checked == 6
    sh.free()
    del rows
    torch.cuda.empty_cache()


def test_sort_by_key_full_size_properties(sc):
    """configs[2] at 5e8 keys (an 80 GB GPU): sort_by_key of 64-bit keys into 8 partitions: sorted, a permutation of the input
    (sum and xor checksums), partitions are contiguous key ranges that never split a key."""
    import torch
    if not _big_gpu():
        pytest.skip("needs an 80 GB GPU")
    n, R = 500_000_000, 8
    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=keys, first=0, n=n, mode="unique", rank_base=3)
    want_sum = int(keys.sum().item())
    want_xor = 0
    for chunk in keys.split(1 << 27):
        want_xor ^= int(np.bitwise_xor.reduce(chunk.cpu().numpy()))
    sh = sc.parallelize(keys, 8).sort(R)._run()
    got_sum, got_xor, prev_last, tot = 0, 0, None, 0
    for r in range(R):
        nk, _ = sh.reduce_size(r)
        out = torch.empty(nk, dtype=torch.int64, device="cuda")
        sh.reduce_device(r, out_keys=out)
        tot += nk
        # the keys travel as an int64 tensor, i.e. key dtype i64: signed order
        u = out
        assert bool((u[1:] >= u[:-1]).all())
        if prev_last is not None and nk:
            assert int(u[0]) > prev_last                         # contiguous ranges, no key split across partitions
        if nk:
            prev_last = int(u[-1])
        got_sum = (got_sum + int(out.sum().item())) % (1 << 64)
        for chunk in out.split(1 << 27):
            got_xor ^= int(np.bitwise_xor.reduce(chunk.cpu().numpy()))
        del out, u
    assert tot == n and got_sum == want_sum % (1 << 64) and got_xor == want_xor
    sh.free()
    del keys
    torch.cuda.empty_cache()


def test_partition_first_for_tables_larger_than_l2(sc):
    """With > 6.7e6 distinct keys the table passes 2^24 slots (256 MB > L2): rows are first radix-partitioned by the
    top bits of the slot hash so each table region is filled while L2-resident.  Results must not change."""
    import torch
    n_half = 5_000_000
    a = torch.empty((n_half, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=a, first=0, n=n_half, mode="unique", rank_base=0, seed_v=2)
    b = torch.empty((n_half, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=b, first=0, n=n_half, mode="unique", rank_base=1_000_000, seed_v=7)   # 4e6 keys overlap with a
    rows = torch.cat([a, b]).contiguous()
    host = rows.cpu().numpy().view(np.uint64)
    keys, vals = host[:, 0].copy(), host[:, 1].copy()
    for op in ("sum", "max"):
        rdd = sc.make_rdd(rows, 4).reduce_by_key(op, 5)
        got = gpu_reduce_parts(rdd)
        assert rdd.stats()["table_slots"] >= 1 << 24
        got = [{k & (2 ** 64 - 1): v & (2 ** 64 - 1) for k, v in d.items()} for d in got]
        assert got == oracle_reduce(op, keys, vals, 4, 5)
    # host-copied (per-map table) path through build_table as well
    rdd = sc.parallelize((torch.from_numpy(keys.view(np.int64)).cuda().clone(), torch.from_numpy(vals.view(np.int64)).cuda().clone()), 2)
    sh = vb.Shuffle(sc, 2, 3, 0, 0, 4, hint=6_000_000)          # count, explicit hint → 2^24 slots
    st = vb.slice_starts(len(keys), 2)
    for m in range(2):
        sh.map(m, vb.rdd._Col(rdd.keys.owner[int(st[m]):int(st[m + 1])].clone()), None, 0, int(st[m + 1] - st[m]))
    sh.seal()
    got = {}
    for r in range(3):
        k, c = sh.reduce(r)
        got.update(zip((k.view(np.uint64)).tolist(), c.tolist()))
    want = {}
    for d in oracle_reduce("count", keys, None, 2, 3):
        want.update(d)
    assert got == want
    sh.free()


# ---- N3: concurrent map tasks, double-buffered H2D staging, device-resident range source -------------------
def test_concurrent_map_tasks_from_8_threads_match_oracle(sc):
    """vega runs its map tasks concurrently on a blocking pool (local_scheduler.rs:336-352): 8 OS threads submit the
    8 map partitions of ONE shuffle at once (host inputs -> the copy-stream staging path), for a reduce op and a
    group op; results must equal the oracle's, whatever the interleaving."""
    import threading
    from vega_b200 import _lib as L
    from vega_b200.rdd import Shuffle, _Col
    rng = np.random.default_rng(11)
    n, M, R = 400_000, 8, 5
    keys, vals = rand_pairs(rng, n, 20_000)
    starts = vb.slice_starts(n, M)
    for agg, op in ((L.VB_AGG_SUM, "sum"), (L.VB_AGG_GROUP, "group")):
        sh = Shuffle(sc, M, R, L.VB_U64, L.VB_U64, agg)
        kc, vc = _Col(keys), _Col(vals, role="value")
        errs = []

        def task(m):
            try:
                sh.map(m, kc, vc, int(starts[m]), int(starts[m + 1]))
            except Exception as e:      # noqa: BLE001
                errs.append(e)

        ts = [threading.Thread(target=task, args=(m,)) for m in range(M)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errs, errs
        sh.seal()
        if op == "sum":
            want = oracle_reduce("sum", keys, vals, M, R)
            for r in range(R):
                k, c = sh.reduce(r)
                assert dict(zip(k.tolist(), c.tolist())) == want[r]
        else:
            want = oracle_group(keys, vals, M, R)
            for r in range(R):
                k, o, v = sh.reduce(r)
                assert {int(kk): v[int(o[i]):int(o[i + 1])].tolist() for i, kk in enumerate(k)} == want[r]
        sh.free()


def test_host_input_larger_than_both_staging_halves(sc):
    """A host map partition of 20M rows crosses the two 8M-row staging halves more than once (buffer reuse,
    copy-stream/kernel-stream events); checked by sums and key count against numpy."""
    n, D = 20_000_000, 50_000
    rng = np.random.default_rng(5)
    keys = (rng.integers(0, D, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15))
    vals = rng.integers(0, 1 << 20, n).astype(np.uint64)
    k, c = sc.parallelize((keys, vals), 1).reduce_by_key("sum", 3).collect()
    assert len(k) == len(np.unique(keys)) and int(c.sum(dtype=np.uint64)) == int(vals.sum(dtype=np.uint64))
    sample = np.unique(keys)[:: D // 64]
    got = dict(zip(k.tolist(), c.tolist()))
    for s_ in sample.tolist():
        assert got[s_] == int(vals[keys == np.uint64(s_)].sum(dtype=np.uint64))
    rows = np.stack([keys, vals], axis=1)                   # AoS host rows through the same path
    k2, c2 = sc.parallelize(rows, 2).reduce_by_key("sum", 3).collect()
    assert dict(zip(k2.tolist(), c2.tolist())) == got


def test_range_source_is_generated_on_device(sc):
    """Context::range (context.rs:419-431): inclusive end, step; count_by_value / distinct over it."""
    r = sc.range(10, 50, 5, 3)
    assert r.n == 9
    assert sorted(r.distinct().collect().tolist()) == list(range(10, 51, 5))
    k, c = sc.range(0, 999_999, 1, 4).count_by_value().collect()
    assert len(k) == 1_000_000 and (c == 1).all() and int(k.astype(np.uint64).sum()) == 999_999 * 1_000_000 // 2
    assert sc.range(5, 4, 1, 2).n == 0


def test_zipf_hot_key_cache_over_many_tiles_matches_oracle(sc):
    """Enough rows per map task (> 16 tiles per CTA) for the CTAs to finish their learning tiles and keep using
    the hot-key cache and its flush at CTA exit over many tiles: sums, extrema, counts and f64 sums
    must still equal the oracle's for every key."""
    import torch
    n, D = 24_000_000, 200_000
    rows = torch.empty((n, 2), dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_rows=rows, first=0, n=n, mode="zipf", n_distinct=D, seed_k=7, seed_v=3, zipf_s=1.1)
    host = rows.cpu().numpy().view(np.uint64)
    keys, vals = host[:, 0].copy(), host[:, 1].copy()
    for op in ("sum", "max", "min"):
        got = gpu_reduce_parts(sc.make_rdd(rows, 2).reduce_by_key(op, 5))
        got = [{k & (2 ** 64 - 1): v & (2 ** 64 - 1) for k, v in d.items()} for d in got]
        assert got == oracle_reduce(op, keys, vals, 2, 5), op
    got = gpu_reduce_parts(sc.make_rdd(rows, 2).count_by_key(5))
    assert [{k & (2 ** 64 - 1): v for k, v in d.items()} for d in got] == oracle_reduce("count", keys, vals, 2, 5)
    fv = vals.astype(np.float64) / 2 ** 20
    gotf = gpu_reduce_parts(sc.make_rdd((keys, fv), 2).reduce_by_key("sum", 5))      # host SoA input: register/bulk staged path
    assert_f64_sums(gotf, keys, fv, 5, exact=True)         # every key; 20-bit values / 2^20 sum exactly in any order


def _medium_sort_and_group_cases(sc):
    """Sizes at which every part of a radix pass holds several FULL tiles of the gather sweep plus a partial one
    (the small cases above only ever see partial tiles): key-only and (key, value) sorts with every order transform,
    group_by_key from SoA columns and from device AoS rows (ids + values inside 16-byte rows in the first pass)."""
    import torch
    rng = np.random.default_rng(77)
    for kd, n in (("u64", 5_000_003), ("i64", 3_000_001), ("f64", 2_500_000)):
        if kd == "u64":
            k = rng.integers(0, 1 << 63, n).astype(np.uint64) * np.uint64(2) + rng.integers(0, 2, n).astype(np.uint64)
        elif kd == "i64":
            k = rng.integers(-(1 << 62), 1 << 62, n).astype(np.int64)
        else:
            k = rng.standard_normal(n) * 1e9
        k[::5] = k[11]                      # a long run of equal keys: stability across tiles and parts
        v = np.arange(n, dtype=np.uint64)
        ok, ov, ps = O.sort_by_key(k, v, 8, kd)
        gk, gv = sc.parallelize((k, v), 5).sort_by_key(8).collect()
        assert np.array_equal(gk.view(np.uint64), ok.view(np.uint64)) and np.array_equal(gv.view(np.uint64), ov), kd
        gk2, _ = sc.parallelize(k, 3).sort(8).collect()
        assert np.array_equal(gk2.view(np.uint64), ok.view(np.uint64)), kd
    keys, vals = rand_pairs(rng, 4_000_000, 300_000)
    want = oracle_group(keys, vals, 6, 8)
    assert gpu_group_parts(sc.parallelize((keys, vals), 6).group_by_key(8)) == want
    rows = torch.from_numpy(np.stack([keys, vals], axis=1).view(np.int64)).cuda()
    got = gpu_group_parts(sc.parallelize(rows, 6).group_by_key(8))         # int64 rows: keys come back signed
    assert [{k & (2 ** 64 - 1): v for k, v in d.items()} for d in got] == want
    keys, vals = rand_pairs(rng, 3_000_000, 37)           # 37 keys: one pass, runs of ~80k rows per digit
    want = oracle_group(keys, vals, 4, 3)
    assert gpu_group_parts(sc.parallelize((keys, vals), 4).group_by_key(3)) == want
    # the same pass from device AoS rows: its loader keeps the values inside the rows, so the scatter does not record
    # the value-run starts and csr_bounds_kernel derives them over full tiles
    rows = torch.from_numpy(np.stack([keys, vals], axis=1).view(np.int64)).cuda()
    got = gpu_group_parts(sc.parallelize(rows, 4).group_by_key(3))
    assert [{k & (2 ** 64 - 1): v for k, v in d.items()} for d in got] == want


def test_gather_sweep_full_and_partial_tiles_match_oracle(sc):
    st = sc.parallelize(np.arange(3_000_000, dtype=np.uint64)[::-1].copy(), 2).sort(2).stats()
    assert st["kernels"]["rp_scatter"]["launches"] >= 1
    _medium_sort_and_group_cases(sc)
    # 1e5-3e5 rows (every part shorter than one gather-sweep tile): group_by_key from SoA columns and from AoS host rows,
    # key-value and key-only sorts
    rng = np.random.default_rng(21)
    keys, vals = rand_pairs(rng, 300_000, 40_000)
    assert gpu_group_parts(sc.parallelize((keys, vals), 5).group_by_key(6)) == oracle_group(keys, vals, 5, 6)
    rows = np.stack([keys, vals], axis=1)
    assert gpu_group_parts(sc.parallelize(rows, 3).group_by_key(4)) == oracle_group(keys, vals, 3, 4)
    for kd, k in (("u64", rng.integers(0, 1 << 63, 200_001).astype(np.uint64)), ("i64", rng.integers(-(1 << 40), 1 << 40, 99_999).astype(np.int64))):
        v = np.arange(len(k), dtype=np.uint64)
        ok, ov, ps = O.sort_by_key(k, v, 4, kd)
        gk, gv = sc.parallelize((k, v), 3).sort_by_key(4).collect()
        assert np.array_equal(gk.view(np.uint64), ok.view(np.uint64)) and np.array_equal(gv.view(np.uint64), ov), kd
        gk2, _ = sc.parallelize(k, 2).sort(3).collect()
        assert np.array_equal(gk2.view(np.uint64), ok.view(np.uint64)), kd
    st = sc.parallelize((keys, vals), 2).group_by_key(2).stats()
    assert st["kernels"]["rp_scan"]["launches"] >= 1

