"""A sealed reduce_by_key / count_by_key / combine_by_key result as a cogroup and join side under the same partitioner,
with no second shuffle (vb_shuffle_create_narrow: CoGroupedRdd::new's OneToOneDependency, co_grouped_rdd.rs:103-112).

The reference of a view is what vega computes: the cogroup of the parent's result rows taken as an ordinary parent
(tests/cogroup_n_ref.py over the C oracle), so every key once, with the one-element list [its result].  Every partition
is compared element for element and bit for bit (NaN payloads, +-0 and the full u64 range included)."""
import ctypes
import os
import subprocess
import threading
import time

import numpy as np
import pytest

import vega_b200 as vb
from tests import cogroup_n_ref as CN
from tests import join_n_outer_ref as JO
from tests import multirank as MR
from tests.test_gpu_cogroup import abi_parts
from tests.test_gpu_cogroup_n import _u64, abi_parts_n, group_all, join_parts_n, shuffles
from tests.test_gpu_join_n_outer import outer_parts
from tests.test_gpu_outer_join import abi_rows, by_key
from tests.util import EMPTY_KEY, assert_parts_equal, rand_pairs
from vega_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_SHUFFLE = ("hash_agg", "merge", "rp_hist", "rp_scan", "rp_scatter")
OUTER = {"left": 0b01, "right": 0b10, "full": 0b00}


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0, profile=True)
    yield c
    c.close()


def parent(sc, k, v, M, R, op):
    """The sealed reduce shuffle of a reduce_by_key(op) / count_by_key over (k, v) in M slices."""
    rdd = sc.parallelize((k, v), M)
    return (rdd.count_by_key(R) if op == "count" else rdd.reduce_by_key(op, R))._run()


def view(sh, col=0, vcode=None):
    return vb.Shuffle.narrow(sh, col, vcode if vcode is not None else L.VB_U64 if sh.agg == L.VB_AGG_COUNT else sh.vcode)


def result_rows(sh, R, col=None, out_dtypes=None):
    """The parent's result rows over every partition, as u64 bits: the rows the reference feeds to an ordinary cogroup."""
    ks, cs = [np.zeros(0, np.uint64)], [np.zeros(0, np.uint64)]
    for r in range(R):
        if col is None:
            k, c = sh.reduce(r)
        else:
            k, outs = sh.reduce_cols(r, out_dtypes)
            c = outs[col]
        ks.append(_u64(k))
        cs.append(_u64(c))
    return np.concatenate(ks), np.concatenate(cs)


def check_sides(sc, shs, sides, R, key_width=8, masks=True):
    """Every N-way entry point over the sealed sides shs against the reference of their rows sides [(k, v, M)]; for
    two sides also vb_cogroup, vb_join and the three vb_join_outer kinds."""
    want = CN.ref_parts_n(sides, R, key_width)
    assert_parts_equal(abi_parts_n(sc, shs, R, key_width), want)
    assert_parts_equal(join_parts_n(sc, shs, R, key_width), CN.join_of_parts(want))
    for m in (range(1 << len(shs)) if masks else ()):
        assert_parts_equal(outer_parts(sc, shs, R, m, key_width), JO.outer_of_parts(want, m))
    if len(shs) == 2:
        assert_parts_equal(abi_parts(sc, *shs, R, key_width), [{k: tuple(l) for k, l in d.items()} for d in want])
        for kind, mask in [(None, 0b11)] + list(OUTER.items()):
            got = [by_key(*abi_rows(sc, *shs, r, kind)) for r in range(R)]
            assert_parts_equal(got, JO.outer_of_parts(want, mask))
    return want


# ---- 1. every reduce op and value dtype as a view, against lazy and grouped COGROUP shuffles and a second view --------
@pytest.mark.parametrize("op,vdtype", [(op, dt) for op in ("sum", "min", "max") for dt in ("u64", "i64", "f64")] + [("count", "u64")])
def test_every_op_and_dtype(sc, op, vdtype):
    rng = np.random.default_rng(len(op) * 7 + len(vdtype))
    values = "special" if vdtype == "f64" else "full"
    R = 4
    ka, va = rand_pairs(rng, 12_000, 1500, vdtype=vdtype, values=values)
    kb, vb_ = rand_pairs(rng, 8000, 2000, vdtype=vdtype, values=values)
    kc, vc = rand_pairs(rng, 6000, 1200, values="full")
    pa, pb = parent(sc, ka, va, 3, R, op), parent(sc, kb, vb_, 2, R, op)
    va_sh, vb_sh = view(pa), view(pb)
    ra, rb = (*result_rows(pa, R), 1), (*result_rows(pb, R), 1)
    side_c = (kc, vc, 3)
    lazy = lambda: shuffles(sc, [side_c], R)[0]
    grouped = shuffles(sc, [side_c], R)[0]
    group_all([grouped], R)
    for shs, sides in [([va_sh, lazy()], [ra, side_c]), ([lazy(), va_sh], [side_c, ra]),
                       ([va_sh, grouped], [ra, side_c]), ([grouped, va_sh], [side_c, ra]),
                       ([va_sh, vb_sh], [ra, rb]), ([vb_sh, va_sh], [rb, ra]),
                       ([va_sh, lazy(), vb_sh], [ra, side_c, rb])]:
        check_sides(sc, shs, sides, R)
    # the view reads back as the parent's result with offsets 0..n
    for r in range(R):
        k, c = pa.reduce(r)
        vk, vo, vv = va_sh.reduce(r)
        assert _u64(vk).tolist() == _u64(k).tolist() and vo.tolist() == list(range(len(k) + 1))
        assert _u64(vv).tolist() == _u64(c).tolist()


# ---- 2. combine_by_key: every output column of a 4-column x 8-aggregate spec, MEAN included ----------------------------
def test_combine_by_key_columns(sc):
    rng = np.random.default_rng(20)
    n, R = 20_000, 5
    k, _ = rand_pairs(rng, n, 2500, values="full")
    cols = (rng.integers(0, 1 << 64, n, dtype=np.uint64), rng.integers(-(1 << 62), 1 << 62, n).astype(np.int64),
            rng.standard_normal(n), rng.integers(0, 1000, n).astype(np.uint64))
    aggs = {"s0": ("sum", 0), "mn1": ("min", 1), "mx2": ("max", 2), "n": ("count", None), "avg0": ("mean", 0),
            "avg1": ("mean", 1), "avg2": ("mean", 2), "s3": ("sum", 3)}
    comb = sc.parallelize(k, 3, values=cols).combine_by_key(aggs, R)
    sh = comb._run()
    kc, vc = rand_pairs(rng, 7000, 2500)
    side_c = (kc, vc, 2)
    views = [view(sh, i, {np.uint64: L.VB_U64, np.int64: L.VB_I64, np.float64: L.VB_F64}[dt]) for i, dt in enumerate(comb.out_dtypes)]
    for i, v in enumerate(views):                              # several views of one parent coexist
        rows = (*result_rows(sh, R, i, comb.out_dtypes), 1)
        check_sides(sc, [v, shuffles(sc, [side_c], R)[0]], [rows, side_c], R, masks=False)
    # and every aggregate as a mirror parent at once
    cg = vb.CoGroupedRdd([comb.aggregate(nm) for nm in comb.names], R)
    want = CN.ref_parts_n([(*result_rows(sh, R, i, comb.out_dtypes), 1) for i in range(len(comb.names))], R)
    assert_parts_equal(abi_parts_n(sc, cg._run(), R), want)


# ---- 3. keys and partitions: 0 and 2^64-1, 4-byte keys, R = 1 and 300, empty parent, empty partitions ----------------
@pytest.mark.parametrize("R", [1, 300])
def test_extreme_keys_and_partition_counts(sc, R):
    rng = np.random.default_rng(R)
    ka, va = rand_pairs(rng, 3000, 200, values="full")          # includes keys 0 and 2^64-1; R = 300 leaves partitions empty
    assert {0, EMPTY_KEY} <= set(ka.tolist())
    kb, vb_ = rand_pairs(rng, 2000, 300, values="full")
    pa = parent(sc, ka, va, 2, R, "sum")
    v = view(pa)
    assert v.stats()["table_restarts"] == 0
    check_sides(sc, [v, shuffles(sc, [(kb, vb_, 3)], R)[0]], [(*result_rows(pa, R), 1), (kb, vb_, 3)], R, masks=R == 1)
    if R == 300:
        assert sum(1 for r in range(R) if pa.reduce_size(r)[0] == 0) > 0


def test_int32_keys(sc):
    rng = np.random.default_rng(31)
    ka, kb = rng.integers(-2000, 1000, 20_000).astype(np.int32), rng.integers(0, 3000, 15_000).astype(np.int32)
    va, vb_ = rng.integers(0, 1 << 62, len(ka)).astype(np.uint64), rng.integers(0, 1 << 62, len(kb)).astype(np.uint64)
    R = 5
    pa = parent(sc, ka, va, 3, R, "max")
    lazy = vb.CoGroupedRdd([sc.parallelize((kb, vb_), 2)], R)._run()[0]
    check_sides(sc, [view(pa), lazy], [(*result_rows(pa, R), 1), (kb, vb_, 2)], R, key_width=4, masks=False)


def test_empty_parent(sc):
    rng = np.random.default_rng(32)
    e = np.zeros(0, np.uint64)
    kb, vb_ = rand_pairs(rng, 2000, 300)
    R = 3
    pe = parent(sc, e, e, 2, R, "sum")
    ve = view(pe)
    assert all(ve.reduce_size(r) == (0, 0) for r in range(R))
    check_sides(sc, [ve, shuffles(sc, [(kb, vb_, 2)], R)[0]], [(e, e, 1), (kb, vb_, 2)], R)
    check_sides(sc, [ve, view(pe)], [(e, e, 1), (e, e, 1)], R)


# ---- 4. narrow equals reshuffle: the view-based join equals the join of the result rows shuffled as a PairRdd ---------
def test_narrow_equals_reshuffle(sc):
    rng = np.random.default_rng(40)
    R = 6
    ka, va = rand_pairs(rng, 15_000, 2000, values="full")
    kb, vb_ = rand_pairs(rng, 10_000, 3000, values="full")
    pa, pb = sc.parallelize((ka, va), 3).reduce_by_key("sum", R), sc.parallelize((kb, vb_), 2).count_by_key(R)
    (ra, ca), (rb, cb) = pa.collect(), pb.collect()
    ha, hb = sc.parallelize((ra, ca), 4), sc.parallelize((rb, cb), 1)          # the result rows as ordinary parents
    for narrow, shuffled in [(pa.join(pb, R), ha.join(hb, R)), (pa.cogroup(pb, R), ha.cogroup(hb, R))]:
        for r in range(R):
            assert sorted(zip(*[_u64(x).tolist() for x in narrow.compute(r)])) == \
                sorted(zip(*[_u64(x).tolist() for x in shuffled.compute(r)]))
            nk, (nlo, nlv), (nro, nrv) = narrow.cogroup_compute(r)
            sk, (slo, slv), (sro, srv) = shuffled.cogroup_compute(r)
            per_key = lambda k, lo, lv, ro, rv: {int(x): (lv[lo[i]:lo[i + 1]].tolist(), rv[ro[i]:ro[i + 1]].tolist())
                                                for i, x in enumerate(_u64(k))}
            assert per_key(nk, nlo, _u64(nlv), nro, _u64(nrv)) == per_key(sk, slo, _u64(slv), sro, _u64(srv))
    for kind in OUTER:
        narrow, shuffled = getattr(pa, f"{kind}_outer_join")(pb, R), getattr(ha, f"{kind}_outer_join")(hb, R)
        rows = lambda j: sorted(zip(*[_u64(np.ma.getdata(x)).tolist() for x in j.collect()]))
        assert rows(narrow) == rows(shuffled)


# ---- 5. no shuffle ran; the parent is unchanged; either can be freed first ------------------------------------------
def test_no_shuffle_and_lifetimes(sc):
    rng = np.random.default_rng(50)
    R = 4
    ka, va = rand_pairs(rng, 20_000, 3000, values="full")
    kb, vb_ = rand_pairs(rng, 8000, 3000, values="full")
    pa = parent(sc, ka, va, 3, R, "sum")
    before = [tuple(_u64(x).tolist() for x in pa.reduce(r)) for r in range(R)]
    rows = (*result_rows(pa, R), 1)
    v1, v2 = view(pa), view(pa)
    kt = v1.stats()["kernels"]
    assert all(kt[c]["launches"] == 0 for c in NO_SHUFFLE), kt
    assert kt["dict"]["launches"] >= 1
    assert [tuple(_u64(x).tolist() for x in pa.reduce(r)) for r in range(R)] == before
    side_b = (kb, vb_, 2)
    pa.free()                                                  # the parent first: the views own their copies
    check_sides(sc, [v1, shuffles(sc, [side_b], R)[0]], [rows, side_b], R, masks=False)
    v2.free()
    check_sides(sc, [v1, shuffles(sc, [side_b], R)[0]], [rows, side_b], R, masks=False)
    pc = parent(sc, kb, vb_, 2, R, "min")
    rows_c = (*result_rows(pc, R), 1)
    before_c = [tuple(_u64(x).tolist() for x in pc.reduce(r)) for r in range(R)]
    vc = view(pc)
    vc.free()                                                  # the view first: the parent still reads and views again
    assert [tuple(_u64(x).tolist() for x in pc.reduce(r)) for r in range(R)] == before_c
    check_sides(sc, [view(pc), v1], [rows_c, rows], R, masks=False)


# ---- 6. multi-rank in one process: a SUM and a COGROUP shuffle per rank, a view per rank ---------------------------------
@pytest.mark.parametrize("W", [2, 3, 8])
def test_multirank(sc, W):
    import torch
    from vega_b200.dist import CudaEngine
    rng = np.random.default_rng(60 + W)
    R, M = 2 * W + 1, 2 * W
    ka, va = rand_pairs(rng, 20_000, 3000, values="full")
    kb, vb_ = rand_pairs(rng, 12_000, 3000, values="full")
    dev = lambda x: torch.from_numpy(x.view(np.int64)).cuda()
    ta, tva, tb, tvb = dev(ka), dev(va), dev(kb), dev(vb_)
    eng = CudaEngine(sc)
    sums, _ = MR.run_ranks(eng, W, L.VB_AGG_SUM, MR.maps_by_rank(len(ka), M, W, lambda m, lo, hi: (ta[lo:hi], tva[lo:hi])),
                           R, L.VB_U64, L.VB_U64)
    cogs, _ = MR.run_ranks(eng, W, L.VB_AGG_COGROUP, MR.maps_by_rank(len(kb), M, W, lambda m, lo, hi: (tb[lo:hi], tvb[lo:hi])),
                           R, L.VB_U64, L.VB_U64)
    # the single-process reference: numpy's wrapping sum per key, then the cogroup with the COGROUP side
    uk, inv = np.unique(ka, return_inverse=True)
    s = np.zeros(len(uk), np.uint64)
    np.add.at(s, inv, va)
    want = CN.ref_parts_n([(uk, s, 1), (kb, vb_, M)], R)
    got = [dict() for _ in range(R)]
    got_j = [dict() for _ in range(R)]
    for d in range(W):
        v = view(sums[d])
        parts = abi_parts_n(sc, [v, cogs[d]], R)
        joins = join_parts_n(sc, [v, cogs[d]], R)
        for r in range(R):
            if r % W == d:
                got[r], got_j[r] = parts[r], joins[r]
            else:
                assert not parts[r] and not joins[r], f"rank {d} has keys of partition {r}"
    assert_parts_equal(got, want)
    assert_parts_equal(got_j, CN.join_of_parts(want))


# ---- 7. blocking and rejected calls ----------------------------------------------------------------------------------
def test_blocks_until_sealed(sc):
    rng = np.random.default_rng(70)
    k, v = rand_pairs(rng, 5000, 700)
    R = 3
    sh = vb.Shuffle(sc, 1, R, L.VB_U64, L.VB_U64, L.VB_AGG_SUM)
    sh.map(0, vb.rdd._Col(k), vb.rdd._Col(v, role="value"), 0, len(k))
    box = {}
    t = threading.Thread(target=lambda: box.setdefault("v", view(sh)))
    t.start()
    time.sleep(0.5)
    assert t.is_alive() and "v" not in box, "the view did not wait for the seal"
    sh.seal()
    t.join(60)
    assert not t.is_alive()
    check_sides(sc, [box["v"], view(sh)], [(*result_rows(sh, R), 1)] * 2, R, masks=False)


def test_rejected_calls(sc):
    rng = np.random.default_rng(71)
    k, v = rand_pairs(rng, 3000, 400)
    R = 3
    lib = sc._lib
    ps = parent(sc, k, v, 2, R, "sum")
    before = [tuple(_u64(x).tolist() for x in ps.reduce(r)) for r in range(R)]
    grp = sc.parallelize((k, v), 2).group_by_key(R)._run()
    cog = shuffles(sc, [(k, v, 2)], R)[0]
    srt = sc.parallelize((k, v), 2).sort_by_key(R)._run()
    strs = sc.parallelize(["a", "b", "a"], 1, values=np.arange(3, dtype=np.uint64)).reduce_by_key("sum", 2)._run()
    comb = sc.parallelize(k, 2, values=(v,)).combine_by_key({"s": ("sum", 0), "n": ("count", None)}, R)._run()
    vw = view(ps)
    out = ctypes.c_void_p()
    calls = [(None, 0, ctypes.byref(out)), (ps._h, 0, None), (grp._h, 0, ctypes.byref(out)), (cog._h, 0, ctypes.byref(out)),
             (vw._h, 0, ctypes.byref(out)), (srt._h, 0, ctypes.byref(out)), (strs._h, 0, ctypes.byref(out)),
             (ps._h, 1, ctypes.byref(out)), (comb._h, 2, ctypes.byref(out))]
    for h, col, o in calls:
        assert lib.vb_shuffle_create_narrow(h, col, o) == L.VB_ERR_INVALID, (h, col)
    assert [tuple(_u64(x).tolist() for x in ps.reduce(r)) for r in range(R)] == before
    check_sides(sc, [view(ps), view(comb, 1, L.VB_U64)], [(*result_rows(ps, R), 1), (*result_rows(comb, R, 1, [np.uint64] * 2), 1)],
                R, masks=False)


# ---- 8. scale: parents of 5e7 rows with 1e7 keys per side, 2 % of them shared ---------------------------------------
def test_scale(sc):
    import torch
    n, D, R = 50_000_000, 10_000_000, 8
    g = torch.Generator(device="cuda").manual_seed(8)
    ra = torch.randint(0, D, (n,), device="cuda", generator=g)
    rb = torch.randint(0, D, (n,), device="cuda", generator=g) + int(D * 0.98)      # ranks [0.98 D, D) are on both sides
    mul = 0x9E3779B97F4A7C15 - (1 << 64)
    ka, kb = ra * mul + 12345, rb * mul + 12345
    va = torch.randint(0, 1 << 40, (n,), device="cuda", generator=g)
    vb_ = torch.randint(0, 1 << 40, (n,), device="cuda", generator=g)
    torch.cuda.synchronize()
    a = sc.parallelize((ka, va), 16).reduce_by_key("sum", R)
    b = sc.parallelize((kb, vb_), 16).reduce_by_key("sum", R)
    k, v, w = a.join(b, R).collect()

    def sums(keys, vals):
        uk, inv = np.unique(keys.cpu().numpy().view(np.uint64), return_inverse=True)
        s = np.zeros(len(uk), np.uint64)
        np.add.at(s, inv, vals.cpu().numpy().view(np.uint64))
        return uk, s
    (ua, sa), (ub, sb) = sums(ka, va), sums(kb, vb_)
    both, ia, ib = np.intersect1d(ua, ub, return_indices=True)
    order = np.argsort(_u64(k))
    assert np.array_equal(_u64(k)[order], both)
    assert np.array_equal(_u64(v)[order], sa[ia]) and np.array_equal(_u64(w)[order], sb[ib])
    assert len(both) > 100_000


# ---- 9. the mirrors -----------------------------------------------------------------------------------------------
def test_mirror_parents(sc):
    rng = np.random.default_rng(90)
    R = 5
    ka, va = rand_pairs(rng, 12_000, 1500, vdtype="i64", values="full")
    kb, vb_ = rand_pairs(rng, 9000, 2000, values="full")
    kc, vc = rand_pairs(rng, 7000, 1800, vdtype="f64")
    a, b, c = sc.parallelize((ka, va), 3), sc.parallelize((kb, vb_), 2), sc.parallelize((kc, vc), 4)
    sa, nb = a.reduce_by_key("sum", R), b.count_by_key(R)
    rows_a, rows_b = (*map(_u64, sa.collect()), 1), (*map(_u64, nb.collect()), 1)
    # reduce_by_key(...).join(...) and count_by_key().cogroup(...)
    j = sa.join(nb, R)
    want = CN.ref_parts_n([rows_a, rows_b], R)
    got_j = [{} for _ in range(R)]
    for r in range(R):
        k, v, w = j.compute(r)
        assert v.dtype == np.int64 and w.dtype == np.uint64
        for x, y, z in zip(_u64(k).tolist(), _u64(v).tolist(), _u64(w).tolist()):
            got_j[r].setdefault(x, []).append((y, z))
    assert_parts_equal(got_j, CN.join_of_parts(want))
    cg = nb.cogroup(c, R)
    want_cg = CN.ref_parts_n([rows_b, (kc, vc, 4)], R)
    got_cg = []
    for r in range(R):
        keys, (lo, lv), (ro, rv) = cg.cogroup_compute(r)
        got_cg.append({x: (_u64(lv)[lo[i]:lo[i + 1]].tolist(), _u64(rv)[ro[i]:ro[i + 1]].tolist()) for i, x in enumerate(_u64(keys).tolist())})
    assert_parts_equal(got_cg, [{k: tuple(l) for k, l in d.items()} for d in want_cg])
    # a PairRdd joined with a result, and CoGroupedRdd with three mixed parents
    assert sorted(zip(*[_u64(x).tolist() for x in c.join(sa, R).collect()])) == \
        sorted((k, *row) for d in CN.join_of_parts(CN.ref_parts_n([(kc, vc, 4), rows_a], R)) for k, rows in d.items() for row in rows)
    mixed = vb.CoGroupedRdd([sa, c, nb], R)
    assert_parts_equal(abi_parts_n(sc, mixed._run(), R), CN.ref_parts_n([rows_a, (kc, vc, 4), rows_b], R))


@pytest.mark.parametrize("R2", [3, 7])
def test_mirror_reshuffle_path(sc, R2):
    """Parents with another num_splits: each result partition is one map task of a COGROUP shuffle, read on the device."""
    rng = np.random.default_rng(91 + R2)
    ka, va = rand_pairs(rng, 12_000, 1500, values="full")
    kb, vb_ = rand_pairs(rng, 9000, 2000, values="full")
    k2 = rng.integers(0, 1 << 63, 5000).astype(np.uint64)
    sa = sc.parallelize((ka, va), 3).reduce_by_key("max", 5)
    comb = sc.parallelize(kb, 2, values=(vb_, vb_)).combine_by_key({"lo": ("min", 1), "avg": ("mean", 0)}, 4)
    b = sc.parallelize((k2, k2), 2)
    cg = vb.CoGroupedRdd([sa, comb.aggregate("avg"), b], R2)
    shs = cg._run()
    assert not any(s.n_map == 0 for s in shs[:2]), "another num_splits must reshuffle"
    k, v = sa.collect()
    kk, aggs = comb.collect()
    want = CN.ref_parts_n([(_u64(k), _u64(v), 5), (_u64(kk), _u64(aggs["avg"]), 4), (k2, k2, 2)], R2)
    assert_parts_equal(abi_parts_n(sc, shs, R2), want)


def test_cpp_narrow_join_example_runs():
    """examples/narrow_join.cpp: two reduce_by_key results joined, cogrouped with a third and left-outer-joined without a
    second shuffle; exit 0 only on the expected rows."""
    path = os.path.join(ROOT, "examples", "_build", "narrow_join")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    out = subprocess.run([path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "join: [(1, (21, 201)), (5, (50, 5))]" in out.stdout, out.stdout
    assert "(2, [20, None, 15])" in out.stdout, out.stdout
