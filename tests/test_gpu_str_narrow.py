"""A sealed String reduce_by_key / count_by_key / combine_by_key result as a cogroup and join side under the same
partitioner, with no second shuffle (vb_shuffle_create_narrow_str: CoGroupedRdd::new's OneToOneDependency over `String`
keys, co_grouped_rdd.rs:103-112).

The reference of a view is what vega computes: the cogroup of the parent's result rows taken as an ordinary parent, so
every key once, with the one-element list [its result].  That reference is an ordinary String GROUP shuffle mapped from
the parent's result rows; for UTF-8 keys the Python references of tests/test_gpu_str_join.py check it as well.  Key
order within a partition is unspecified, so partitions are compared as maps from key bytes to lists or rows; values are
compared bit for bit (NaN payloads, +-0 and the full u64 range included)."""
import ctypes
import os
import subprocess
import threading
import time

import numpy as np
import pytest

import vega_b200 as vb
from tests.test_gpu_str_join import POOL, check_cogroup, check_join, cogroup_part, join_part, words
from tests.test_gpu_str_keys import _device_words
from vega_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHUFFLE_CLASSES = ("hash_agg", "dict", "merge", "rp_hist", "rp_scan", "rp_scatter")
_NP = {L.VB_U64: np.uint64, L.VB_I64: np.int64, L.VB_F64: np.float64}
_CODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0, profile=True)
    yield c
    c.close()


# ---- helpers --------------------------------------------------------------------------------------------------------
def values(rng, n, dt):
    if dt == "u64":
        return rng.integers(0, 1 << 64, n, dtype=np.uint64)
    if dt == "i64":
        return rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
    v = rng.standard_normal(n) * 1e3
    special = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, np.float64(1e308), -np.float64(5e-324)])
    v[:: max(1, n // 40)] = np.resize(special, len(v[:: max(1, n // 40)]))
    bits = v.view(np.uint64).copy()
    bits[1::97] = np.uint64(0x7FF8_0000_0000_0001)          # NaN with a payload
    bits[2::101] = np.uint64(0xFFF0_0000_0000_0042)         # negative signalling NaN
    return bits.view(np.float64)


def str_parent(sc, keys, vals, M, R, op):
    """The sealed String reduce shuffle of reduce_by_key(op) / count_by_key over (keys, vals) in M slices."""
    rdd = sc.parallelize(keys, M, values=vals)
    return (rdd.count_by_key(R) if op == "count" else rdd.reduce_by_key(op, R))._run()


def comb_parent(sc, keys, cols, M, R, aggs):
    return sc.parallelize(keys, M, values=tuple(cols)).combine_by_key(aggs, R)


def view(sh, col=0, vcode=None):
    return vb.StrShuffle.narrow(sh, col, vcode if vcode is not None else L.VB_U64 if sh.agg == L.VB_AGG_COUNT else sh.vcode)


def _kb(ko, kb, i):
    return bytes(kb[int(ko[i]):int(ko[i + 1])])


def result_parts(sh, R, col=None, out_dtypes=None):
    """Per partition {key bytes: result bits} of the parent (one column of a combine with col / out_dtypes)."""
    out = []
    for r in range(R):
        if col is None:
            ko, kb, comb = sh.reduce_raw(r)
        else:
            ko, kb, outs = sh.reduce_cols(r, out_dtypes)
            comb = outs[col]
        bits = np.asarray(comb).view(np.uint64).tolist()
        d = {_kb(ko, kb, i): bits[i] for i in range(len(ko) - 1)}
        assert len(d) == len(ko) - 1
        out.append(d)
    return out


def check_view_reads(v, parts):
    """vb_shuffle_reduce_str(_size) of every view partition: the parent's keys, offsets 0..n, the column bit for bit."""
    for r, want in enumerate(parts):
        nk, nb, nv = v.reduce_size(r)
        assert nk == nv == len(want) and nb == sum(len(k) for k in want), r
        ko, kb, offs, vals = v.reduce_raw(r)
        assert ko[0] == 0 and np.array_equal(offs, np.arange(nk + 1, dtype=np.uint64)), r
        got = {_kb(ko, kb, i): x for i, x in enumerate(np.asarray(vals).view(np.uint64).tolist())}
        assert got == want, r


def rows_side(sc, parts, vcode, R):
    """The parent's result rows taken as an ordinary parent: a String GROUP shuffle mapped from them (one map task per
    result partition, key bytes as they are)."""
    sh = vb.StrShuffle(sc, max(1, len(parts)), R, vcode, L.VB_AGG_GROUP)
    for m, d in enumerate(parts):
        ks = list(d)
        offs = np.zeros(len(ks) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(k) for k in ks], dtype=np.uint64)
        keys = vb.StrKeys(offs, np.frombuffer(b"".join(ks), dtype=np.uint8).copy())
        vals = np.array([d[k] for k in ks], dtype=np.uint64).view(_NP[vcode])
        sh.map(m, vb.rdd._StrCol(keys), vb.rdd._Col(vals, role="value"), 0, len(ks))
    sh.seal()
    return sh


def _arr(shs):
    return (ctypes.c_void_p * len(shs))(*[s._h.value for s in shs])


def cogroup_map(sc, shs, R):
    """Per partition {key bytes: [list of each side as u64 bits]} through vb_cogroup_n_str(_size); every key in the
    partition vb_get_partition_str places it in."""
    out = []
    for r in range(R):
        keys, lists, ko = cogroup_part(sc, shs, r)
        d = {}
        for i, k in enumerate(keys):
            kb = k.encode("utf-8", "surrogateescape")
            assert sc._lib.vb_get_partition_str(kb, len(kb), R) == r, (r, kb)
            d[kb] = [v[int(o[i]):int(o[i + 1])].tolist() for o, v in lists]
        assert len(d) == len(keys), f"a key twice in partition {r}"
        out.append(d)
    return out


def join_map(sc, shs, R, mask):
    """Per partition {key bytes: [(v_0, .., v_{n-1}, valid_0, ..) per row]} through vb_join_n_str(_size)."""
    out = []
    for r in range(R):
        keys, ro, vs, ok, _, nrows = join_part(sc, shs, r, mask)
        assert int(ro[-1]) == nrows if len(keys) else nrows == 0
        d = {}
        for i, k in enumerate(keys):
            a, b = int(ro[i]), int(ro[i + 1])
            d[k.encode("utf-8", "surrogateescape")] = [tuple(int(x[j]) for x in vs + ok) for j in range(a, b)]
        assert len(d) == len(keys)
        out.append(d)
    return out


def check_same(sc, shs, ref, R, masks=None):
    """Every String cogroup and join entry point over shs equals the same call over the reference sides ref."""
    got = cogroup_map(sc, shs, R)
    assert got == cogroup_map(sc, ref, R)
    for m in (range(1 << len(shs)) if masks is None else masks):
        assert join_map(sc, shs, R, m) == join_map(sc, ref, R, m), m
    return got


def _launches(sh):
    return {k: v["launches"] for k, v in sh.stats()["kernels"].items()}


# ---- 1. every reduce op and value dtype ------------------------------------------------------------------------------
@pytest.mark.parametrize("op,dt", [(op, dt) for op in ("sum", "min", "max") for dt in ("u64", "i64", "f64")] + [("count", "u64")])
def test_every_op_and_dtype(sc, op, dt):
    rng = np.random.default_rng(10 * ("sum", "min", "max", "count").index(op) + ("u64", "i64", "f64").index(dt))
    R = 5
    ka, kb_ = words(rng, 4000, POOL), words(rng, 1500, POOL[4:] + ["b-only"])
    va, vb_ = values(rng, len(ka), dt), values(rng, len(kb_), "u64")
    pa = str_parent(sc, ka, va, 3, R, op)
    pb = str_parent(sc, kb_, vb_, 2, R, "sum")
    parts_a, parts_b = result_parts(pa, R), result_parts(pb, R)
    va_, vb2 = view(pa), view(pb)
    assert va_.vcode == (L.VB_U64 if op == "count" else _CODE[dt])
    check_view_reads(va_, parts_a)
    check_view_reads(vb2, parts_b)
    g = sc.parallelize(words(rng, 2000, POOL), 2, values=values(rng, 2000, "u64")).group_by_key(R)._run()
    ra, rb = rows_side(sc, parts_a, va_.vcode, R), rows_side(sc, parts_b, L.VB_U64, R)
    check_same(sc, [va_, g], [ra, g], R)                      # a view next to a GROUP side
    check_same(sc, [g, va_, vb2], [g, ra, rb], R)             # views next to a GROUP side, n = 3
    check_same(sc, [va_, vb2], [ra, rb], R)                   # view with view
    check_same(sc, [va_, g, va_], [ra, g, ra], R)             # one view used twice
    # the Python reference of the result rows as an ordinary parent
    data = [([k.decode() for d in parts_a for k in d], np.array([x for d in parts_a for x in d.values()], dtype=np.uint64)),
            ([k.decode() for d in parts_b for k in d], np.array([x for d in parts_b for x in d.values()], dtype=np.uint64))]
    check_cogroup(sc, [va_, vb2], data, R)
    for mask in range(4):
        check_join(sc, [va_, vb2], data, R, mask)


# ---- 2. every combine_by_key column -----------------------------------------------------------------------------------
def test_combine_columns(sc):
    rng = np.random.default_rng(20)
    R, n = 6, 5000
    keys = words(rng, n, POOL)
    cols = [values(rng, n, "u64"), values(rng, n, "i64"), values(rng, n, "f64")]
    aggs = {"s": ("sum", 0), "lo": ("min", 1), "hi": ("max", 2), "avg": ("mean", 2), "n": ("count", None), "fs": ("sum", 2)}
    comb = comb_parent(sc, keys, cols, 3, R, aggs)
    sh = comb._run()
    vs, refs = [], []
    for i, name in enumerate(comb.names):
        col, n_cols, vcode = comb.aggregate(name)._result_col(sh)
        assert (col, n_cols) == (i, len(aggs))
        parts = result_parts(sh, R, col, comb.out_dtypes)
        v = view(sh, col, vcode)
        assert v.vcode == {"s": L.VB_U64, "lo": L.VB_I64, "hi": L.VB_F64, "avg": L.VB_F64, "n": L.VB_U64, "fs": L.VB_F64}[name]
        check_view_reads(v, parts)
        vs.append(v)
        refs.append(rows_side(sc, parts, vcode, R))
    check_same(sc, vs, refs, R, masks=(0, (1 << len(vs)) - 1, 0b000101, 0b100000))
    check_same(sc, [vs[3], vs[4]], [refs[3], refs[4]], R)     # MEAN and COUNT, every mask
    red = str_parent(sc, keys, cols[0], 2, R, "max")           # a reduce view next to combine views
    check_same(sc, [vs[0], view(red), vs[3]], [refs[0], rows_side(sc, result_parts(red, R), L.VB_U64, R), refs[3]], R)


# ---- 3. the device reshuffle and the views give the same results --------------------------------------------------------
def test_views_equal_the_reshuffle(sc):
    rng = np.random.default_rng(30)
    R = 7
    ka, kb_ = words(rng, 3000, POOL), words(rng, 3000, POOL[10:])
    pa = sc.parallelize(ka, 3, values=values(rng, len(ka), "i64")).reduce_by_key("min", R)
    comb = comb_parent(sc, kb_, [values(rng, len(kb_), "f64")], 2, R, {"avg": ("mean", 0), "n": ("count", None)})
    cg = vb.StrCoGroupedRdd([pa], R)
    resh = [cg._reshuffled(pa._run(), 0, None, L.VB_I64), cg._reshuffled(comb._run(), 0, 2, L.VB_F64),
            cg._reshuffled(comb._run(), 1, 2, L.VB_U64)]
    views = [view(pa._run()), view(comb._run(), 0, L.VB_F64), view(comb._run(), 1, L.VB_U64)]
    check_same(sc, views, resh, R)
    check_same(sc, views[1:], resh[1:], R)


# ---- 4. key shapes, partition counts, empty parents and partitions ---------------------------------------------------------
def _raw_keys(ks):
    offs = np.zeros(len(ks) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(k) for k in ks], dtype=np.uint64)
    return vb.StrKeys(offs, np.frombuffer(b"".join(ks), dtype=np.uint8).copy())


@pytest.mark.parametrize("R", [1, 4, 300])
def test_key_shapes(sc, R):
    rng = np.random.default_rng(40 + R)
    shapes = [b""] + [b"k" * n for n in range(1, 9)] + [b"z" * 1024, b"z" * 1023 + b"y", b"z" * 4000] + \
             [b"\x00", b"\x00\x00", b"a\x00b", b"\xff", b"\xff\xfe\x00", b"ab", b"abc", b"abcd", b"a", b"abd", "日本".encode()]
    ks = [shapes[i] for i in rng.integers(0, len(shapes), 3000)]
    pa = sc.parallelize(_raw_keys(ks), 3, values=values(rng, len(ks), "u64")).reduce_by_key("sum", R)._run()
    pc = sc.parallelize(_raw_keys(ks[::3]), 2, values=np.zeros(len(ks[::3]), dtype=np.uint64)).count_by_key(R)._run()
    parts_a, parts_c = result_parts(pa, R), result_parts(pc, R)
    assert sorted(k for d in parts_a for k in d) == sorted(set(ks))
    va_, vc = view(pa), view(pc)
    check_view_reads(va_, parts_a)
    check_view_reads(vc, parts_c)
    g = sc.parallelize(_raw_keys(ks[1::2]), 2, values=values(rng, len(ks[1::2]), "u64")).group_by_key(R)._run()
    ra, rc = rows_side(sc, parts_a, L.VB_U64, R), rows_side(sc, parts_c, L.VB_U64, R)
    check_same(sc, [va_, vc, g], [ra, rc, g], R, masks=(0, 0b111, 0b001, 0b110) if R == 300 else None)
    if R == 300:                                              # more partitions than keys: most are empty
        assert sum(1 for d in parts_a if not d) > 250


def test_empty_parent_and_empty_partitions(sc):
    R = 6
    empty = sc.parallelize(vb.StrKeys.from_strs([]), 2, values=np.zeros(0, dtype=np.uint64)).reduce_by_key("sum", R)._run()
    ve = view(empty)
    assert all(ve.reduce_size(r) == (0, 0, 0) for r in range(R))
    check_view_reads(ve, [{} for _ in range(R)])
    one = str_parent(sc, ["only"] * 5, np.arange(5, dtype=np.uint64), 2, R, "sum")  # one key: R - 1 empty partitions
    parts = result_parts(one, R)
    assert sum(1 for d in parts if d) == 1
    vo = view(one)
    check_view_reads(vo, parts)
    g = sc.parallelize(["only", "x", "y"], 1, values=np.arange(3, dtype=np.uint64)).group_by_key(R)._run()
    check_same(sc, [ve, vo, g], [rows_side(sc, [{} for _ in range(R)], L.VB_U64, R), rows_side(sc, parts, L.VB_U64, R), g], R)
    check_same(sc, [ve], [rows_side(sc, [{} for _ in range(R)], L.VB_U64, R)], R)


# ---- 5. no shuffle work, the lazy index, lifetimes ------------------------------------------------------------------------
def test_no_shuffle_work_and_lifetimes(sc):
    rng = np.random.default_rng(50)
    R = 4
    ka, kb_ = words(rng, 20_000, POOL), words(rng, 8000, POOL)
    pa = str_parent(sc, ka, values(rng, len(ka), "u64"), 3, R, "sum")
    parts_a = result_parts(pa, R)
    v1, v2 = view(pa), view(pa)
    for v in (v1, v2):
        kt = _launches(v)
        assert all(kt[c] == 0 for c in SHUFFLE_CLASSES), kt       # copies and one range_kernel (misc) only
    assert result_parts(pa, R) == parts_a                          # the parent is unchanged
    g = sc.parallelize(kb_, 2, values=values(rng, len(kb_), "u64")).group_by_key(R)._run()
    ref = [rows_side(sc, parts_a, L.VB_U64, R), g]
    check_same(sc, [v1, g], ref, R, masks=(0b11,))
    kt = _launches(v1)
    assert kt["dict"] == 1 and all(kt[c] == 0 for c in SHUFFLE_CLASSES if c != "dict"), kt   # the index, once
    check_same(sc, [v1, g], ref, R)
    assert _launches(v1)["dict"] == 1                              # later joins build nothing
    pa.free()                                                      # the parent first: the views own their copies
    check_same(sc, [v1, g], ref, R, masks=(0, 0b01))
    v2.free()
    check_same(sc, [g, v1], ref[::-1], R, masks=(0b10,))
    pc = str_parent(sc, kb_, values(rng, len(kb_), "i64"), 2, R, "max")
    parts_c = result_parts(pc, R)
    vc = view(pc)
    vc.free()                                                      # the view first: the parent still reads and views again
    assert result_parts(pc, R) == parts_c
    check_same(sc, [view(pc), v1], [rows_side(sc, parts_c, L.VB_I64, R), ref[0]], R, masks=(0b11, 0))


# ---- 6. ranks in one process --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [2, 3, 8])
def test_multirank(sc, W):
    from tests.test_gpu_str_combine_multirank import run_world
    from tests.test_gpu_str_multirank import run_ranks
    rng = np.random.default_rng(60 + W)
    R, M = 2 * W + 1, 2 * W
    keys = words(rng, 6000, POOL + [f"r{i}" for i in range(500)])
    vals = values(rng, len(keys), "u64")
    ckeys = words(rng, 5000, POOL + [f"r{i}" for i in range(300)])
    cols = [values(rng, len(ckeys), "i64"), values(rng, len(ckeys), "f64")]
    # MIN / MAX / COUNT and the u64 SUM do not depend on the order partials merge in, so the views of every rank equal
    # the one-process views bit for bit; an f64 MEAN does, and is checked against its own rank's parent instead
    multi = ([L.VB_I64, L.VB_F64], [(L.VB_AGG_MIN, 0), (L.VB_AGG_MAX, 1), (L.VB_AGG_COUNT, 0), (L.VB_AGG_MEAN, 1)])
    dts = [np.int64, np.float64, np.uint64, np.float64]
    red = run_ranks(sc, W, "sum", "u64", keys, vals, M, R)
    comb, _ = run_world(sc, W, multi, ckeys, cols, M, R)
    red1 = run_ranks(sc, 1, "sum", "u64", keys, vals, M, R)[0]
    comb1, _ = run_world(sc, 1, multi, ckeys, cols, M, R)
    one = [view(red1), view(comb1[0], 1, L.VB_F64), view(comb1[0], 2, L.VB_U64)]
    want_cg = cogroup_map(sc, one, R)
    want_j = {m: join_map(sc, one, R, m) for m in (0b111, 0b001, 0)}
    for d in range(W):
        vs = [view(red[d]), view(comb[d], 1, L.VB_F64), view(comb[d], 2, L.VB_U64)]
        check_view_reads(view(comb[d], 3, L.VB_F64), result_parts(comb[d], R, 3, dts))
        got = cogroup_map(sc, vs, R)
        got_j = {m: join_map(sc, vs, R, m) for m in want_j}
        for r in range(R):
            if r % W == d:
                assert got[r] == want_cg[r], (d, r)
                assert all(got_j[m][r] == want_j[m][r] for m in want_j), (d, r)
            else:
                assert not got[r] and all(not got_j[m][r] for m in want_j), f"rank {d} has keys of partition {r}"
                assert all(v.reduce_size(r) == (0, 0, 0) for v in vs)


# ---- 7. blocking ---------------------------------------------------------------------------------------------------------
def test_blocks_until_sealed(sc):
    R = 3
    sh = vb.StrShuffle(sc, 1, R, L.VB_U64, L.VB_AGG_SUM)
    ks = ["x", "z", "x", "y"]
    sh.map(0, vb.rdd._StrCol(ks), vb.rdd._Col(np.array([1, 2, 3, 4], dtype=np.uint64), role="value"), 0, len(ks))
    box = {}
    t = threading.Thread(target=lambda: box.setdefault("v", view(sh)))
    t.start()
    time.sleep(0.5)
    assert t.is_alive() and "v" not in box, "the view did not wait for the seal"
    sh.seal()
    t.join(60)
    assert not t.is_alive()
    parts = result_parts(sh, R)
    assert {k: v for d in parts for k, v in d.items()} == {b"x": 4, b"y": 4, b"z": 2}
    check_view_reads(box["v"], parts)


# ---- 8. refusals ----------------------------------------------------------------------------------------------------------
def test_rejected_calls_leave_the_parent_usable(sc):
    rng = np.random.default_rng(80)
    R = 3
    lib = sc._lib
    ks = words(rng, 2000, POOL)
    vals = values(rng, len(ks), "u64")
    ps = str_parent(sc, ks, vals, 2, R, "sum")
    before = result_parts(ps, R)
    comb = comb_parent(sc, ks, [vals], 2, R, {"s": ("sum", 0), "n": ("count", None)})._run()
    grp = sc.parallelize(ks, 2, values=vals).group_by_key(R)._run()
    srt = vb.StrSortedRdd(sc.parallelize(ks, 2, values=vals), R)._run()
    ints = sc.parallelize((np.arange(10, dtype=np.uint64), np.arange(10, dtype=np.uint64)), 2).reduce_by_key("sum", R)._run()
    vw = view(ps)
    out = ctypes.c_void_p()
    calls = [(None, 0, ctypes.byref(out)), (ps._h, 0, None), (ints._h, 0, ctypes.byref(out)), (grp._h, 0, ctypes.byref(out)),
             (srt._h, 0, ctypes.byref(out)), (vw._h, 0, ctypes.byref(out)), (ps._h, 1, ctypes.byref(out)),
             (comb._h, 2, ctypes.byref(out)), (comb._h, 1 << 31, ctypes.byref(out))]
    for h, col, o in calls:
        assert lib.vb_shuffle_create_narrow_str(h, col, o) == L.VB_ERR_INVALID, (h, col)
    # the neighbouring contracts are unchanged: the integer call refuses String parents, the String joins a raw reduce
    for sh in (ps, comb, vw):
        assert lib.vb_shuffle_create_narrow(sh._h, 0, ctypes.byref(out)) == L.VB_ERR_INVALID
    u = ctypes.c_uint64()
    assert lib.vb_cogroup_n_str_size(_arr([vw, ps]), 2, 0, ctypes.byref(u), None, None) == L.VB_ERR_INVALID
    assert lib.vb_join_n_str_size(_arr([ps, vw]), 2, 0, 0, ctypes.byref(u), None, None) == L.VB_ERR_INVALID
    assert result_parts(ps, R) == before
    check_view_reads(view(ps), before)
    check_same(sc, [view(ps), view(comb, 1, L.VB_U64), vw], [rows_side(sc, before, L.VB_U64, R),
               rows_side(sc, result_parts(comb, R, 1, [np.uint64, np.uint64]), L.VB_U64, R), rows_side(sc, before, L.VB_U64, R)],
               R, masks=(0b111, 0))


# ---- 9. scale: 5e7 rows over about 1e6 words per side, 2 % of the words shared ------------------------------------------
def test_scale(sc):
    import torch
    n, D, R = 50_000_000, 1_000_000, 16
    ranks, vals, shs = [], [], []
    for j, base in enumerate((0, int(D * 0.98))):
        r = torch.empty(n, dtype=torch.int64, device="cuda")
        sc.gen_pairs(out_keys=r, n=n, mode="uniform", n_distinct=D, seed_k=11 + j * 1_000_000_007)
        r = (r % D) + base
        v = torch.randint(0, 1 << 20, (n,), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        shs.append(sc.parallelize(_device_words(r), 8, values=v).reduce_by_key("sum", R)._run())
        ranks.append(r.cpu().numpy())
        vals.append(v.cpu().numpy())
        del r, v
    # the numpy reference on integer word ids: per id its sum (exact in f64, every sum < 2^53) and whether it occurs
    sums = [(np.bincount(r, weights=v.astype(np.float64), minlength=2 * D).astype(np.int64), np.bincount(r, minlength=2 * D) > 0)
            for r, v in zip(ranks, vals)]
    del ranks, vals
    views = [view(sh) for sh in shs]
    for v in views:
        assert all(_launches(v)[c] == 0 for c in SHUFFLE_CLASSES)
    shared = np.nonzero(sums[0][1] & sums[1][1])[0]
    pick = np.random.default_rng(0).choice(shared, 500, replace=False)
    total, joined, keys_cg = 0, [], 0
    for p in range(R):
        keys, ro, vs, _, _, nrows = join_part(sc, views, p, 0b11, dev=True, valid=False)
        total += nrows
        ids = np.array([int(k[1:], 16) for k in keys], dtype=np.int64)
        assert np.array_equal(np.diff(ro.astype(np.int64)), np.ones(len(keys), dtype=np.int64))
        for j in range(2):                                  # every joined key's two sums
            assert np.array_equal(vs[j].view(np.int64), sums[j][0][ids]), (p, j)
        joined.append(ids)
        keys_cg += len(cogroup_part(sc, views, p, dev=True)[0])
    joined = np.concatenate(joined)
    assert total == len(shared) and np.array_equal(np.sort(joined), shared)
    assert np.isin(pick, joined).all()
    assert keys_cg == int((sums[0][1] | sums[1][1]).sum())


# ---- 10. the mirrors ------------------------------------------------------------------------------------------------------
def _host_ref(rows_by_parent):
    """{key: [list per parent]} of parents given as {key: [values]}"""
    keys = set().union(*rows_by_parent)
    return {k: [list(p.get(k, [])) for p in rows_by_parent] for k in keys}


def test_mirror_same_splits_uses_views(sc):
    rng = np.random.default_rng(100)
    R = 5
    ka, kb_, kc = words(rng, 3000, POOL), words(rng, 2000, POOL[6:]), words(rng, 1500, POOL[:40])
    va = values(rng, len(ka), "u64")
    cb = [values(rng, len(kb_), "i64"), values(rng, len(kb_), "f64")]
    pa = sc.parallelize(ka, 3, values=va)
    red = pa.reduce_by_key("sum", R)
    comb = sc.parallelize(kb_, 2, values=tuple(cb)).combine_by_key({"lo": ("min", 0), "avg": ("mean", 1), "n": ("count", None)}, R)
    vcv = values(rng, len(kc), "u64")
    pc = sc.parallelize(kc, 2, values=vcv)
    cg = vb.StrCoGroupedRdd([red, comb.aggregate("avg"), comb.aggregate("n"), pc, pc.count_by_key(R)], R)
    shs, _ = cg._sides()
    for j in (0, 1, 2, 4):
        assert shs[j].n_map == 0 and shs[j].agg == L.VB_AGG_GROUP
        assert all(v == 0 for c, v in _launches(shs[j]).items() if c in SHUFFLE_CLASSES), j   # no encode, no seal kernels
    assert shs[1].vcode == L.VB_F64 and shs[2].vcode == L.VB_U64
    assert comb._sh is not None and red._sh is not None
    # the host reference: wrapping sums, counts and lists per key; the mean as the combine computed it
    sums, cnt_b, lists_c = {}, {}, {}
    for k, v in zip(ka, va.tolist()):
        sums[k] = (sums.get(k, 0) + v) % (1 << 64)
    for k in kb_:
        cnt_b[k] = cnt_b.get(k, 0) + 1
    for k, v in zip(kc, vcv.tolist()):
        lists_c.setdefault(k, []).append(v)
    keys, outs = comb.collect()
    avg_bits = dict(zip(keys.tolist(), outs["avg"].view(np.uint64).tolist()))
    assert dict(zip(keys.tolist(), outs["n"].tolist())) == cnt_b
    got = {k: ls for k, ls in cg.collect()}
    assert len(got) == len(set(ka) | set(kb_) | set(kc))
    for k, ls in got.items():
        assert ls[0].tolist() == ([sums[k]] if k in sums else []), k
        assert ls[1].view(np.uint64).tolist() == ([avg_bits[k]] if k in avg_bits else []), k
        assert ls[2].tolist() == ([cnt_b[k]] if k in cnt_b else []), k
        assert ls[3].tolist() == lists_c.get(k, []), k
        assert ls[4].tolist() == ([len(lists_c[k])] if k in lists_c else []), k
    k, vs = cg.join_collect()
    assert len(k) == sum(len(lists_c[x]) for x in set(ka) & set(kb_) & set(kc))
    assert sorted(zip(k.tolist(), vs[0].tolist(), vs[3].tolist())) == \
        sorted((x, sums[x], v) for x in set(ka) & set(kb_) & set(kc) for v in lists_c[x])


@pytest.mark.parametrize("R2", [3, 7])
def test_mirror_other_splits_reshuffle(sc, R2):
    rng = np.random.default_rng(110 + R2)
    R = 5
    ka, kb_ = words(rng, 3000, POOL), words(rng, 2000, POOL[6:])
    red = sc.parallelize(ka, 3, values=values(rng, len(ka), "i64")).reduce_by_key("max", R)
    comb = sc.parallelize(kb_, 2, values=(values(rng, len(kb_), "f64"),)).combine_by_key({"hi": ("max", 0), "avg": ("mean", 0)}, R)
    parents = [red, comb.aggregate("hi"), comb.aggregate("avg")]
    same = vb.StrCoGroupedRdd(parents, R)
    other = vb.StrCoGroupedRdd(parents, R2)
    shs, _ = other._sides()
    assert all(s.n_map == R for s in shs)                          # reshuffled: one map task per result partition
    assert {k: [l.view(np.uint64).tolist() for l in ls] for k, ls in same.collect()} == \
        {k: [l.view(np.uint64).tolist() for l in ls] for k, ls in other.collect()}
    a, b = same.outer_join_collect([0]), other.outer_join_collect([0])
    ra = sorted(zip(a[0].tolist(), *[np.ma.getdata(v).view(np.uint64).tolist() for v in a[1]]))
    rb = sorted(zip(b[0].tolist(), *[np.ma.getdata(v).view(np.uint64).tolist() for v in b[1]]))
    assert ra == rb and len(ra) == len(set(ka))


def test_cpp_narrow_join_string_example_runs():
    """examples/narrow_join_string.cpp: String reduce_by_key results joined, cogrouped and left-outer-joined without a
    second shuffle; exit 0 only on the expected rows."""
    path = os.path.join(ROOT, "examples", "_build", "narrow_join_string")
    if not os.path.exists(path):
        pytest.skip("examples not built (run __graft_entry__.build())")
    out = subprocess.run([path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert 'join: [("", (50, 5)), ("x", (21, 201))]' in out.stdout, out.stdout
    assert '("y", [20, None, 15])' in out.stdout and "cogroup: 4 keys" in out.stdout, out.stdout
