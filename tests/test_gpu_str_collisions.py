"""String and Vec<u8> keys crafted to share their full 64-bit MetroHash64_1 (tests/metro_collide_ref.py), mixed into
ordinary rows, through every String-key path: reduce and counting ops, combine_by_key, index growth, group_by_key,
sort, cogroup and the joins, narrow views, the import across ranks, blobs and the hash calls.

Distinct keys of one hash share their home bucket at every index size, so the dictionary can only tell them apart by
their bytes, and a chain of n such keys spans n / 4 buckets.  Every result is checked against a plain Python or
numpy reference keyed by the key bytes, and every key against its partition hash % R.  The solved bytes are not
UTF-8: String keys come back as surrogate-escaped strs and are compared as bytes."""
import ctypes
import math

import numpy as np
import pytest
import torch

import vega_b200 as vb
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from tests import metro_collide_ref as MC
from tests import multirank as MR
from tests import str_blob_ref as SB
from tests import str_group_ref as S
from tests.test_gpu_combine import check_f64_means
from tests.test_gpu_str_keys import _bits
from tests.util import f64_total_key, rand_pairs

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1
KIND = {MC.STR: L.VB_STRKEY_STR, MC.BYTES: L.VB_STRKEY_BYTES}
KINDS = (MC.STR, MC.BYTES)
SIZES = (2, 3, 255, 256, 257, 1024, 3000)
AGG = {"sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT, "group": L.VB_AGG_GROUP}
VCODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}
N_ROWS, N_KEYS = 200_000, 20_000


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


# ---- inputs ---------------------------------------------------------------------------------------------------------
_ORD = {}


def ordinary(seed):
    """str_group_ref.rank_rows: about 200k rows over 20k keys, as bytes."""
    if seed not in _ORD:
        o, d = S.encode(S.rank_rows(np.random.default_rng(seed), N_ROWS, N_KEYS))
        raw, oo = d.tobytes(), o.astype(np.int64).tolist()
        _ORD[seed] = [raw[oo[i]:oo[i + 1]] for i in range(len(oo) - 1)]
    return _ORD[seed]


def mixed(crafted, seed, hot=2000, base=None):
    """Ordinary rows plus 1 to 20 rows of every crafted key (the first one hot), shuffled."""
    rng = np.random.default_rng(seed)
    rows = list(ordinary(seed % 3) if base is None else base)
    for i, k in enumerate(crafted):
        rows += [k] * (int(rng.integers(1, 21)) + (hot if i == 0 else 0))
    return [rows[i] for i in rng.permutation(len(rows))]


def values(n, vdt, seed):
    rng = np.random.default_rng(seed)
    if vdt == "f64":
        return rand_pairs(rng, n, 50, "f64", values="special")[1]
    return rand_pairs(rng, n, 50, vdt, values="full")[1]


def key_col(kind, keys, where="host"):
    """The keys as a map column: vb.BytesKeys, or vb.StrKeys over the raw bytes; host, device (copied in the call)
    or borrowed."""
    b = vb.BytesKeys.from_bytes(keys)
    cls = vb.BytesKeys if kind == MC.BYTES else vb.StrKeys
    if where == "host":
        return cls(b.offsets, b.data)
    return cls(torch.from_numpy(b.offsets.view(np.int64)).cuda(), torch.from_numpy(b.data.copy()).cuda())


def raw(k):
    """A key as it comes back, as bytes."""
    return k if isinstance(k, bytes) else k.encode("utf-8", "surrogateescape")


class Placement:
    """hash % R of every distinct key, from the numpy restatements."""

    def __init__(self, kind, keys):
        u = list(dict.fromkeys(keys))
        self.h = dict(zip(u, MC.hashes(kind, u).tolist()))

    def check(self, keys, r, R, fam=None):
        ks = [raw(k) for k in keys]
        assert len(set(ks)) == len(ks), f"a key twice in partition {r}"
        bad = [k for k in ks if self.h[k] % R != r]
        assert not bad, f"partition {r} of {R}: {len(bad)} keys placed elsewhere, first {bad[0][:16]!r}"
        if fam is not None:
            assert all(fam.hash % R == r for k in ks if k in fam.set)
        return ks


def family(kind, n, seed=0):
    f = MC.same_hash(kind, n, seed=1000 * n + seed)
    f.set = set(f.keys)
    return f


def ids_of(keys):
    """Dense ids of the keys in first-seen order, and the id of every row."""
    d = {}
    return d, np.array([d.setdefault(k, len(d)) for k in keys], np.int64)


def ref_reduce(keys, vals, op, vdt):
    """{key bytes: result} of reduce_by_key(op): exact integer sums mod 2^64, MIN/MAX of i64 signed and of f64 by its
    total order with NaN as the identity (an all-NaN key gives NaN)."""
    d, ids = ids_of(keys)
    order = np.argsort(ids, kind="stable")
    starts = np.flatnonzero(np.r_[True, np.diff(ids[order]) != 0])
    ukeys = list(d)
    if op == "count":
        return dict(zip(ukeys, np.diff(np.r_[starts, len(ids)]).tolist()))
    v = np.asarray(vals)[order]
    if vdt == "f64":
        t = f64_total_key(v)
        nan = np.isnan(v)
        ident = np.uint64(M64) if op == "min" else np.uint64(0)
        t = np.where(nan, ident, t)
        r = (np.minimum if op == "min" else np.maximum).reduceat(t, starts)
        back = np.where(r >> np.uint64(63), r & np.uint64((1 << 63) - 1), ~r).view(np.float64)
        return dict(zip(ukeys, back.tolist()))
    with np.errstate(over="ignore"):
        r = {"sum": np.add, "min": np.minimum, "max": np.maximum}[op].reduceat(v, starts)
    return dict(zip(ukeys, r.tolist()))


def norm(x, vdt):
    return _bits(x, vdt) if vdt == "f64" else int(x) & M64


def run_single(sc, kind, kc, vc, op, vdt, n, M, R, hint=0):
    starts = vb.slice_starts(n, M)
    sh = vb.StrShuffle(sc, len(starts) - 1, R, VCODE[vdt], AGG[op], hint=hint, key_kind=KIND[kind])
    kcol = vb.rdd._StrCol(kc)
    vcol = None if op == "count" else vb.rdd._Col(vc, role="value")
    for m in range(len(starts) - 1):
        sh.map(m, kcol, vcol, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    return sh


def collect_reduce(sh, R, place, vdt, fam=None):
    got = {}
    for r in range(R):
        ks, comb = sh.reduce(r)[:2]
        got.update(zip(place.check(ks.tolist(), r, R, fam), [norm(x, vdt) for x in comb.tolist()]))
    return got


# ---- reduce and the counting ops ------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", SIZES)
def test_reduce_and_counting_ops(sc, kind, size):
    fam = family(kind, size)
    keys = mixed(fam.keys, seed=size)
    place = Placement(kind, keys)
    n, M, R = len(keys), 4, 7
    kc = key_col(kind, keys)
    for op, vdt in (("sum", "u64"), ("sum", "i64"), ("min", "i64"), ("max", "i64"), ("min", "f64"), ("max", "f64"),
                    ("count", "u64")):
        v = values(n, vdt, seed=size + len(op))
        sh = run_single(sc, kind, kc, v, op, vdt, n, M, R)
        want = {k: norm(x, vdt) for k, x in ref_reduce(keys, v, op, vdt).items()}
        got = collect_reduce(sh, R, place, vdt, fam)
        assert got == want, (op, vdt)
        assert all(k in got for k in fam.keys)
        sh.free()
    rdd = sc.parallelize(kc, M)
    cbv = rdd.count_by_value()
    got = collect_reduce(cbv._run(), cbv.num_slices, Placement(kind, keys), "u64")
    assert got == ref_reduce(keys, None, "count", "u64")
    d = rdd.distinct(R)
    dsh = d.sh._run()
    seen = []
    for r in range(R):
        seen += place.check(dsh.reduce(r)[0].tolist(), r, R, fam)
    assert sorted(seen) == sorted(set(keys))


# ---- combine_by_key -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", [257, 3000])
def test_combine_by_key_two_columns(sc, kind, size):
    fam = family(kind, size, seed=1)
    keys = mixed(fam.keys, seed=size + 1)
    place = Placement(kind, keys)
    n, R = len(keys), 5
    i = values(n, "i64", seed=3)
    f = values(n, "f64", seed=4)
    c = sc.parallelize(key_col(kind, keys), 4, values=(i, f)).combine_by_key(
        {"s": ("sum", 0), "lo": ("min", 0), "hi": ("max", 1), "n": ("count", None), "avg": ("mean", 1)}, R)
    want_s, want_lo = ref_reduce(keys, i, "sum", "i64"), ref_reduce(keys, i, "min", "i64")
    want_hi, want_n = ref_reduce(keys, f, "max", "f64"), ref_reduce(keys, None, "count", "u64")
    d, ids = ids_of(keys)
    means = []
    for r in range(R):
        ks, outs = c.compute(r)
        ks = place.check(ks.tolist(), r, R, fam)
        for j, k in enumerate(ks):
            assert int(outs["s"][j]) & M64 == want_s[k] & M64 and int(outs["lo"][j]) == want_lo[k], k[:16]
            assert _bits(float(outs["hi"][j]), "f64") == _bits(want_hi[k], "f64") and int(outs["n"][j]) == want_n[k]
        means.append({d[k]: float(outs["avg"][j]) for j, k in enumerate(ks)})
        assert all(k in d for k in ks)
    assert sum(len(m) for m in means) == len(d)
    check_f64_means(means, ids.astype(np.uint64), f)


# ---- index growth ---------------------------------------------------------------------------------------------------
def control_keys(kind, n, seed):
    """n random distinct keys of the family's length, none equal to a crafted one (almost surely distinct hashes)."""
    rng = np.random.default_rng(seed)
    L_ = MC.DEFAULT_LEN[kind]
    return [bytes(r) for r in np.unique(rng.integers(0, 256, (n + 8, L_), dtype=np.uint8), axis=0)[:n]]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", [257, 3000])
@pytest.mark.parametrize("hint,M,where", [(0, 1, "host"), (1, 1, "host"), (1, 4, "device"), (0, 4, "borrowed"),
                                          (1, 3, "borrowed"), (0, 2, "device")])
def test_index_growth_is_bounded(sc, kind, size, hint, M, where):
    fam = family(kind, size, seed=2)
    absent_keys = MC.absent(fam, 64)
    rng = np.random.default_rng(size + M)
    base = ordinary(1)
    keys = mixed(fam.keys, seed=7 * size + M, base=base)
    ctrl = mixed(control_keys(kind, size, seed=size), seed=7 * size + M, base=base)
    n = len(keys)
    assert len(ctrl) == n
    v = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    R = 3
    stats = []
    for ks in (ctrl, keys):
        place = Placement(kind, ks)
        vc = v if where == "host" else torch.from_numpy(v.view(np.int64)).cuda()
        kc = key_col(kind, ks, where)
        kcol, vcol = vb.rdd._StrCol(kc), vb.rdd._Col(vc, role="value")
        if where == "device":
            kcol.loc = vcol.loc = L.VB_DEVICE
        starts = vb.slice_starts(n, M)
        sh = vb.StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, hint=hint, key_kind=KIND[kind])
        for m in range(M):
            sh.map(m, kcol, vcol, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        got = collect_reduce(sh, R, place, "u64")
        assert got == {k: x & M64 for k, x in ref_reduce(ks, v, "sum", "u64").items()}
        assert not set(absent_keys) & set(got)
        stats.append(sh.stats())
        sh.free()
    c, x = stats
    assert x["table_slots"] <= 4 * c["table_slots"], (x["table_slots"], c["table_slots"])
    assert x["table_restarts"] <= c["table_restarts"] + 1, (x["table_restarts"], c["table_restarts"])


# ---- group_by_key and sort ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", [257, 3000])
@pytest.mark.parametrize("sort_values", [False, True])
def test_group_by_key(sc, kind, size, sort_values):
    fam = family(kind, size, seed=3)
    keys = mixed(fam.keys, seed=size + 3, hot=500)
    place = Placement(kind, keys)
    v = np.random.default_rng(size).integers(0, 1 << 64, len(keys), dtype=np.uint64)
    R = 6
    sh = sc.parallelize(key_col(kind, keys), 3, values=v).group_by_key(R, sort_values=sort_values)._run()
    want = {}
    for k, x in zip(keys, v.tolist()):
        want.setdefault(k, []).append(x)
    if sort_values:
        want = {k: sorted(x) for k, x in want.items()}
    got = {}
    for r in range(R):
        ks, offs, vals = sh.reduce(r)
        o = offs.astype(np.int64)
        got.update({k: vals[o[i]:o[i + 1]].tolist() for i, k in enumerate(place.check(ks.tolist(), r, R, fam))})
    assert got == want


@pytest.mark.parametrize("kind", KINDS)
def test_sort_orders_colliding_keys_by_bytes_and_stays_stable(sc, kind):
    fam = family(kind, 1024, seed=4)
    lengths = MC.same_hash_lengths(300, seed=4).keys if kind == MC.BYTES else []
    keys = mixed(fam.keys + lengths, seed=44, hot=300)
    v = np.arange(len(keys), dtype=np.uint64)                     # the row number: stability is visible
    order = sorted(range(len(keys)), key=lambda i: keys[i])
    R = 5
    ks, vs = vb.StrSortedRdd(sc.parallelize(key_col(kind, keys), 3, values=v), R).collect()
    assert [raw(k) for k in ks.tolist()] == [keys[i] for i in order]
    assert vs.tolist() == order
    got = vb.StrSortedRdd(sc.parallelize(key_col(kind, keys), 4), R).collect()       # keys only
    assert [raw(k) for k in got.tolist()] == sorted(keys)


# ---- cogroup and the joins ------------------------------------------------------------------------------------------
def side(sc, kind, keys, seed, M=3):
    v = np.random.default_rng(seed).integers(0, 1 << 40, len(keys), dtype=np.uint64)
    want = {}
    for k, x in zip(keys, v.tolist()):
        want.setdefault(k, []).append(x)
    return sc.parallelize(key_col(kind, keys), M, values=v), want


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n_sides", [2, 3])
def test_cogroup_and_joins_match_only_equal_bytes(sc, kind, n_sides):
    fam = family(kind, 1024, seed=5)
    ab = MC.absent(fam, 200)
    F = fam.keys
    base = ordinary(2)
    subsets = [F[:600], F[400:], F[::3] + ab][:n_sides]
    rng = np.random.default_rng(n_sides)
    sides = [side(sc, kind, mixed(s, seed=50 + j, hot=20, base=base[j::3]), seed=j) for j, s in enumerate(subsets)]
    rdds, wants = [s[0] for s in sides], [s[1] for s in sides]
    place = Placement(kind, [k for w in wants for k in w])
    R = 7
    cg = vb.StrCoGroupedRdd(rdds, R)
    seen = set()
    for r in range(R):
        ks, lists = cg.compute(r)
        for i, k in enumerate(place.check(ks.tolist(), r, R, fam)):
            seen.add(k)
            for (o, v), w in zip(lists, wants):
                assert v[int(o[i]):int(o[i + 1])].tolist() == w.get(k, [])
    assert seen == set().union(*wants)
    inner = set(wants[0]).intersection(*wants[1:])
    assert not inner & set(ab) and (n_sides == 2 or not set(ab) & set(wants[0]))
    for r in range(R):
        k, cols = cg.join_compute(r)
        ks = [raw(q) for q in k.tolist()]
        assert set(ks) <= inner and all(place.h[q] % R == r for q in ks)
        assert len(ks) == sum(math.prod(len(w[q]) for w in wants) for q in inner if place.h[q] % R == r)
        rows = sorted(zip(ks, *[c.tolist() for c in cols]))
        want_rows = []
        for q in {q for q in inner if place.h[q] % R == r}:
            for combo in np.array(np.meshgrid(*[wants[j][q] for j in range(n_sides)], indexing="ij")).reshape(n_sides, -1).T:
                want_rows.append((q, *[int(x) for x in combo]))
        assert rows == sorted(want_rows)
        for required, need in ((1, [0]), (0, [])):                  # left outer, full outer
            k, cols = cg.outer_join_compute(r, required)
            ks = [raw(q) for q in k.tolist()]
            keep = {q for q in set().union(*wants) if place.h[q] % R == r and all(q in wants[j] for j in need)}
            assert set(ks) == keep
            assert len(ks) == sum(math.prod(max(len(w.get(q, [])), 1) for w in wants) for q in keep)


@pytest.mark.parametrize("kind", KINDS)
def test_narrow_views_joined_with_a_group_side(sc, kind):
    fam = family(kind, 1024, seed=6)
    ab = MC.absent(fam, 100)
    base = ordinary(0)
    a, wa = side(sc, kind, mixed(fam.keys[:700], seed=61, base=base[::2]), seed=1)
    b, wb = side(sc, kind, mixed(fam.keys[300:] + ab, seed=62, base=base[1::2]), seed=2)
    R = 5
    red = a.reduce_by_key("sum", R)
    sums = {q: sum(x) & M64 for q, x in wa.items()}
    place = Placement(kind, list(wa) + list(wb))
    nj = vb.StrCoGroupedRdd([red, b], R)
    n = 0
    for r in range(R):
        k, (x, y) = nj.join_compute(r)
        ks = [raw(q) for q in k.tolist()]
        assert all(place.h[q] % R == r for q in ks)
        for q, s_, v_ in zip(ks, x.tolist(), y.tolist()):
            assert s_ == sums[q] and v_ in wb[q]
        n += len(ks)
    assert n == sum(len(wb[q]) for q in wa if q in wb)


# ---- across ranks ---------------------------------------------------------------------------------------------------
def swap(exports):
    recv = MR.swap_columns([(cols, (nk, nb, nk, nv)) for (nk, nb, nv), cols in exports])
    return [(tuple(cols), (n[0], n[1], n[3])) for cols, n in recv]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("W", [2, 3])
def test_multirank_reduce_group_and_combine(sc, kind, W):
    fam = family(kind, 3000, seed=7)
    keys = mixed(fam.keys, seed=70 + W)
    place = Placement(kind, keys)
    n, M, R = len(keys), 6, 7
    v = np.random.default_rng(W).integers(0, 1 << 64, n, dtype=np.uint64)
    kcol, vcol = vb.rdd._StrCol(key_col(kind, keys)), vb.rdd._Col(v, role="value")
    starts = vb.slice_starts(n, M)
    for op in ("sum", "group"):
        shs = [vb.StrShuffle(sc, M, R, L.VB_U64, AGG[op], rank=r, world=W, key_kind=KIND[kind]) for r in range(W)]
        for r, sh in enumerate(shs):
            lo, hi = vdist.map_block(r, W, M)
            for m in range(lo, hi):
                sh.map(m, kcol, vcol, int(starts[m]), int(starts[m + 1]))
        for sh, (cols, counts) in zip(shs, swap([sh.export() for sh in shs])):
            sh.import_(*cols, *counts)
        got = {}
        for d, sh in enumerate(shs):
            sh.seal()
            for r in range(R):
                p = sh.reduce(r)
                if r % W != d:
                    assert len(p[0]) == 0
                    continue
                ks = place.check(p[0].tolist(), r, R, fam)
                if op == "group":
                    o = p[1].astype(np.int64)
                    got.update({q: p[2][o[i]:o[i + 1]].tolist() for i, q in enumerate(ks)})
                else:
                    got.update(zip(ks, p[1].tolist()))
            sh.free()
        if op == "group":
            want = {}
            for k, x in zip(keys, v.tolist()):
                want.setdefault(k, []).append(x)
            assert got == want
        else:
            assert got == {k: x & M64 for k, x in ref_reduce(keys, v, "sum", "u64").items()}
    multi = ([L.VB_U64], [(L.VB_AGG_COUNT, 0), (L.VB_AGG_SUM, 0), (L.VB_AGG_MAX, 0)])
    shs = [vb.StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, rank=r, world=W, multi=multi, key_kind=KIND[kind]) for r in range(W)]
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        for m in range(lo, hi):
            sh.map_cols(m, kcol, (vcol,), int(starts[m]), int(starts[m + 1]))
    exports = [sh.export_cols() for sh in shs]
    recv = MR.swap_columns([([lens, data, accs.t()], [nk, nb, nk]) for (nk, nb), (lens, data, accs) in exports])
    for sh, (rc, rs) in zip(shs, recv):
        sh.import_cols(rc[0], rc[1], rc[2].t().contiguous(), rs[0], rs[1])
    cnt, s, mx = (ref_reduce(keys, v, op, "u64") for op in ("count", "sum", "max"))
    n_keys = 0
    for d, sh in enumerate(shs):
        sh.seal()
        for r in range(R):
            ko, kb, (c0, c1, c2) = sh.reduce_cols(r, [np.uint64] * 3)
            ks = vb.rdd._decode_keys(ko, kb, KIND[kind]).tolist()
            if r % W != d:
                assert not ks
                continue
            ks = place.check(ks, r, R, fam)
            n_keys += len(ks)
            assert all(int(a) == cnt[q] and int(b) == s[q] & M64 and int(c) == mx[q] for q, a, b, c in zip(ks, c0, c1, c2))
        sh.free()
    assert n_keys == len(cnt)


# ---- blobs and the hash calls ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_reduce_blobs_round_trip(sc, kind):
    fam = family(kind, 1024, seed=8)
    keys = mixed(fam.keys, seed=80)
    place = Placement(kind, keys)
    n, M, R = len(keys), 4, 6
    v = np.random.default_rng(8).integers(0, 1 << 64, n, dtype=np.uint64)
    sh = run_single(sc, kind, key_col(kind, keys), v, "sum", "u64", n, M, R)
    want = {k: x & M64 for k, x in ref_reduce(keys, v, "sum", "u64").items()}
    blobs = []
    for r in range(R):
        ks = place.check(sh.reduce(r)[0].tolist(), r, R, fam)
        blob = sh.reduce_blob(r)
        assert blob == SB.encode_str_pairs([(k, want[k]) for k in ks])
        blobs.append(blob)
    sh.free()
    out = vb.StrShuffle(sc, R, 3, L.VB_U64, L.VB_AGG_SUM, key_kind=KIND[kind])
    for m, blob in enumerate(blobs):
        out.map_blob(m, blob)
    out.seal()
    assert collect_reduce(out, 3, place, "u64", fam) == want
    out.free()


def test_hash_calls_return_the_family_hash(sc):
    lib = vb.lib()
    for kind, fn in ((MC.STR, lib.vb_hash_str), (MC.BYTES, lib.vb_hash_bytes)):
        for fam in (family(kind, 3000, seed=9), MC.wrap(kind, 300)):
            assert {fn(ctypes.c_char_p(k), len(k)) for k in fam.keys} == {fam.hash}
        p = MC.pairs(kind, 500)
        assert [fn(ctypes.c_char_p(k), len(k)) for k in p] == MC.hashes(kind, p).tolist()
    lk = MC.same_hash_lengths(200)
    assert {lib.vb_hash_bytes(ctypes.c_char_p(k), len(k)) for k in lk.keys} == {lk.hash}


@pytest.mark.parametrize("kind", KINDS)
def test_wrap_and_pairs_families(sc, kind):
    """Keys homed at the last bucket (the chain wraps to bucket 0), 2-key collisions all over the index, and absent
    keys: reduce with a tiny initial index, and group."""
    w = MC.wrap(kind, 1500, seed=1)
    p = MC.pairs(kind, 4000, seed=2)
    extra = MC.same_hash_lengths(300, seed=3).keys if kind == MC.BYTES else []
    crafted = w.keys + p + extra
    keys = mixed(crafted, seed=90, hot=100)
    place = Placement(kind, keys)
    n, R = len(keys), 9
    v = np.random.default_rng(9).integers(0, 1 << 64, n, dtype=np.uint64)
    for hint in (1, 0):
        sh = run_single(sc, kind, key_col(kind, keys), v, "sum", "u64", n, 3, R, hint=hint)
        got = collect_reduce(sh, R, place, "u64")
        assert got == {k: x & M64 for k, x in ref_reduce(keys, v, "sum", "u64").items()}
        assert not set(MC.absent(w, 50)) & set(got)
        sh.free()
    gsh = sc.parallelize(key_col(kind, keys), 5, values=v).group_by_key(R)._run()
    want = {}
    for k, x in zip(keys, v.tolist()):
        want.setdefault(k, []).append(x)
    got = {}
    for r in range(R):
        ks, offs, vals = gsh.reduce(r)
        o = offs.astype(np.int64)
        got.update({k: vals[o[i]:o[i + 1]].tolist() for i, k in enumerate(place.check(ks.tolist(), r, R))})
    assert got == want
