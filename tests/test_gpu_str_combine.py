"""combine_by_key over String keys (vb_shuffle_create_str_multi), one process, against the single-column references.

Every output column is checked on its own against the vb_shuffle_create_str shuffle of that op and column: integer
SUM / MIN / MAX, COUNT and f64 MIN / MAX bit for bit, f64 SUM within the bound of any summation order, MEAN as
(double)S / n from the SUM and COUNT shuffles (f64 MEAN within the f64 SUM bound over n).  Every key must sit in the
partition vb_get_partition_str gives it, and the whole result must equal the integer combine over the same rows keyed
by each word's rank, and oracle/pyref.py at small sizes."""
import ctypes
import math
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref
from tests.test_gpu_combine import SPECS
from tests.test_gpu_str_keys import _device_keys, _device_words, _fold, _host_keys, key_pool, rows_from_pool
from tests.util import rand_pairs
from vega_b200 import _lib as L
from vega_b200.rdd import Shuffle, StrShuffle, _Col, _StrCol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
AGG = {"sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT, "mean": L.VB_AGG_MEAN}
NP = {"u64": np.uint64, "i64": np.int64, "f64": np.float64}
CODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


def special_keys():
    """The empty key, NUL bytes, multibyte UTF-8, 700-byte keys and keys that share their first 8 bytes."""
    return (["", "\x00", "a\x00b", "é", "日本語", "🙂🙂"] + ["L" * 700 + str(i) for i in range(4)]
            + ["prefix08" + s for s in ("", "a", "b", "ab", "\x00")])


def make_rows(seed, spec, n, n_pool=400):
    rng = np.random.default_rng(seed)
    pool = sorted(set(key_pool(rng, n_random=n_pool) + special_keys()))
    keys = rows_from_pool(rng, pool, n)
    cols = [rand_pairs(rng, n, 100, d, values=m)[1] for d, m in SPECS[spec][0]]
    return keys, cols


def out_dtypes(spec):
    dts, aggs = SPECS[spec]
    return [np.uint64 if op == "count" else np.float64 if op == "mean" else NP[dts[c][0]] for op, c in aggs]


def multi_of(spec):
    dts, aggs = SPECS[spec]
    return [CODE[d] for d, _ in dts], [(AGG[op], c) for op, c in aggs]


def str_combine(sc, spec, kcol, vcols, n, M, R, hint=0):
    """The String combine: M map tasks over rows [0, n), seal -> ([{key: (output per aggregate)}] per partition, stats)."""
    starts = vb.slice_starts(n, M)
    sh = StrShuffle(sc, len(starts) - 1, R, L.VB_U64, L.VB_AGG_SUM, hint=hint, multi=multi_of(spec))
    try:
        for m in range(len(starts) - 1):
            sh.map_cols(m, kcol, vcols, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        parts = [decode(sh.reduce_cols(r, out_dtypes(spec))) for r in range(R)]
        st = sh.stats()
    finally:
        sh.free()
    return parts, st


def decode(raw):
    ko, kb, outs = raw
    keys = vb.rdd._decode_keys(ko, kb).tolist()
    assert len(set(keys)) == len(keys), "a key twice in one partition"
    return dict(zip(keys, zip(*[o.tolist() for o in outs]))) if keys else {}


def single(sc, kcol, vcol, op, vcode, n, M, R):
    """The single-column String shuffle of op over one column: [{key: value}] per partition."""
    starts = vb.slice_starts(n, M)
    sh = StrShuffle(sc, len(starts) - 1, R, vcode, AGG[op])
    try:
        for m in range(len(starts) - 1):
            sh.map(m, kcol, None if op == "count" else vcol, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        out = []
        for r in range(R):
            k, c = sh.reduce(r)[:2]
            out.append(dict(zip(k.tolist(), c.tolist())))
    finally:
        sh.free()
    return out


def bits(x):
    if isinstance(x, float):
        return "nan" if math.isnan(x) else np.float64(x).view(np.uint64).item()
    return int(x)


def sum_bound_ok(got, xs):
    """f64 SUM of xs in any order: NaN / inf rules, else |got - fsum| within the order-independent bound."""
    if any(math.isnan(v) for v in xs) or (math.inf in xs and -math.inf in xs):
        return math.isnan(got)
    if math.inf in xs or -math.inf in xs:
        return got == (math.inf if math.inf in xs else -math.inf)
    m, u = len(xs), 2.0 ** -53
    bound = (m - 1) * u / (1 - (m - 1) * u) * sum(abs(v) for v in xs) * (1 + 2 * m * u)
    s = math.fsum(xs)
    return abs(got - s) <= bound + math.ulp(s)


def mean_bound_ok(got, xs):
    """f64 MEAN of finite xs: |got - fsum / m| within the f64 SUM bound over m (non-finite inputs are not checked)."""
    if not all(math.isfinite(x) for x in xs):
        return True
    m, u = len(xs), 2.0 ** -53
    s = math.fsum(xs)
    bound = ((m - 1) * u / (1 - (m - 1) * u) * sum(abs(x) for x in xs) * (1 + 2 * m * u) + math.ulp(s)) / m + math.ulp(got)
    return abs(got - s / m) <= bound


def check_against_singles(sc, spec, parts, keys, cols, kcol, vcols, n, M, R):
    dts, aggs = SPECS[spec]
    R_ = len(parts)
    for r, p in enumerate(parts):
        for k in p:
            b = k.encode("utf-8", "surrogateescape")
            assert L.lib().vb_get_partition_str(ctypes.c_char_p(b), len(b), R_) == r, (k[:20], r)
    cache = {}

    def ref(op, c):
        if (op, c) not in cache:
            cache[(op, c)] = single(sc, kcol, vcols[c], op, CODE[dts[c][0]], n, M, R)
        return cache[(op, c)]

    per_key = {}
    for c, (d, _) in enumerate(dts):
        if d == "f64":
            for k, v in zip(keys, cols[c].tolist()):
                per_key.setdefault((c, k), []).append(v)
    count = ref("count", 0)
    assert [set(p) for p in parts] == [set(p) for p in count], "the key sets differ from the COUNT shuffle's"
    for a, (op, c) in enumerate(aggs):
        d = dts[c][0]
        for r, p in enumerate(parts):
            if op == "sum" and d == "f64":
                bad = [k for k, v in p.items() if not sum_bound_ok(v[a], per_key[(c, k)])]
            elif op == "mean" and d == "f64":
                bad = [k for k, v in p.items() if not mean_bound_ok(v[a], per_key[(c, k)])]
            elif op == "mean":
                sums = ref("sum", c)[r]
                bad = [k for k, v in p.items()
                       if bits(v[a]) != bits(float(np.float64(sums[k]) / np.float64(count[r][k])))]
            else:
                w = ref(op, c)[r]
                bad = [k for k, v in p.items() if bits(v[a]) != bits(w[k])]
            assert not bad, f"aggregate {a} ({op} of column {c}, {d}), partition {r}: {len(bad)} keys, e.g. {bad[:3]}"


def check_against_int_combine(sc, spec, parts, keys, cols, M):
    """The integer combine over the same rows keyed by each word's rank: every column but f64 SUM / MEAN bit for bit."""
    dts, aggs = SPECS[spec]
    words = sorted(set(keys))
    rank = {w: i for i, w in enumerate(words)}
    ik = np.array([rank[k] for k in keys], dtype=np.uint64)
    starts = vb.slice_starts(len(keys), M)
    sh = Shuffle(sc, len(starts) - 1, 5, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, multi=multi_of(spec))
    try:
        vc = tuple(_Col(c, role="value") for c in cols)
        for m in range(len(starts) - 1):
            sh.map_cols(m, _Col(ik), vc, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        want = {}
        for r in range(5):
            k, outs = sh.reduce_cols(r, out_dtypes(spec))
            want.update({words[int(x)]: v for x, v in zip(k.tolist(), zip(*[o.tolist() for o in outs]))})
    finally:
        sh.free()
    got = {}
    for p in parts:
        got.update(p)
    assert got.keys() == want.keys()
    exact = [a for a, (op, c) in enumerate(aggs) if not (dts[c][0] == "f64" and op in ("sum", "mean"))]
    bad = [k for k in got if [bits(got[k][a]) for a in exact] != [bits(want[k][a]) for a in exact]]
    assert not bad, f"{len(bad)} keys differ from the integer combine, e.g. {bad[:3]}"


@pytest.mark.parametrize("spec", sorted(SPECS))
@pytest.mark.parametrize("M,R", [(1, 1), (7, 8), (64, 300)])
def test_specs_match_single_column_shuffles(sc, spec, M, R):
    n = 40_000
    keys, cols = make_rows(sorted(SPECS).index(spec) * 10 + M, spec, n)
    kcol = _StrCol(keys)
    vcols = tuple(_Col(c, role="value") for c in cols)
    parts, st = str_combine(sc, spec, kcol, vcols, n, M, R)
    assert st["rows_in"] == n and st["rows_out"] == len(set(keys))
    check_against_singles(sc, spec, parts, keys, cols, kcol, vcols, n, M, R)
    check_against_int_combine(sc, spec, parts, keys, cols, M)


def test_small_against_pyref(sc):
    """Python strs through Context.parallelize and StrCombinedRdd, against pyref's reduce_by_key of each op."""
    rng = np.random.default_rng(3)
    pool = special_keys() + ["x", "y", "z"]
    keys = rows_from_pool(rng, pool, 500)
    u = rng.integers(0, 1 << 64, 500, dtype=np.uint64)
    i = rng.integers(-(1 << 63), (1 << 63) - 1, 500, dtype=np.int64)
    M, R = 3, 4
    c = sc.parallelize(keys, M, values=(u, i)).combine_by_key(
        {"n": ("count", None), "s": ("sum", 0), "lo": ("min", 1), "hi": ("max", 0), "avg": ("mean", 1), "s1": ("sum", 1)}, R)
    got_keys, got = c.collect()
    assert len(got_keys) == len(set(keys))

    def want(op, vals, vdt):
        return dict(pyref.reduce_by_key(list(zip(keys, vals)), _fold(op, vdt), M, R))
    n = want("sum", [1] * len(keys), "u64")
    ref = {"n": n, "s": want("sum", u.tolist(), "u64"), "lo": want("min", i.tolist(), "i64"),
           "hi": want("max", u.tolist(), "u64"), "s1": want("sum", i.tolist(), "i64")}
    for name, w in ref.items():
        assert dict(zip(got_keys.tolist(), got[name].tolist())) == w, name
    assert dict(zip(got_keys.tolist(), got["avg"].tolist())) == {k: float(np.float64(ref["s1"][k]) / np.float64(n[k])) for k in n}
    # each key in the partition pyref gives it
    for r in range(R):
        k, _ = c.compute(r)
        assert all(pyref.get_partition(x, R) == r for x in k.tolist())


@pytest.mark.parametrize("where", ["host", "device", "borrowed"])
def test_input_locations_and_device_output(sc, where):
    import torch
    spec = "mixed"
    n, M, R = 20_000, 3, 11
    keys, cols = make_rows(41, spec, n)
    if where == "host":
        kcol = _StrCol(_host_keys(keys, 13))
        vcols = tuple(_Col(c, role="value") for c in cols)
    else:
        kcol = _StrCol(_device_keys(keys, 13))
        vcols = tuple(_Col(torch.from_numpy(c.copy()).cuda(), role="value") for c in cols)
        if where == "device":
            kcol.loc = L.VB_DEVICE
            for v in vcols:
                v.loc = L.VB_DEVICE
    parts, _ = str_combine(sc, spec, kcol, vcols, n, M, R)
    host_kcol, host_vcols = _StrCol(keys), tuple(_Col(c, role="value") for c in cols)
    want, _ = str_combine(sc, spec, host_kcol, host_vcols, n, M, R)
    for p, w in zip(parts, want):
        assert p.keys() == w.keys()
        dts, aggs = SPECS[spec]
        exact = [a for a, (op, c) in enumerate(aggs) if not (dts[c][0] == "f64" and op in ("sum", "mean"))]
        assert all([bits(p[k][a]) for a in exact] == [bits(w[k][a]) for a in exact] for k in p)
    check_against_singles(sc, spec, parts, keys, cols, host_kcol, host_vcols, n, M, R)
    # device output == host output, through StrCombinedRdd.compute_device
    rdd = sc.parallelize(keys, M, values=tuple(cols)).combine_by_key(
        {f"a{a}": (op, c) for a, (op, c) in enumerate(SPECS[spec][1])}, R)
    for r in range(R):
        ko, kb, outs = rdd.compute_raw(r)
        sh = rdd._run()
        nk, nb, nv = sh.reduce_size(r)
        assert nv == nk
        tko = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
        tkb = torch.empty(max(nb, 1), dtype=torch.uint8, device="cuda")
        tout = [torch.empty(max(nk, 1), dtype=torch.int64, device="cuda") for _ in outs]
        rdd.compute_device(r, tko, tkb, tout)
        assert tko.cpu().numpy().view(np.uint64).tolist() == ko.tolist()
        assert tkb.cpu().numpy()[:nb].tobytes() == kb.tobytes()
        for t, o in zip(tout, outs):
            assert t.cpu().numpy()[:nk].view(np.uint64).tolist() == o.view(np.uint64).tolist()


@pytest.mark.parametrize("shape", ["one_hot", "zipf", "all_distinct"])
def test_warp_paths(sc, shape):
    """One key for every row (each warp folds into one leader), Zipf keys, and warps of distinct keys (the shortcut)."""
    spec = "four"
    n = 100_000
    rng = np.random.default_rng(9)
    if shape == "one_hot":
        keys = ["the"] * n
    elif shape == "zipf":
        r = np.minimum(rng.zipf(1.3, n), 5000)
        keys = [f"w{x}" for x in r.tolist()]
    else:
        keys = [f"k{x:07d}" for x in rng.permutation(n).tolist()]
    cols = [rand_pairs(rng, n, 100, d, values=m)[1] for d, m in SPECS[spec][0]]
    kcol, vcols = _StrCol(keys), tuple(_Col(c, role="value") for c in cols)
    parts, st = str_combine(sc, spec, kcol, vcols, n, 4, 8)
    assert sum(len(p) for p in parts) == len(set(keys))
    check_against_singles(sc, spec, parts, keys, cols, kcol, vcols, n, 4, 8)


def test_index_growth_million_keys(sc):
    """10^6 distinct keys with hint 1: the dictionary index grows (table_restarts > 0) and the rerun encodes agree."""
    n = 1_200_000
    rng = np.random.default_rng(2)
    ids = rng.integers(0, 1_000_000, n)
    ids[:1_000_000] = rng.permutation(1_000_000)
    keys = [f"key-{x}" for x in ids.tolist()]
    v = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
    starts = vb.slice_starts(n, 4)
    sh = StrShuffle(sc, 4, 16, L.VB_U64, L.VB_AGG_SUM, hint=1,
                    multi=([L.VB_I64], [(L.VB_AGG_COUNT, 0), (L.VB_AGG_SUM, 0), (L.VB_AGG_MAX, 0)]))
    kcol, vc = _StrCol(keys), (_Col(v, role="value"),)
    for m in range(4):
        sh.map_cols(m, kcol, vc, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    st = sh.stats()
    assert st["table_restarts"] > 0
    cnt = np.bincount(ids, minlength=1_000_000)
    sums = np.bincount(ids, weights=v.astype(np.float64), minlength=1_000_000)     # |sums| < 2^53: exact
    mx = np.full(1_000_000, np.iinfo(np.int64).min)
    np.maximum.at(mx, ids, v)
    total = 0
    for r in range(16):
        ko, kb, (c, s, x) = sh.reduce_cols(r, [np.uint64, np.int64, np.int64])
        idx = np.array([int(k[4:]) for k in vb.rdd._decode_keys(ko, kb).tolist()], dtype=np.int64)
        total += len(idx)
        assert (c == cnt[idx]).all() and (s == sums[idx].astype(np.int64)).all() and (x == mx[idx]).all()
    assert total == 1_000_000
    sh.free()


def _fp_cases(sc):
    for spec, seed in (("mixed", 1), ("four", 2)):
        n, M, R = 20_000, 4, 13
        keys, cols = make_rows(seed, spec, n, n_pool=2000)
        kcol, vcols = _StrCol(keys), tuple(_Col(c, role="value") for c in cols)
        for hint in (0, 1):
            parts, _ = str_combine(sc, spec, kcol, vcols, n, M, R, hint=hint)
            check_against_singles(sc, spec, parts, keys, cols, kcol, vcols, n, M, R)


def test_forced_fingerprint_collisions():
    """VEGA_B200_STR_FP_BITS=4: distinct keys share fingerprints and are told apart by their bytes (a subprocess: the
    switch is read once per process)."""
    code = r'''
import vega_b200 as vb
from tests.test_gpu_str_combine import _fp_cases
with vb.Context(0) as sc:
    _fp_cases(sc)
print("fp ok")
'''
    env = dict(os.environ, VEGA_B200_STR_FP_BITS="4")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert out.returncode == 0 and "fp ok" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


SMALL = ([L.VB_U64, L.VB_I64], [(L.VB_AGG_SUM, 0), (L.VB_AGG_MIN, 1), (L.VB_AGG_MEAN, 1)])


def _map(sh, m, keys, u, i):
    sh.map_cols(m, _StrCol(keys), (_Col(np.asarray(u, dtype=np.uint64), role="value"),
                                   _Col(np.asarray(i, dtype=np.int64), role="value")), 0, len(keys))


def _all(sh, R):
    got = {}
    for r in range(R):
        got.update(decode(sh.reduce_cols(r, [np.uint64, np.int64, np.float64])))
    return got


def test_resubmitted_empty_maps_and_empty_shuffle(sc):
    sh = StrShuffle(sc, 3, 4, L.VB_U64, L.VB_AGG_SUM, multi=SMALL)
    _map(sh, 0, ["a", "gone", "a"], [1, 2, 3], [5, -1, 7])
    _map(sh, 1, [], [], [])
    _map(sh, 2, ["b"], [10], [-4])
    _map(sh, 0, ["a", "c"], [4, 6], [8, 9])                # replaces map 0: "gone" is dropped
    sh.seal()
    assert _all(sh, 4) == {"a": (4, 8, 8.0), "b": (10, -4, -4.0), "c": (6, 9, 9.0)}
    sh.free()
    sh = StrShuffle(sc, 2, 3, L.VB_U64, L.VB_AGG_SUM, multi=SMALL)
    _map(sh, 0, [], [], [])
    _map(sh, 1, [], [], [])
    sh.seal()
    assert _all(sh, 3) == {} and all(sh.reduce_size(r) == (0, 0, 0) for r in range(3))
    sh.free()
    # an unread column may be NULL and is not copied
    sh = StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_SUM, multi=([L.VB_U64, L.VB_I64], [(L.VB_AGG_COUNT, 0), (L.VB_AGG_MAX, 1)]))
    i = np.array([3, -9, 4], dtype=np.int64)
    sh.map_cols(0, _StrCol(["x", "y", "x"]), (None, _Col(i, role="value")), 0, 3)
    sh.seal()
    assert sh.stats()["h2d_bytes"] == 4 * 8 + 3 + 3 * 8                 # offsets, key bytes and column 1 only
    got = {}
    for r in range(2):
        got.update(decode(sh.reduce_cols(r, [np.uint64, np.int64])))
    assert got == {"x": (2, 4), "y": (1, -9)}
    sh.free()


def test_eight_threads_map_concurrently(sc):
    spec = "mixed"
    n, M, R = 80_000, 16, 9
    keys, cols = make_rows(77, spec, n)
    kcol, vcols = _StrCol(keys), tuple(_Col(c, role="value") for c in cols)
    starts = vb.slice_starts(n, M)
    sh = StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, multi=multi_of(spec))
    with ThreadPoolExecutor(8) as ex:
        list(ex.map(lambda m: sh.map_cols(m, kcol, vcols, int(starts[m]), int(starts[m + 1])), range(M)))
    sh.seal()
    parts = [decode(sh.reduce_cols(r, out_dtypes(spec))) for r in range(R)]
    sh.free()
    check_against_singles(sc, spec, parts, keys, cols, kcol, vcols, n, M, R)


def _code(fn, *args):
    return getattr(L.lib(), fn)(*args)


def test_rejected_calls(sc):
    lib = L.lib()
    h = ctypes.c_void_p()
    dts = (ctypes.c_int32 * 2)(L.VB_U64, L.VB_I64)
    spec = (L.vb_agg_col * 2)(L.vb_agg_col(L.VB_AGG_SUM, 0), L.vb_agg_col(L.VB_AGG_MAX, 1))
    # bad specs
    bad_spec = (L.vb_agg_col * 1)(L.vb_agg_col(L.VB_AGG_GROUP, 0))
    assert lib.vb_shuffle_create_str_multi(sc._h, 1, 1, 2, 2, dts, 1, bad_spec, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_create_str_multi(sc._h, 1, 1, 2, 5, dts, 2, spec, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_create_str_multi(sc._h, 1, 1, 2, 2, dts, 0, spec, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_create_str_multi_dist(sc._h, 1, 1, 2, 2, dts, 2, spec, 2, 2, ctypes.byref(h)) == L.VB_ERR_INVALID
    sh = StrShuffle(sc, 2, 3, L.VB_U64, L.VB_AGG_SUM, multi=([L.VB_U64, L.VB_I64], [(L.VB_AGG_SUM, 0), (L.VB_AGG_MAX, 1)]))
    s = sh._h
    offs = np.array([0, 1, 2], dtype=np.uint64)
    data = np.frombuffer(b"ab", dtype=np.uint8)
    u = np.array([1, 2], dtype=np.uint64)
    i = np.array([-1, 4], dtype=np.int64)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    vals = (ctypes.c_void_p * 2)(u.ctypes.data, i.ctypes.data)
    one = np.zeros(4, dtype=np.uint64)
    n = ctypes.c_uint64()
    # other calls on this shuffle kind
    assert lib.vb_shuffle_map_str(s, 0, p(offs), p(data), 2, p(u), 2, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_map_soa(s, 0, p(u), p(u), 2, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_map_aos(s, 0, p(one), 2, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_map_cols(s, 0, p(u), vals, 2, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_set_key_width(s, 4) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_set_dist(s, 0, 2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_map_blob(s, 0, p(one), 8, L.VB_HOST) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_exchange(s, L.VB_XCHG_P2P) == L.VB_ERR_UNSUPPORTED
    na, nb_ = (ctypes.c_uint64 * 1)(), (ctypes.c_uint64 * 1)()
    assert lib.vb_shuffle_export_str_cols_prepare(s, na, nb_) == L.VB_ERR_STATE              # world 1
    assert lib.vb_shuffle_import_str_cols(s, None, None, None, 2, na, nb_) == L.VB_ERR_STATE
    assert lib.vb_shuffle_export_str_prepare(s, na, nb_, na) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_export_cols_prepare(s, na) == L.VB_ERR_INVALID
    # a NULL column that an aggregate reads
    assert lib.vb_shuffle_map_str_cols(s, 0, p(offs), p(data), 2, (ctypes.c_void_p * 2)(u.ctypes.data, None), 2, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_map_str_cols(s, 2, p(offs), p(data), 2, vals, 2, L.VB_HOST) == L.VB_ERR_INVALID     # map id
    assert lib.vb_shuffle_map_str_cols(s, 0, p(offs), p(data), 1, vals, 2, L.VB_HOST) == L.VB_ERR_INVALID     # offsets past n_bytes
    assert lib.vb_shuffle_map_str_cols(s, 0, p(offs), p(data), 2, vals, 2, L.VB_HOST) == L.VB_OK
    assert lib.vb_shuffle_map_str_cols(s, 1, p(offs), p(data), 2, vals, 2, L.VB_HOST) == L.VB_OK
    assert lib.vb_shuffle_seal(s) == L.VB_OK
    assert lib.vb_shuffle_reduce_size(s, 0, ctypes.byref(n), None) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce(s, 0, None, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_cols(s, 0, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_blob_size(s, 0, ctypes.byref(n)) == L.VB_ERR_UNSUPPORTED
    nt = ctypes.c_void_p()
    assert lib.vb_shuffle_create_narrow(s, 0, ctypes.byref(nt)) == L.VB_ERR_INVALID
    sides = (ctypes.c_void_p * 1)(s)
    assert lib.vb_cogroup_n_str_size(sides, 1, 0, ctypes.byref(n), ctypes.byref(n), None) == L.VB_ERR_INVALID
    assert lib.vb_join_n_str_size(sides, 1, 0, 1, ctypes.byref(n), ctypes.byref(n), ctypes.byref(n)) == L.VB_ERR_INVALID
    assert lib.vb_cogroup_n_size(sides, 1, 0, ctypes.byref(n), None) == L.VB_ERR_INVALID
    assert lib.vb_join_size(s, s, 0, ctypes.byref(n)) == L.VB_ERR_INVALID
    # vb_shuffle_reduce_str: the keys only
    r = next(r for r in range(3) if sh.reduce_size(r)[0])
    nk, nbytes, nv = sh.reduce_size(r)
    ko, kb, comb = np.empty(nk + 1, np.uint64), np.empty(nbytes, np.uint8), np.empty(nk, np.uint64)
    assert lib.vb_shuffle_reduce_str(s, r, p(ko), p(kb), p(comb), None, None, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_str(s, r, p(ko), p(kb), None, p(ko), None, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_str(s, r, p(ko), p(kb), None, None, p(comb), L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_str(s, r, p(ko), p(kb), None, None, None, L.VB_HOST) == L.VB_OK
    assert ko[0] == 0 and ko[-1] == nbytes
    sh.free()
    # the new calls on any other shuffle
    others = [StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_SUM),
              Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, multi=([L.VB_U64], [(L.VB_AGG_SUM, 0)])),
              Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM)]
    for o in others:
        assert lib.vb_shuffle_map_str_cols(o._h, 0, p(offs), p(data), 2, vals, 2, L.VB_HOST) == L.VB_ERR_INVALID
        assert lib.vb_shuffle_reduce_str_cols(o._h, 0, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
        assert lib.vb_shuffle_export_str_cols_prepare(o._h, na, nb_) == L.VB_ERR_INVALID
        assert lib.vb_shuffle_export_str_cols_buffers(o._h, None, None, None, None) == L.VB_ERR_INVALID
        assert lib.vb_shuffle_import_str_cols(o._h, None, None, None, 1, na, nb_) == L.VB_ERR_INVALID
        o.free()


def test_property_twenty_million_rows(sc):
    """2 x 10^7 word-like device keys (Zipf over 10^6 ranks) with the combine spec of tools/bench_ops.py, against the
    integer combine over the same rows keyed by each word's rank: every column bit for bit (integer values)."""
    import torch
    n, D = 20_000_000, 1_000_000
    ranks = torch.empty(n, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=ranks, n=n, mode="zipf", n_distinct=D, zipf_s=1.1)
    ranks = ranks & ((1 << 40) - 1)
    g = torch.Generator(device="cuda").manual_seed(5)
    v0 = torch.randint(-(1 << 62), 1 << 62, (n,), device="cuda", generator=g)
    v1 = torch.randint(-(1 << 62), 1 << 62, (n,), device="cuda", generator=g)
    keys = _device_words(ranks)
    torch.cuda.synchronize()
    aggs = {"s": ("sum", 0), "lo": ("min", 1), "hi": ("max", 1), "avg": ("mean", 0), "n": ("count", None)}
    M, R = 8, 16
    got_k, got = sc.parallelize(keys, M, values=(v0, v1)).combine_by_key(aggs, R).collect()
    want_k, want = sc.parallelize(ranks, M, values=(v0, v1)).combine_by_key(aggs, R).collect()
    assert len(got_k) == len(want_k) == len(torch.unique(ranks))
    assert int(got["n"].sum()) == n
    idx = np.array([int(w[1:], 16) for w in got_k.tolist()], dtype=np.uint64)
    order_g, order_w = np.argsort(idx), np.argsort(want_k.view(np.uint64))
    assert (idx[order_g] == want_k.view(np.uint64)[order_w]).all()
    for name in aggs:
        assert (got[name][order_g].view(np.uint64) == want[name][order_w].view(np.uint64)).all(), name


def test_cpp_example_combine_by_key_string():
    exe = os.path.join(ROOT, "examples", "_build", "combine_by_key_string")
    assert os.path.exists(exe), "built by __graft_entry__.build()"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ok" in out.stdout.splitlines()[-1]
