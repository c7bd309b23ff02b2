"""combine_by_key: several named aggregates per key in one shuffle, through every hash-aggregate path, against the
single-column references.

Every output column is checked on its own: integer SUM/MIN/MAX, COUNT and f64 MIN/MAX bit for bit against the CPU
oracle's single-column shuffle, f64 SUM with tests/util.py:assert_f64_sums, integer MEAN as (double)oracle_sum /
oracle_count with the sum read with the column's signedness, and f64 MEAN as the f64 SUM outcome of
tests/f64_sum_ref.py divided by the count.  Each path asserts the statistic that proves it ran."""
import ctypes
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import vega_b200 as vb
from oracle import oracle as O
from tests.test_gpu_reduce_paths import _col, _dev
from tests import f64_sum_ref as F
from tests.util import assert_f64_sums, assert_parts_equal, bits_dict, oracle_reduce_bits, rand_pairs
from vega_b200 import _lib as L
from vega_b200.rdd import Shuffle, _Col

pytestmark = pytest.mark.gpu

AGG = {"sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT, "mean": L.VB_AGG_MEAN}
NP = {"u64": np.uint64, "i64": np.int64, "f64": np.float64}
CODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}
# (value column dtypes with their rand_pairs modes, aggregates as (op, column))
SPECS = {
    # 4 columns, 8 aggregates; the MEANs share the spec's COUNT
    "four": ([("u64", "full"), ("i64", "full"), ("f64", "exact"), ("f64", "special")],
             [("count", 0), ("sum", 0), ("max", 1), ("mean", 1), ("sum", 2), ("mean", 2), ("min", 3), ("max", 3)]),
    # 3 columns, 7 aggregates + the internal COUNT of the MEANs
    "mixed": ([("u64", "full"), ("i64", "full"), ("f64", "cancel")],
              [("min", 0), ("max", 0), ("mean", 0), ("sum", 1), ("min", 1), ("mean", 2), ("sum", 2)]),
    # 1 column, 8 aggregates
    "one": ([("f64", "subnormal")],
            [("count", 0), ("sum", 0), ("min", 0), ("max", 0), ("mean", 0), ("sum", 0), ("min", 0), ("max", 0)]),
}


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def spec_of(spec):
    """(value dtypes with modes, aggregates) of a SPECS name, or such a pair itself."""
    return SPECS[spec] if isinstance(spec, str) else spec


def make_data(seed, spec, n, n_keys, hot=0.0):
    """Keys and the value columns of a spec.  The keys come with the first f64 column (cancelling pairs share a key);
    the other columns are drawn independently over the same rows."""
    rng = np.random.default_rng(seed)
    dts = SPECS[spec][0]
    lead = next((i for i, (d, _) in enumerate(dts) if d == "f64"), 0)
    keys, lead_vals = rand_pairs(rng, n, n_keys, dts[lead][0], values=dts[lead][1], hot=hot)
    cols = [lead_vals if i == lead else rand_pairs(rng, n, n_keys, d, values=m)[1] for i, (d, m) in enumerate(dts)]
    return keys, cols


def out_dtype(spec, a):
    op, c = spec_of(spec)[1][a]
    return np.uint64 if op == "count" else np.float64 if op == "mean" else NP[spec_of(spec)[0][c][0]]


def run_combine(sc, spec, kcol, vcols, n, M, R, hint=0, key_width=8, dst=L.VB_HOST):
    """One multi-aggregate shuffle: M map tasks over rows [0, n) as ParallelCollection slices them, seal, every
    reduce partition as (keys, [column per aggregate])."""
    dts, aggs = spec_of(spec)
    starts = vb.slice_starts(n, M)
    sh = Shuffle(sc, len(starts) - 1, R, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, key_width=key_width, hint=hint,
                 multi=([CODE[d] for d, _ in dts], [(AGG[op], c) for op, c in aggs]))
    try:
        for m in range(len(starts) - 1):
            sh.map_cols(m, kcol, vcols, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        outs = [out_dtype(spec, a) for a in range(len(aggs))]
        if dst == L.VB_HOST:
            parts = [sh.reduce_cols(r, outs) for r in range(R)]
        else:
            import torch
            parts = []
            for r in range(R):
                nk, _ = sh.reduce_size(r)
                tk = torch.empty(nk, dtype=torch.int64, device="cuda")
                ta = [torch.empty(nk, dtype=torch.int64, device="cuda") for _ in outs]
                sh.reduce_cols(r, outs, L.VB_DEVICE, tk, ta)
                parts.append((tk.cpu().numpy().view(np.uint64), [t.cpu().numpy().view(dt) for t, dt in zip(ta, outs)]))
        st = sh.stats()
    finally:
        sh.free()
    return parts, st


def check_f64_means(got_parts, keys, vals, exact=False, lenient=None):
    """Per key: a mean tests/f64_sum_ref.py admits, the SUM outcome over the count: fl(sum / m) bit for bit where the
    sum is exact, NaN and infinities as the sum's, within the SUM bound over m (plus the division's rounding) otherwise."""
    got = {}
    for d in got_parts:
        got.update(d)
    F.assert_outcomes(got, F.key_outcomes(keys, vals, mean=True), "f64 means", exact=exact, lenient=lenient)


def check_combine(parts, spec, keys, cols, R, key_width=8, lenient=None):
    """lenient: the keys whose f64 SUM / MEAN may take more than one outcome class (tests/f64_sum_ref.py)."""
    dts, aggs = spec_of(spec)
    kw = key_width
    oracle = {}

    def ref(op, c):
        if (op, c) not in oracle:
            d = dts[c][0] if op != "count" else "u64"
            oracle[(op, c)] = oracle_reduce_bits(op, keys, None if op == "count" else cols[c], 4, R, d, kw, threads=4)
        return oracle[(op, c)]

    count = ref("count", 0)
    for a, (op, c) in enumerate(aggs):
        d, mode = dts[c]
        if op == "sum" and d == "f64":
            got = [dict(zip(k.view(np.uint64).tolist(), o[a].tolist())) for k, o in parts]
            assert_f64_sums(got, keys, cols[c], R, key_width=kw, exact=mode in ("exact", "subnormal"), lenient=lenient)
        elif op == "mean" and d == "f64":
            got = [dict(zip(k.view(np.uint64).tolist(), o[a].tolist())) for k, o in parts]
            check_f64_means(got, keys, cols[c], exact=mode in ("exact", "subnormal"), lenient=lenient)
        elif op == "mean":
            sums = ref("sum", c)
            want = []
            for sp, cp in zip(sums, count):
                w = {}
                for k, s in sp.items():
                    s = s - (1 << 64) if d == "i64" and s >= 1 << 63 else s
                    w[k] = int(np.float64(np.float64(s) / np.float64(cp[k])).view(np.uint64))
                want.append(w)
            assert_parts_equal([bits_dict(k, o[a]) for k, o in parts], want)
        else:
            assert_parts_equal([bits_dict(k, o[a]) for k, o in parts], ref(op, c))


# ---- the path matrix ------------------------------------------------------------------------------------------------
# name: (rows, keys, hot-key share, R)
PATHS = {
    "register_small": (150_000, 20_000, 0.0, 7),      # host input, 5 map tasks of 30k rows: register-staged kernel
    "bulk_soa_tail": (1_000_003, 50_000, 0.0, 7),     # device columns, 1 map task, n % 1024 != 0
    "shared_borrowed": (400_000, 100_000, 0.0, 7),    # device input, 4 map tasks: one shared table, no merge
    "per_map_merge": (400_000, 100_000, 0.0, 7),      # host input, 4 map tasks: per-map tables merged at seal
    "restart_per_map": (300_000, 120_000, 0.0, 7),    # host input, hint=100: the per-map tables overflow
    "restart_shared": (300_000, 120_000, 0.0, 7),     # device input, hint=100: the shared table overflows
    "hot_key_cache": (4_000_000, 200_000, 0.12, 7),   # one map task, top key 12 % of rows: the per-CTA cache absorbs it
    "register_hot": (4_000_000, 200_000, 0.12, 7),    # the hot_key_cache rows as misaligned device columns: the
                                                      # register-staged kernel keeps its cache past the learning tiles
}


def _cols(keys, cols, spec, device, misalign=False):
    dts = spec_of(spec)[0]
    if not device:
        return _Col(keys), tuple(_Col(c, role="value") for c in cols)
    return _col(_dev(keys, misalign), L.VB_U64), tuple(_col(_dev(c, misalign), CODE[d]) for c, (d, _) in zip(cols, dts))


def _run_path(sc, path, spec, keys, cols):
    R, n = PATHS[path][3], len(keys)
    device = path in ("bulk_soa_tail", "shared_borrowed", "restart_shared", "hot_key_cache", "register_hot")
    kc, vcs = _cols(keys, cols, spec, device, misalign=path == "register_hot")
    M = {"register_small": 5, "bulk_soa_tail": 1, "shared_borrowed": 4, "per_map_merge": 4, "restart_per_map": 2,
         "restart_shared": 4, "hot_key_cache": 1, "register_hot": 1}[path]
    hint = 100 if path.startswith("restart") else 0
    parts, st = run_combine(sc, spec, kc, vcs, n, M, R, hint=hint)
    if path in ("register_small", "register_hot"):
        assert st["hot_kernel_variant"] == 0
    elif path in ("bulk_soa_tail", "hot_key_cache"):
        assert st["hot_kernel_variant"] == 1
    elif path == "shared_borrowed":
        assert st["hot_kernel_variant"] == 1 and st["kernels"]["merge"]["launches"] == 0
    elif path == "per_map_merge":
        assert st["kernels"]["merge"]["launches"] >= 1
    else:
        assert st["table_restarts"] >= 1
    return parts, R


def _path_data(path, spec):
    data = "hot_key_cache" if path == "register_hot" else path     # register_hot: the same rows, placed differently
    n, nkeys, hot, R = PATHS[data]
    return make_data([sorted(set(PATHS) - {"register_hot"}).index(data), sorted(SPECS).index(spec), 1], spec, n, nkeys, hot)


@pytest.mark.parametrize("spec", list(SPECS))
@pytest.mark.parametrize("path", list(PATHS))
def test_combine_path_matches_single_column_references(sc, path, spec):
    keys, cols = _path_data(path, spec)
    if path in ("hot_key_cache", "register_hot"):
        assert np.unique(keys, return_counts=True)[1].max() > 0.05 * len(keys)
    parts, R = _run_path(sc, path, spec, keys, cols)
    check_combine(parts, spec, keys, cols, R)


@pytest.mark.parametrize("R", [1, 65536])
def test_combine_partition_counts(sc, R):
    keys, cols = make_data([R, 1], "four", 200_000, 60_000)
    kc, vcs = _cols(keys, cols, "four", device=False)
    parts, _ = run_combine(sc, "four", kc, vcs, len(keys), 3, R)
    check_combine(parts, "four", keys, cols, R)


@pytest.mark.parametrize("key_width", [8, 4])
def test_combine_places_keys_like_a_single_column_shuffle(sc, key_width):
    rng = np.random.default_rng(key_width)
    n, R = 100_000, 13
    if key_width == 4:
        k32 = rng.integers(-3000, 3000, n).astype(np.int32)
        k32[:4] = [-1, -(1 << 31), (1 << 31) - 1, 0]
        kc, wide = _Col(k32), k32.astype(np.int64).view(np.uint64)
    else:
        wide, _ = rand_pairs(rng, n, 20_000, "u64", values="full")
        kc = _Col(wide)
    assert kc.key_width == key_width
    v = rng.integers(0, 1 << 40, n).astype(np.uint64)
    parts, _ = run_combine(sc, "one", kc, (_Col(v.view(np.float64), role="value"),), n, 3, R, key_width=key_width)
    single = Shuffle(sc, 3, R, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, key_width=key_width)
    starts = vb.slice_starts(n, 3)
    for m in range(3):
        single.map(m, kc, _Col(v, role="value"), int(starts[m]), int(starts[m + 1]))
    single.seal()
    for r, (k, _) in enumerate(parts):
        ku = k.view(np.uint64)
        assert all(vb.lib().vb_get_partition(int(x), key_width, R) == r for x in ku.tolist())
        assert set(ku.tolist()) == set(single.reduce(r)[0].view(np.uint64).tolist())
    single.free()
    assert sum(len(k) for k, _ in parts) == len(np.unique(wide))


def test_combine_empty_map_partitions(sc):
    keys, cols = make_data(5, "mixed", 3, 2)
    for device in (False, True):
        kc, vcs = _cols(keys, cols, "mixed", device)
        parts, _ = run_combine(sc, "mixed", kc, vcs, 3, 8, 4)          # 8 map tasks over 3 rows: most are empty
        check_combine(parts, "mixed", keys, cols, 4)
    kc, vcs = _cols(keys[:0], [c[:0] for c in cols], "mixed", False)
    parts, st = run_combine(sc, "mixed", kc, vcs, 0, 3, 4)
    assert all(len(k) == 0 for k, _ in parts) and st["rows_out"] == 0


def test_combine_concurrent_map_threads(sc):
    keys, cols = make_data(6, "four", 800_000, 50_000)
    dts, aggs = SPECS["four"]
    kc, vcs = _cols(keys, cols, "four", device=False)
    M, R = 8, 5
    starts = vb.slice_starts(len(keys), M)
    sh = Shuffle(sc, M, R, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, multi=([CODE[d] for d, _ in dts], [(AGG[o], c) for o, c in aggs]))
    with ThreadPoolExecutor(M) as ex:
        list(ex.map(lambda m: sh.map_cols(m, kc, vcs, int(starts[m]), int(starts[m + 1])), range(M)))
    sh.seal()
    parts = [sh.reduce_cols(r, [out_dtype("four", a) for a in range(len(aggs))]) for r in range(R)]
    sh.free()
    check_combine(parts, "four", keys, cols, R)


def test_combine_device_output_equals_host_output(sc):
    keys, cols = make_data(7, "four", 300_000, 40_000)
    kc, vcs = _cols(keys, cols, "four", device=True)
    host, _ = run_combine(sc, "four", kc, vcs, len(keys), 2, 6)
    dev, _ = run_combine(sc, "four", kc, vcs, len(keys), 2, 6, dst=L.VB_DEVICE)
    for (hk, ho), (dk, do) in zip(host, dev):
        oh, od = np.argsort(hk.view(np.uint64)), np.argsort(dk)
        assert np.array_equal(hk.view(np.uint64)[oh], dk[od])
        for a, b in zip(ho, do):
            assert np.array_equal(a.view(np.uint64)[oh], b.view(np.uint64)[od])


def test_combine_by_key_python_api(sc):
    keys, cols = make_data(8, "mixed", 200_000, 30_000)
    aggs = {"lo": ("min", 0), "n": ("count", None), "avg": ("mean", 1), "hi": ("max", 1)}
    tk, tcols = _dev(keys), (_dev(cols[0]), _dev(cols[1]))
    rdd = sc.parallelize(keys, 4, values=(cols[0], cols[1]))
    k, out = rdd.combine_by_key(aggs, 5).collect()
    assert list(out) == ["lo", "n", "avg", "hi"]
    assert out["n"].dtype == np.uint64 and out["avg"].dtype == np.float64 and out["lo"].dtype == np.uint64
    assert out["hi"].dtype == np.int64
    want_n = {k: v for p in oracle_reduce_bits("count", keys, None, 4, 5) for k, v in p.items()}
    want_hi = {k: v for p in oracle_reduce_bits("max", keys, cols[1], 4, 5, "i64") for k, v in p.items()}
    assert dict(zip(k.view(np.uint64).tolist(), out["n"].tolist())) == want_n
    assert bits_dict(k, out["hi"]) == want_hi
    # torch CUDA tensors (int64 carrying u64 bits): same keys and counts, compute(r) gives one partition
    kd, od = sc.parallelize(tk, 4, values=(tcols[0], tcols[1])).combine_by_key({"n": ("count", None)}, 5).collect()
    assert dict(zip(kd.view(np.uint64).tolist(), od["n"].tolist())) == want_n
    k0, o0 = rdd.combine_by_key(aggs, 5).compute(0)
    assert set(k0.view(np.uint64).tolist()) == {x for x in want_n if O.get_partition(x, 5, 8) == 0}


def test_combine_rejections(sc):
    dts, aggs = SPECS["four"]
    multi = ([CODE[d] for d, _ in dts], [(AGG[o], c) for o, c in aggs])
    keys = np.arange(100, dtype=np.uint64)
    sh = Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, multi=multi)
    lib, h = vb.lib(), sh._h
    p = keys.ctypes.data
    assert lib.vb_shuffle_set_dist(h, 0, 2) == L.VB_ERR_UNSUPPORTED
    assert b"not supported" in lib.vb_last_error()
    assert lib.vb_shuffle_map_aos(h, 0, p, 50, L.VB_HOST) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_map_soa(h, 0, p, p, 100, L.VB_HOST) == L.VB_ERR_INVALID
    cnt = (ctypes.c_uint64 * 2)()
    assert lib.vb_shuffle_export_prepare(h, cnt) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_counts(h, cnt) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_import(h, None, None, cnt) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_direct(h, cnt, cnt) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_import_arena(h, cnt) == L.VB_ERR_UNSUPPORTED
    kp, vp = ctypes.c_void_p(), ctypes.c_void_p()
    assert lib.vb_shuffle_export_buffers(h, ctypes.byref(kp), ctypes.byref(vp)) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_exchange(h, L.VB_XCHG_AUTO) == L.VB_ERR_UNSUPPORTED
    blob = np.zeros(3, dtype=np.uint64)
    assert lib.vb_shuffle_map_blob(h, 0, blob.ctypes.data, 24, L.VB_HOST) == L.VB_ERR_UNSUPPORTED
    vcs = tuple(_Col(keys.view(NP[d]) if d != "f64" else keys.astype(np.float64), role="value") for d, _ in dts)
    sh.map_cols(0, _Col(keys), vcs, 0, 100)
    sh.seal()
    n = ctypes.c_uint64()
    assert lib.vb_shuffle_reduce_blob_size(h, 0, ctypes.byref(n)) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_reduce_blob(h, 0, blob.ctypes.data, L.VB_HOST) == L.VB_ERR_UNSUPPORTED
    out = np.empty(100, dtype=np.uint64)
    assert lib.vb_shuffle_reduce(h, 0, out.ctypes.data, out.ctypes.data, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce(h, 0, out.ctypes.data, None, None, None, L.VB_HOST) == L.VB_OK
    assert lib.vb_join_size(h, h, 0, ctypes.byref(n)) == L.VB_ERR_INVALID
    sh.free()
    # bad specs: too many aggregates (a MEAN's COUNT included), column out of range, a group op
    for bad in ([(L.VB_AGG_MEAN, 0)] * 8, [(L.VB_AGG_SUM, 4)], [(L.VB_AGG_GROUP, 0)], [(L.VB_AGG_SORT, 0)], [(L.VB_AGG_SUM, 0)] * 9):
        with pytest.raises(vb.VegaB200Error) as e:
            Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, multi=(multi[0], bad))
        assert e.value.code == L.VB_ERR_INVALID
    with pytest.raises(vb.VegaB200Error) as e:
        Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, multi=([L.VB_U64] * 5, [(L.VB_AGG_SUM, 0)]))
    assert e.value.code == L.VB_ERR_INVALID
