"""String keys on the device (vb_shuffle_create_str and the StrRdd / StrPairRdd mirror): every partition is checked
against oracle/pyref.py, which hashes a `str` as Rust's `impl Hash for str` does (UTF-8 bytes, then 0xFF).  Each key
appears exactly once, in pyref.get_partition's partition, with its value bit for bit (f64 SUM within the error bound
of any summation order)."""
import ctypes
import math
import os
import struct
import subprocess
import sys
import threading

import numpy as np
import pytest

import vega_b200 as vb
from vega_b200 import _lib as L
from oracle import oracle as O
from oracle import pyref
from tests.util import rand_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


# ---- references ---------------------------------------------------------------------------------------------------
def _tkey(x):
    b = struct.unpack("<Q", struct.pack("<d", x))[0]
    return (~b & M64) if b >> 63 else (b | (1 << 63))


def _fmin(a, b):      # f64::min: a NaN is ignored; -0.0 < +0.0
    if math.isnan(a):
        return b
    if math.isnan(b):
        return a
    return a if _tkey(a) <= _tkey(b) else b


def _fmax(a, b):
    if math.isnan(a):
        return b
    if math.isnan(b):
        return a
    return a if _tkey(a) >= _tkey(b) else b


def _fold(op, vdt):
    if op == "sum":
        if vdt == "u64":
            return lambda a, b: (a + b) & M64
        if vdt == "i64":
            return lambda a, b: ((a + b + (1 << 63)) & M64) - (1 << 63)
        return lambda a, b: a + b            # checked against fsum with a bound, not bit for bit
    if vdt == "f64":
        return _fmin if op == "min" else _fmax
    return min if op == "min" else max


def ref_parts(keys, vals, op, vdt, M, R):
    """pyref reduce_by_key / count_by_key / group_by_key, bucketed by pyref.get_partition."""
    py_vals = [1] * len(keys) if op == "count" else vals.tolist()
    rows = list(zip(keys, py_vals))
    if op == "group":
        res = pyref.group_by_key(rows, M, R)
    else:
        res = pyref.reduce_by_key(rows, _fold("sum" if op == "count" else op, "u64" if op == "count" else vdt), M, R)
    parts = [dict() for _ in range(R)]
    for k, v in res:
        parts[pyref.get_partition(k, R)][k] = v
    return parts


def _bits(x, vdt):
    if vdt == "f64":
        return "nan" if math.isnan(x) else struct.unpack("<Q", struct.pack("<d", x))[0]
    return int(x)


def gpu_parts(sh, op):
    out = []
    for r in range(sh.n_reduce):
        p = sh.reduce(r)
        keys = p[0].tolist()
        assert len(set(keys)) == len(keys), f"a key twice in partition {r}"
        if op == "group":
            o, v = p[1].astype(np.int64), p[2]
            out.append({k: v[o[i]:o[i + 1]].tolist() for i, k in enumerate(keys)})
        else:
            out.append(dict(zip(keys, p[1].tolist())))
    return out


def check_parts(got, want, op, vdt):
    assert len(got) == len(want)
    for r, (g, w) in enumerate(zip(got, want)):
        assert g.keys() == w.keys(), (r, sorted(g.keys() - w.keys())[:5], sorted(w.keys() - g.keys())[:5])
        for k in w:
            if op == "group":
                assert [_bits(x, vdt) for x in g[k]] == [_bits(x, vdt) for x in w[k]], (r, k)
            else:
                assert _bits(g[k], vdt) == _bits(w[k], vdt), (r, k, g[k], w[k])


def run_case(sc, keys, vals, op, vdt, M, R, hint=0):
    """keys: list of str; vals: numpy array (ignored by count).  Runs the mirror and checks it against pyref; f64 SUM
    against the exact sum of each key's values within the error bound of any summation order."""
    rdd = sc.parallelize(keys, M, values=vals)
    if op == "group":
        s = rdd.group_by_key(R)
    elif op == "count":
        s = rdd.count_by_key(R, hint)
    else:
        s = rdd.reduce_by_key(op, R, hint)
    got = gpu_parts(s._run(), op)
    want = ref_parts(keys, vals, op, vdt, len(vb.slice_starts(len(keys), M)) - 1, R)
    if op == "sum" and vdt == "f64":
        per_key = {}
        for k, v in zip(keys, vals.tolist()):
            per_key.setdefault(k, []).append(v)
        for r, (g, w) in enumerate(zip(got, want)):
            assert g.keys() == w.keys(), r
            for k, x in g.items():
                xs = per_key[k]
                if any(math.isnan(v) for v in xs) or (math.inf in xs and -math.inf in xs):
                    assert math.isnan(x), k
                elif math.inf in xs or -math.inf in xs:
                    assert x == (math.inf if math.inf in xs else -math.inf), k
                else:
                    m, u = len(xs), 2.0 ** -53
                    bound = (m - 1) * u / (1 - (m - 1) * u) * sum(abs(v) for v in xs) * (1 + 2 * m * u)
                    s_ = math.fsum(xs)
                    assert abs(x - s_) <= bound + math.ulp(s_), (k, x, s_)
    else:
        check_parts(got, want, op, vdt)
    return s


# ---- key pools ------------------------------------------------------------------------------------------------------
def key_pool(rng, n_random=200):
    """Lengths around MetroHash's 8 / 16 / 32-byte steps, prefixes of one another, last-byte differences, NULs,
    non-ASCII UTF-8, and a 10 kB key."""
    ks = ["", "\x00", "\x00\x00", "a\x00", "\x00a", "x", "y", "é", "日本語", "ünïcödé-ключ", "🙂" * 5]
    for n in list(range(1, 9)) + [15, 16, 17, 31, 32, 33, 63, 64, 65]:
        ks.append("k" * n)
        ks.append("k" * (n - 1) + "j")
    base = "abcdefghijklmnopqrstuvwxyz0123456789" * 3
    ks += [base[:i] for i in range(1, 80, 3)]
    ks += ["z" * 10_000, "z" * 9_999 + "y"]
    alpha = list("abcdefgh\x00é")
    for _ in range(n_random):
        ks.append("".join(rng.choice(alpha, int(rng.integers(0, 24)))))
    return sorted(set(ks))


def rows_from_pool(rng, pool, n):
    idx = rng.integers(0, len(pool), n)
    return [pool[i] for i in idx]


# ---- the reference's own test -----------------------------------------------------------------------------------------
def test_reference_group_by_key_string_keys(sc):
    """tests/test_pair_rdd.rs:8-37 / examples/group_by.rs with the real "x" / "y" keys."""
    vec = [("x", i) for i in range(1, 8)] + [("y", i) for i in range(1, 9)]
    keys = [k for k, _ in vec]
    vals = np.array([v for _, v in vec], dtype=np.int64)
    g = sc.parallelize(keys, 4, values=vals).group_by_key(4).collect()
    res = sorted((k, v.tolist()) for k, v in g.to_list())
    assert res == [("x", [1, 2, 3, 4, 5, 6, 7]), ("y", [1, 2, 3, 4, 5, 6, 7, 8])]
    assert sorted(g.to_dict()) == ["x", "y"]
    run_case(sc, keys, vals, "group", "i64", 4, 4)


def test_cpp_example_group_by_string():
    exe = os.path.join(ROOT, "examples", "_build", "group_by_string")
    if not os.path.exists(exe):
        pytest.skip("examples not built")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert 'result: [("x", [1, 2, 3, 4, 5, 6, 7]), ("y", [1, 2, 3, 4, 5, 6, 7, 8])]' in out.stdout, out.stdout
    assert '("question", 2)' in out.stdout and '("word", 1)' in out.stdout, out.stdout


# ---- ops x dtypes at full value range -----------------------------------------------------------------------------
OPS = [("sum", "u64", "full"), ("sum", "i64", "full"), ("min", "u64", "full"), ("min", "i64", "full"), ("max", "u64", "full"),
       ("max", "i64", "full"), ("min", "f64", "special"), ("max", "f64", "special"), ("sum", "f64", "cancel"),
       ("sum", "f64", "exact"), ("sum", "f64", "default"), ("count", "u64", "default"), ("group", "u64", "full"), ("group", "f64", "special")]


@pytest.mark.parametrize("op,vdt,mode", OPS)
@pytest.mark.parametrize("R", [1, 7, 300])
def test_ops_match_reference(sc, op, vdt, mode, R):
    rng = np.random.default_rng(hash((op, vdt, mode, R)) & 0xFFFF)
    pool = key_pool(rng)
    n = 6000
    keys = rows_from_pool(rng, pool, n)
    _, vals = rand_pairs(rng, n, 100, vdtype=vdt, values=mode)
    run_case(sc, keys, vals, op, vdt, 5, R)


def test_count_by_value_and_distinct(sc):
    rng = np.random.default_rng(3)
    pool = key_pool(rng)
    xs = rows_from_pool(rng, pool, 5000)
    rdd = sc.parallelize(xs, 6)
    k, c = rdd.count_by_value().collect()
    want = dict(pyref.count_by_value(xs, 6))
    assert dict(zip(k.tolist(), c.tolist())) == want
    assert len(k) == len(set(k.tolist()))
    d = rdd.distinct(5).collect()
    assert sorted(d.tolist()) == sorted(pyref.distinct(xs, 6, 5))
    assert len(d) == len(set(xs))


def test_partition_by_key(sc):
    rng = np.random.default_rng(4)
    pool = key_pool(rng)
    keys = rows_from_pool(rng, pool, 3000)
    vals = np.arange(3000, dtype=np.uint64)
    parts = sc.parallelize(keys, 4, values=vals).partition_by_key(5).glom()
    for r, p in enumerate(parts):
        assert sorted(p.tolist()) == sorted(i for i, k in enumerate(keys) if pyref.get_partition(k, 5) == r)


# ---- input / output locations -------------------------------------------------------------------------------------
def _device_keys(keys, shift=0):
    """StrKeys on the device whose offsets start at `shift` (junk bytes before the first key)."""
    import torch
    h = vb.StrKeys.from_strs(keys)
    data = np.concatenate([np.full(shift, 0xAB, dtype=np.uint8), h.data])
    offs = h.offsets.astype(np.int64) + shift
    return vb.StrKeys(torch.from_numpy(offs).cuda(), torch.from_numpy(data).cuda())


def _host_keys(keys, shift=0):
    h = vb.StrKeys.from_strs(keys)
    return vb.StrKeys(h.offsets + np.uint64(shift), np.concatenate([np.full(shift, 7, dtype=np.uint8), h.data]))


@pytest.mark.parametrize("where", ["host", "device", "borrowed"])
@pytest.mark.parametrize("op", ["sum", "max", "count", "group"])
def test_input_locations_and_offsets_not_from_zero(sc, where, op):
    import torch
    rng = np.random.default_rng(5)
    pool = key_pool(rng)
    n = 4000
    keys = rows_from_pool(rng, pool, n)
    vals = rng.integers(-(1 << 62), 1 << 62, n).astype(np.int64)
    M, R = 3, 11
    agg = {"sum": L.VB_AGG_SUM, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT, "group": L.VB_AGG_GROUP}[op]
    sh = vb.StrShuffle(sc, M, R, L.VB_I64, agg)
    if where == "host":
        col, vcol = vb.rdd._StrCol(_host_keys(keys, 13)), vb.rdd._Col(vals, role="value")
    else:
        col = vb.rdd._StrCol(_device_keys(keys, 13))
        tv = torch.from_numpy(vals).cuda()
        vcol = vb.rdd._Col(tv, role="value")
        if where == "device":
            col.loc = vcol.loc = L.VB_DEVICE
    starts = vb.slice_starts(n, M)
    for m in range(M):
        sh.map(m, col, None if op == "count" else vcol, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    got = gpu_parts(sh, op)
    check_parts(got, ref_parts(keys, vals, op, "i64", M, R), op, "i64")
    # device output == host output
    for r in range(R):
        nk, nb, nv = sh.reduce_size(r)
        ko = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
        kb = torch.empty(max(nb, 1), dtype=torch.uint8, device="cuda")
        comb = torch.empty(max(nk, 1), dtype=torch.int64, device="cuda")
        offs = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
        vv = torch.empty(max(nv, 1), dtype=torch.int64, device="cuda")
        if op == "group":
            sh.reduce_device(r, out_key_offsets=ko, out_key_bytes=kb, out_offs=offs, out_vals=vv)
        else:
            sh.reduce_device(r, out_key_offsets=ko, out_key_bytes=kb, out_comb=comb)
        h = sh.reduce_raw(r)
        assert ko.cpu().numpy().view(np.uint64).tolist() == h[0].tolist()
        assert kb.cpu().numpy()[:nb].tobytes() == h[1].tobytes()
        if op == "group":
            assert offs.cpu().numpy().view(np.uint64).tolist() == h[2].tolist()
            assert vv.cpu().numpy()[:nv].tolist() == h[3].tolist()
        else:
            assert comb.cpu().numpy()[:nk].view(np.uint64).tolist() == h[2].view(np.uint64).tolist()
    sh.free()


# ---- dictionary growth and forced fingerprint collisions -------------------------------------------------------------
def test_index_growth_million_keys(sc):
    n = 1_000_000
    keys = [f"key-{i * 7919 % n}" for i in range(n)] + [f"key-{i}" for i in range(0, n, 3)]
    s = sc.parallelize(keys, 4).count_by_value()
    s.hint = 1
    sh = s._run()
    st = sh.stats()
    assert st["table_restarts"] > 0, st
    k, c = s.collect()
    assert len(k) == n
    got = dict(zip(k.tolist(), c.tolist()))
    assert sum(got.values()) == len(keys)
    for i in range(0, n, 997):
        assert got[f"key-{i}"] == (2 if i % 3 == 0 else 1)
    for r in (0, 3):
        for kk in sh.reduce(r)[0][:200].tolist():
            assert O.metrohash64_1(kk.encode() + b"\xff", 0) % sh.n_reduce == r


def _fp_cases(sc):
    rng = np.random.default_rng(11)
    pool = key_pool(rng, n_random=2000)
    keys = rows_from_pool(rng, pool, 20000)
    for op, vdt, mode in [("sum", "u64", "full"), ("max", "f64", "special"), ("count", "u64", "default"), ("group", "i64", "full")]:
        _, vals = rand_pairs(rng, len(keys), 100, vdtype=vdt, values=mode)
        run_case(sc, keys, vals, op, vdt, 4, 13)
        run_case(sc, keys, vals, op, vdt, 4, 13, hint=1)


def test_forced_fingerprint_collisions():
    """VEGA_B200_STR_FP_BITS=4 keeps 4 bits of the hash in the index: distinct keys share fingerprints all the time and
    must be told apart by their bytes.  The switch is read once per process: a subprocess."""
    code = r'''
import vega_b200 as vb
from tests.test_gpu_str_keys import _fp_cases
with vb.Context(0) as sc:
    _fp_cases(sc)
print("fp ok")
'''
    env = dict(os.environ, VEGA_B200_STR_FP_BITS="4")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert out.returncode == 0 and "fp ok" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


# ---- resubmission, map order, concurrency, empty inputs ---------------------------------------------------------
def _map(sh, m, keys, vals):
    col = vb.rdd._StrCol(keys)
    vcol = vb.rdd._Col(np.asarray(vals, dtype=np.uint64), role="value") if vals is not None else None
    sh.map(m, col, vcol, 0, len(keys))


@pytest.mark.parametrize("agg", [L.VB_AGG_SUM, L.VB_AGG_GROUP])
def test_resubmitted_map_drops_its_stale_keys(sc, agg):
    sh = vb.StrShuffle(sc, 2, 3, L.VB_U64, agg)
    _map(sh, 0, ["stale-a", "stale-b", "shared"], [1, 2, 3])
    _map(sh, 1, ["other", "shared"], [10, 20])
    _map(sh, 0, ["fresh", "shared", "fresh"], [100, 200, 300])        # replaces map 0
    sh.seal()
    got = {}
    for d in gpu_parts(sh, "group" if agg == L.VB_AGG_GROUP else "sum"):
        got.update(d)
    if agg == L.VB_AGG_GROUP:
        assert got == {"fresh": [100, 300], "shared": [200, 20], "other": [10]}
    else:
        assert got == {"fresh": 400, "shared": 220, "other": 10}
    assert sh.stats()["rows_in"] == 5


def test_maps_submitted_out_of_order_group_in_map_order(sc):
    sh = vb.StrShuffle(sc, 4, 2, L.VB_U64, L.VB_AGG_GROUP)
    for m in (3, 1, 0, 2):
        _map(sh, m, ["k", "j", "k"], [10 * m, 10 * m + 1, 10 * m + 2])
    sh.seal()
    got = {}
    for d in gpu_parts(sh, "group"):
        got.update(d)
    assert got == {"k": [0, 2, 10, 12, 20, 22, 30, 32], "j": [1, 11, 21, 31]}


def test_eight_threads_map_concurrently(sc):
    rng = np.random.default_rng(8)
    pool = key_pool(rng, n_random=3000)
    M, R = 8, 17
    per = [rows_from_pool(rng, pool, 20000) for _ in range(M)]
    vals = [rng.integers(0, 1 << 63, 20000, dtype=np.uint64) for _ in range(M)]
    for agg, op in [(L.VB_AGG_SUM, "sum"), (L.VB_AGG_GROUP, "group")]:
        sh = vb.StrShuffle(sc, M, R, L.VB_U64, agg)
        errs = []

        def work(m):
            try:
                _map(sh, m, per[m], vals[m])
            except Exception as e:         # pragma: no cover - reported below
                errs.append(e)
        ts = [threading.Thread(target=work, args=(m,)) for m in range(M)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        assert not errs, errs
        sh.seal()
        keys = [k for p in per for k in p]
        allv = np.concatenate(vals)
        got = gpu_parts(sh, op)
        want = [dict() for _ in range(R)]
        fold = _fold("sum", "u64")
        for k, v in zip(keys, allv.tolist()):
            d = want[pyref.get_partition(k, R)]
            if op == "group":
                d.setdefault(k, []).append(v)
            else:
                d[k] = fold(d[k], v) if k in d else v
        check_parts(got, want, op, "u64")
        sh.free()


def test_empty_maps_and_empty_shuffle(sc):
    sh = vb.StrShuffle(sc, 3, 4, L.VB_U64, L.VB_AGG_SUM)
    _map(sh, 0, [], [])
    _map(sh, 1, ["a", "b", "a"], [1, 2, 3])
    _map(sh, 2, [], [])
    sh.seal()
    got = {}
    for d in gpu_parts(sh, "sum"):
        got.update(d)
    assert got == {"a": 4, "b": 2}
    for agg in (L.VB_AGG_SUM, L.VB_AGG_GROUP, L.VB_AGG_COUNT):
        e = vb.StrShuffle(sc, 2, 3, L.VB_U64, agg)
        _map(e, 0, [], [])
        _map(e, 1, [], [])
        e.seal()
        for r in range(3):
            assert e.reduce_size(r) == (0, 0, 0)
            p = e.reduce_raw(r)
            assert p[0].tolist() == [0] and len(p[1]) == 0
    z = vb.StrShuffle(sc, 0, 2, L.VB_U64, L.VB_AGG_GROUP)
    z.seal()
    assert z.reduce_size(1) == (0, 0, 0)


# ---- rejected calls -----------------------------------------------------------------------------------------------------
def test_rejected_calls(sc):
    lib = sc._lib
    sh = vb.StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_GROUP)
    ish = vb.Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_GROUP)
    u = ctypes.c_uint64()
    keys = np.array([1, 2], dtype=np.uint64)
    p = keys.ctypes.data_as(ctypes.c_void_p)
    inv, uns = L.VB_ERR_INVALID, L.VB_ERR_UNSUPPORTED
    h = sh._h
    assert lib.vb_shuffle_set_key_width(h, 4) == inv
    assert lib.vb_shuffle_map_soa(h, 0, p, p, 2, L.VB_HOST) == inv
    assert lib.vb_shuffle_map_aos(h, 0, p, 1, L.VB_HOST) == inv
    assert lib.vb_shuffle_map_cols(h, 0, p, None, 0, L.VB_HOST) == inv
    assert lib.vb_shuffle_set_dist(h, 0, 2) == uns
    assert lib.vb_shuffle_set_dist(h, 0, 1) == 0
    assert lib.vb_shuffle_export_prepare(h, ctypes.byref(u)) == uns
    assert lib.vb_shuffle_export_counts(h, ctypes.byref(u)) == uns
    assert lib.vb_shuffle_exchange(h, 0) == uns
    assert lib.vb_shuffle_import(h, None, None, ctypes.byref(u)) == uns
    assert lib.vb_shuffle_map_blob(h, 0, p, 16, L.VB_HOST) == uns
    assert lib.vb_shuffle_reduce_blob_size(h, 0, ctypes.byref(u)) == uns
    # malformed offsets, on the host and on the device
    data = np.frombuffer(b"abcdef", dtype=np.uint8)
    dp = data.ctypes.data_as(ctypes.c_void_p)
    vals = np.zeros(3, dtype=np.uint64)
    vp = vals.ctypes.data_as(ctypes.c_void_p)
    for offs, nb, code in [([0, 3, 2, 6], 6, inv), ([0, 3, 7], 6, inv), ([9, 9], 6, inv), ([0, 1 << 32], 1 << 33, L.VB_ERR_TOO_LARGE)]:
        o = np.array(offs, dtype=np.uint64)
        assert lib.vb_shuffle_map_str(h, 0, o.ctypes.data_as(ctypes.c_void_p), dp, nb, vp, len(offs) - 1, L.VB_HOST) == code, offs
        import torch
        od = torch.from_numpy(o.view(np.int64)).cuda()
        dd = torch.from_numpy(data.copy()).cuda()
        vd = torch.zeros(3, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        assert lib.vb_shuffle_map_str(h, 0, ctypes.c_void_p(od.data_ptr()), ctypes.c_void_p(dd.data_ptr()), nb,
                                      ctypes.c_void_p(vd.data_ptr()), len(offs) - 1, L.VB_DEVICE) == code, offs
    assert lib.vb_shuffle_map_str(h, 5, None, None, 0, None, 0, L.VB_HOST) == inv                    # map id
    assert lib.vb_shuffle_map_str(h, 0, np.array([0, 1], dtype=np.uint64).ctypes.data_as(ctypes.c_void_p), dp, 6,
                                  None, 1, L.VB_HOST) == inv                                          # GROUP needs values
    # string calls on an integer shuffle, integer calls on a string shuffle after seal
    assert lib.vb_shuffle_map_str(ish._h, 0, None, None, 0, None, 0, L.VB_HOST) == inv
    assert lib.vb_shuffle_reduce_str_size(ish._h, 0, None, None, None) == inv
    assert lib.vb_shuffle_reduce_str(ish._h, 0, None, None, None, None, None, L.VB_HOST) == inv
    _map(sh, 0, ["a", "b"], [1, 2])
    sh.seal()
    ish.map(0, vb.rdd._Col(keys), vb.rdd._Col(keys, role="value"), 0, 2)
    ish.seal()
    assert lib.vb_shuffle_reduce_size(h, 0, ctypes.byref(u), ctypes.byref(u)) == inv
    assert lib.vb_shuffle_reduce(h, 0, None, None, None, None, L.VB_HOST) == inv
    assert lib.vb_join_size(h, h, 0, ctypes.byref(u)) == inv
    assert lib.vb_join_size(ish._h, h, 0, ctypes.byref(u)) == inv
    assert lib.vb_join_outer_size(h, ish._h, 0, L.VB_JOIN_FULL, ctypes.byref(u)) == inv
    assert lib.vb_cogroup_size(h, h, 0, None, None, None) == inv
    assert lib.vb_shuffle_reduce_str_size(h, 2, None, None, None) == inv                            # reduce id
    # unsupported aggregators
    for agg in (L.VB_AGG_COGROUP, L.VB_AGG_SORT, L.VB_AGG_MEAN, 99):
        out = ctypes.c_void_p()
        assert lib.vb_shuffle_create_str(sc._h, 0, 1, 1, L.VB_U64, agg, ctypes.byref(out)) == uns
    # the shuffle still works after the rejected calls
    got = {}
    for d in gpu_parts(sh, "group"):
        got.update(d)
    assert got == {"a": [1], "b": [2]}


# ---- one large property test -----------------------------------------------------------------------------------------
def _device_words(ranks):
    """Word-like keys built on the device from u64 ranks: 'w' + the rank's hex digits (2 to 17 bytes)."""
    import torch
    r = ranks
    nd = torch.ones_like(r)
    for s in range(4, 64, 4):
        nd += (r >> s) > 0
    lens = nd + 1
    offs = torch.zeros(len(r) + 1, dtype=torch.int64, device=r.device)
    offs[1:] = torch.cumsum(lens, 0)
    total = int(offs[-1])
    row = torch.repeat_interleave(torch.arange(len(r), device=r.device), lens)
    j = torch.arange(total, device=r.device) - offs[:-1][row]
    shift = 4 * (nd[row] - j).clamp(min=0)
    digit = (r[row] >> shift.clamp(max=63)) & 15
    hexc = torch.tensor(list(b"0123456789abcdef"), dtype=torch.uint8, device=r.device)
    data = torch.where(j == 0, torch.full_like(digit, ord("w")), hexc[digit].to(torch.int64)).to(torch.uint8)
    return vb.StrKeys(offs, data)


def test_property_twenty_million_rows(sc):
    import torch
    n, D = 20_000_000, 1_000_000
    ranks = torch.empty(n, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=ranks, n=n, mode="zipf", n_distinct=D, zipf_s=1.1)
    ranks = ranks & ((1 << 40) - 1)
    keys = _device_words(ranks)
    torch.cuda.synchronize()
    s = sc.parallelize(keys, 8).count_by_value()
    k, c = s.collect()
    uniq, counts = torch.unique(ranks, return_counts=True)
    assert len(k) == len(uniq)
    assert int(c.sum()) == n
    got = dict(zip(k.tolist(), c.tolist()))
    rng = np.random.default_rng(0)
    for i in rng.choice(len(uniq), 200, replace=False).tolist() + [0, len(uniq) - 1]:
        word = "w" + format(int(uniq[i]), "x")
        assert got[word] == int(counts[i]), word
