"""Cogroup and join of String-key shuffles on the device (vb_cogroup_n_str / vb_join_n_str and StrCoGroupedRdd).
Every partition is checked against the Python references: each key once, in pyref.get_partition's partition, every
side's list equal to that side's group_by_key list bit for bit, and each join key's rows in nested order with their
validity.  Offsets start at 0, never decrease and end at the value / row count."""
import ctypes
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import vega_b200 as vb
from vega_b200 import _lib as L
from oracle import pyref
from tests.test_gpu_str_keys import _device_words

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
_NP = {L.VB_U64: np.uint64, L.VB_I64: np.int64, L.VB_F64: np.float64}


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


# ---- helpers --------------------------------------------------------------------------------------------------------
def side(sc, keys, vals, M, R):
    """A sealed string GROUP shuffle of (keys, vals) over M map slices and R partitions."""
    keys = vb.StrKeys.from_strs(keys) if len(keys) == 0 else keys
    return sc.parallelize(keys, M, values=vals).group_by_key(R)._run()


def _arr(shs):
    return (ctypes.c_void_p * len(shs))(*[s._h.value for s in shs])


def _out(n, dtype, dev):
    import torch
    if dev:
        return torch.empty(n, dtype={np.uint8: torch.uint8}.get(dtype, torch.int64), device="cuda")
    return np.empty(n, dtype=dtype)


def _ptr(x):
    if x is None:
        return None
    return ctypes.c_void_p(x.data_ptr() if hasattr(x, "data_ptr") else x.ctypes.data)


def _host(x, dtype):
    if x is None:
        return None
    if hasattr(x, "data_ptr"):
        return x.cpu().numpy().view(dtype)
    return x.view(dtype)


def _keys(ko, kb):
    return [bytes(kb[int(ko[i]):int(ko[i + 1])]).decode("utf-8", "surrogateescape") for i in range(len(ko) - 1)]


def cogroup_part(sc, shs, r, dev=False):
    """(keys, [(offsets, values as u64) per side]) of partition r through vb_cogroup_n_str."""
    n, lib = len(shs), sc._lib
    nk, nb, nv = ctypes.c_uint64(), ctypes.c_uint64(), (ctypes.c_uint64 * n)()
    L.check(lib.vb_cogroup_n_str_size(_arr(shs), n, r, ctypes.byref(nk), ctypes.byref(nb), nv))
    ko, kb = _out(nk.value + 1, np.uint64, dev), _out(nb.value, np.uint8, dev)
    offs = [_out(nk.value + 1, np.uint64, dev) for _ in shs]
    vals = [_out(nv[j], np.uint64, dev) for j in range(n)]
    L.check(lib.vb_cogroup_n_str(_arr(shs), n, r, _ptr(ko), _ptr(kb), (ctypes.c_void_p * n)(*[_ptr(o) for o in offs]),
                                 (ctypes.c_void_p * n)(*[_ptr(v) for v in vals]), L.VB_DEVICE if dev else L.VB_HOST))
    ko, kb = _host(ko, np.uint64), _host(kb, np.uint8)
    return _keys(ko, kb), [(_host(o, np.uint64), _host(v, np.uint64)) for o, v in zip(offs, vals)], ko


def join_part(sc, shs, r, mask, dev=False, valid=True):
    """(keys, row offsets, [values as u64], [validity or None]) of partition r through vb_join_n_str."""
    n, lib = len(shs), sc._lib
    nr, nk, nb = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    L.check(lib.vb_join_n_str_size(_arr(shs), n, r, mask, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)))
    ko, kb, ro = _out(nk.value + 1, np.uint64, dev), _out(nb.value, np.uint8, dev), _out(nk.value + 1, np.uint64, dev)
    vs = [_out(nr.value, np.uint64, dev) for _ in shs]
    ok = [_out(nr.value, np.uint8, dev) for _ in shs] if valid else None
    L.check(lib.vb_join_n_str(_arr(shs), n, r, mask, _ptr(ko), _ptr(kb), _ptr(ro), (ctypes.c_void_p * n)(*[_ptr(v) for v in vs]),
                              (ctypes.c_void_p * n)(*[_ptr(v) for v in ok]) if valid else None, L.VB_DEVICE if dev else L.VB_HOST))
    ko, kb, ro = _host(ko, np.uint64), _host(kb, np.uint8), _host(ro, np.uint64)
    return (_keys(ko, kb), ro, [_host(v, np.uint64) for v in vs], [_host(v, np.uint8) for v in ok] if valid else None, ko, nr.value)


def u64(vals):
    return np.asarray(vals).view(np.uint64) if np.asarray(vals).dtype.itemsize == 8 else np.asarray(vals, dtype=np.uint64)


def ref_lists(data):
    """[(keys, vals), ...] -> per side {key: [u64 bits in input order]} (group_by_key's list of a contiguous slicing)"""
    out = []
    for keys, vals in data:
        d = {}
        for k, v in zip(keys, u64(vals).tolist()):
            d.setdefault(k, []).append(v)
        out.append(d)
    return out


def check_offsets(o, total):
    o = np.asarray(o).astype(np.int64)
    assert o[0] == 0 and (np.diff(o) >= 0).all() and o[-1] == total, (o[:5], o[-5:], total)


def check_cogroup(sc, shs, data, R, dev=False):
    want = ref_lists(data)
    part = {}
    for w in want:
        for k in w:
            part.setdefault(k, pyref.get_partition(k, R))
    seen = 0
    for r in range(R):
        keys, lists, ko = cogroup_part(sc, shs, r, dev)
        check_offsets(ko, int(ko[-1]))
        assert len(set(keys)) == len(keys), f"a key twice in partition {r}"
        assert set(keys) == {k for k, p in part.items() if p == r}, r
        seen += len(keys)
        for j, (o, v) in enumerate(lists):
            check_offsets(o, len(v))
            for i, k in enumerate(keys):
                assert v[int(o[i]):int(o[i + 1])].tolist() == want[j].get(k, []), (r, j, k)
    assert seen == len(part)


def ref_join(want, required):
    """{key: [row tuples (v_0.., valid_0..)]} of the keys the mask keeps"""
    out = {}
    keys = set().union(*want)
    for k in keys:
        lists = [w.get(k, []) for w in want]
        if not all(lists[j] for j in range(len(lists)) if required >> j & 1):
            continue
        rows = [()]
        for l in lists:
            slots = [(v, 1) for v in l] if l else [(0, 0)]
            rows = [r + (s,) for r in rows for s in slots]
        out[k] = [tuple(v for v, _ in row) + tuple(o for _, o in row) for row in rows]
    return out


def check_join(sc, shs, data, R, required, dev=False, valid=True):
    want = ref_join(ref_lists(data), required)
    seen = 0
    for r in range(R):
        keys, ro, vs, ok, ko, nrows = join_part(sc, shs, r, required, dev, valid)
        check_offsets(ko, int(ko[-1]))
        check_offsets(ro, nrows)
        assert len(set(keys)) == len(keys), f"a key twice in partition {r}"
        assert set(keys) == {k for k in want if pyref.get_partition(k, R) == r}, (r, required)
        assert (np.diff(ro.astype(np.int64)) > 0).all(), "a listed key without rows"
        for i, k in enumerate(keys):
            a, b = int(ro[i]), int(ro[i + 1])
            got = [tuple(int(v[x]) for v in vs) for x in range(a, b)]
            assert got == [w[:len(vs)] for w in want[k]], (r, k, required)
            if valid:
                assert [tuple(int(o[x]) for o in ok) for x in range(a, b)] == [w[len(vs):] for w in want[k]], (r, k)
        seen += len(keys)
    assert seen == len(want)


def words(rng, n, pool):
    return [pool[i] for i in rng.integers(0, len(pool), n)]


POOL = ["", "a", "ab", "abc", "b", "x", "y", "\x00", "a\x00", "\x00a", "é", "日本語", "naïve", "🙂"] + \
       [f"word{i}" for i in range(80)]


# ---- n = 1, 2, 3 ------------------------------------------------------------------------------------------------------
def test_one_side_is_reduce_str(sc):
    rng = np.random.default_rng(1)
    keys = words(rng, 3000, POOL)
    vals = rng.integers(0, 1 << 64, len(keys), dtype=np.uint64)
    a = side(sc, keys, vals, 3, 5)
    for r in range(5):
        ko, kb, offs, v = a.reduce_raw(r)
        keys_g, lists, _ = cogroup_part(sc, [a], r)
        want = {k: v[int(offs[i]):int(offs[i + 1])].tolist() for i, k in enumerate(_keys(ko, kb))}
        got = {k: lists[0][1][int(lists[0][0][i]):int(lists[0][0][i + 1])].tolist() for i, k in enumerate(keys_g)}
        assert got == want
    check_join(sc, [a], [(keys, vals)], 5, 1)
    check_join(sc, [a], [(keys, vals)], 5, 0)


@pytest.mark.parametrize("n", [2, 3])
def test_sides_every_mask(sc, n):
    rng = np.random.default_rng(10 + n)
    R = 6
    data = []
    for j in range(n):
        pool = POOL[: 40 + 20 * j] + [f"only{j}-{i}" for i in range(10)]
        keys = words(rng, int(rng.integers(200, 700)), pool)
        data.append((keys, rng.integers(0, 1 << 64, len(keys), dtype=np.uint64)))
    shs = [side(sc, k, v, int(rng.integers(1, 5)), R) for k, v in data]
    check_cogroup(sc, shs, data, R)
    for mask in range(1 << n):
        check_join(sc, shs, data, R, mask)


def test_sixteen_sides_and_seventeen_refused(sc):
    rng = np.random.default_rng(16)
    data = [(words(rng, 40, POOL[:30]), rng.integers(0, 1000, 40, dtype=np.uint64)) for _ in range(16)]
    shs = [side(sc, k, v, 2, 3) for k, v in data]
    check_cogroup(sc, shs, data, 3)
    check_join(sc, shs[:4], data[:4], 3, 0b1111)
    check_join(sc, shs, data, 3, 1)
    u = ctypes.c_uint64()
    seventeen = shs + shs[:1]
    assert sc._lib.vb_cogroup_n_str_size(_arr(seventeen), 17, 0, None, None, None) == L.VB_ERR_INVALID
    assert sc._lib.vb_join_n_str_size(_arr(seventeen), 17, 0, 0, ctypes.byref(u), None, None) == L.VB_ERR_INVALID


# ---- key shapes -------------------------------------------------------------------------------------------------------
def test_key_shapes(sc):
    base = [("k" * L_) for L_ in list(range(0, 18)) + [31, 32, 33, 63, 64, 65]]
    long_ = ["z" * 10_000, "z" * 9_999 + "y", "z" * 10_001]
    prefixes = ["ab", "abc", "abcd", "a", "abd"]
    last = ["same-prefix-%c" % c for c in "abcdefgh"] + ["x" * 63 + c for c in "pq"] + ["x" * 32 + c for c in "pq"]
    odd = ["\x00", "\x00\x00", "a\x00b", "a\x00c", "é", "é", "日本", "日本語", "🙂", "￿"]
    all_keys = base + long_ + prefixes + last + odd
    rng = np.random.default_rng(3)
    a_keys = [k for k in all_keys for _ in range(2)]
    b_keys = [k for i, k in enumerate(all_keys) if i % 3 != 1] + ["b-only", "abcde"]
    c_keys = [k for i, k in enumerate(all_keys) if i % 2 == 0]
    data = [(a_keys, rng.integers(0, 1 << 64, len(a_keys), dtype=np.uint64)),
            (b_keys, rng.integers(0, 1 << 64, len(b_keys), dtype=np.uint64)),
            (c_keys, rng.integers(0, 1 << 64, len(c_keys), dtype=np.uint64))]
    for R in (1, 4):
        shs = [side(sc, k, v, 3, R) for k, v in data]
        check_cogroup(sc, shs, data, R)
        check_cogroup(sc, shs, data, R, dev=True)
        for mask in (0, 0b111, 0b010, 0b101):
            check_join(sc, shs, data, R, mask)


# ---- empty, disjoint, identical, repeated sides -------------------------------------------------------------------------
def test_empty_disjoint_identical_and_repeated_sides(sc):
    rng = np.random.default_rng(4)
    R = 5
    a_keys = words(rng, 500, POOL)
    a = (a_keys, rng.integers(0, 1 << 64, 500, dtype=np.uint64))
    d_keys = [f"disjoint-{i % 37}" for i in range(300)]
    d = (d_keys, rng.integers(0, 1 << 64, 300, dtype=np.uint64))
    e = ([], np.zeros(0, dtype=np.uint64))
    sa, sd, se = side(sc, *a, 2, R), side(sc, *d, 3, R), side(sc, *e, 2, R)
    sa2 = side(sc, *a, 4, R)                        # identical rows, another slicing
    for shs, dat in [([sa, sd], [a, d]), ([se], [e]), ([se, sa], [e, a]), ([sa, se, sd], [a, e, d]), ([sa, sa2], [a, a]),
                     ([sa, sd, sa], [a, d, a]), ([se, se], [e, e])]:
        check_cogroup(sc, shs, dat, R)
        for mask in range(1 << len(shs)):
            check_join(sc, shs, dat, R, mask)


# ---- value dtypes and partition counts ---------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 7, 300])
def test_mixed_dtypes_and_partition_counts(sc, R):
    rng = np.random.default_rng(R)
    ka, kb_, kc = words(rng, 2000, POOL), words(rng, 1500, POOL[5:]), words(rng, 1000, POOL[:50])
    fa = rng.standard_normal(len(kc))
    fa[:4] = [np.nan, -0.0, np.inf, -np.inf]
    data = [(ka, rng.integers(0, 1 << 64, len(ka), dtype=np.uint64)),
            (kb_, rng.integers(-(1 << 63), (1 << 63) - 1, len(kb_), dtype=np.int64)),
            (kc, fa)]
    shs = [side(sc, k, v, 3, R) for k, v in data]
    assert [s.vcode for s in shs] == [L.VB_U64, L.VB_I64, L.VB_F64]
    check_cogroup(sc, shs, data, R)
    for mask in (0, 0b111, 0b001, 0b110):
        check_join(sc, shs, data, R, mask)


# ---- a hot key --------------------------------------------------------------------------------------------------------
def test_million_values_on_a_middle_side(sc):
    n = 1_000_000
    rng = np.random.default_rng(5)
    mid_keys = ["hot"] * n + ["cold", "warm"]
    mid_vals = rng.integers(0, 1 << 64, len(mid_keys), dtype=np.uint64)
    a = (["hot", "cold", "hot"], np.array([1, 2, 3], dtype=np.uint64))
    c = (["hot", "warm"], np.array([7, 8], dtype=np.uint64))
    R = 3
    shs = [side(sc, *a, 1, R), side(sc, mid_keys, mid_vals, 4, R), side(sc, *c, 1, R)]
    r = pyref.get_partition("hot", R)
    keys, lists, _ = cogroup_part(sc, shs, r)
    i = keys.index("hot")
    o, v = lists[1]
    assert np.array_equal(v[int(o[i]):int(o[i + 1])], mid_vals[:n])
    for dev in (False, True):
        keys, ro, vs, ok, _, nrows = join_part(sc, shs, r, 0b111, dev)
        i = keys.index("hot")
        a_, b_ = int(ro[i]), int(ro[i + 1])
        assert b_ - a_ == 2 * n
        assert np.array_equal(vs[0][a_:b_], np.repeat(np.array([1, 3], dtype=np.uint64), n))
        assert np.array_equal(vs[1][a_:b_], np.tile(mid_vals[:n], 2))
        assert (vs[2][a_:b_] == 7).all() and all((x[a_:b_] == 1).all() for x in ok)


# ---- output locations and NULL outputs -----------------------------------------------------------------------------------
def test_device_and_host_outputs_and_null_outputs(sc):
    rng = np.random.default_rng(6)
    data = [(words(rng, 800, POOL), rng.integers(0, 1 << 64, 800, dtype=np.uint64)) for _ in range(3)]
    R = 4
    shs = [side(sc, k, v, 2, R) for k, v in data]
    for r in range(R):
        h, d = cogroup_part(sc, shs, r), cogroup_part(sc, shs, r, dev=True)
        assert h[0] == d[0] and all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(h[1], d[1]))
        for mask in (0, 0b101):
            h, d = join_part(sc, shs, r, mask), join_part(sc, shs, r, mask, dev=True)
            assert h[0] == d[0] and np.array_equal(h[1], d[1])
            assert all(np.array_equal(x, y) for x, y in zip(h[2] + h[3], d[2] + d[3]))
    check_join(sc, shs, data, R, 0b011, valid=False)              # out_valid NULL
    lib, n = sc._lib, 3
    nk, nb, nv = ctypes.c_uint64(), ctypes.c_uint64(), (ctypes.c_uint64 * n)()
    for r in range(R):                                            # cogroup: every output may be NULL
        keys, lists, _ = cogroup_part(sc, shs, r)
        L.check(lib.vb_cogroup_n_str_size(_arr(shs), n, r, ctypes.byref(nk), ctypes.byref(nb), nv))
        o1 = np.empty(nk.value + 1, dtype=np.uint64)
        L.check(lib.vb_cogroup_n_str(_arr(shs), n, r, None, None, (ctypes.c_void_p * n)(None, _ptr(o1), None), None, L.VB_HOST))
        assert np.array_equal(o1, lists[1][0])
        L.check(lib.vb_cogroup_n_str(_arr(shs), n, r, None, None, None, None, L.VB_HOST))
    # join: NULL values, keys or row offsets once the partition has rows are refused
    nr = ctypes.c_uint64()
    r = next(r for r in range(R) if lib.vb_join_n_str_size(_arr(shs), n, r, 0, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)) == 0
             and nr.value)
    ko, kb, ro = np.empty(nk.value + 1, np.uint64), np.empty(nb.value, np.uint8), np.empty(nk.value + 1, np.uint64)
    vs = [np.empty(nr.value, np.uint64) for _ in range(n)]
    vp = (ctypes.c_void_p * n)(*[_ptr(v) for v in vs])
    for args in [(None, _ptr(kb), _ptr(ro), vp), (_ptr(ko), None, _ptr(ro), vp), (_ptr(ko), _ptr(kb), None, vp),
                 (_ptr(ko), _ptr(kb), _ptr(ro), None), (_ptr(ko), _ptr(kb), _ptr(ro), (ctypes.c_void_p * n)(vp[0], None, vp[2]))]:
        assert lib.vb_join_n_str(_arr(shs), n, r, 0, *args, None, L.VB_HOST) == L.VB_ERR_INVALID
    check_join(sc, shs, data, R, 0)


# ---- fingerprint collisions --------------------------------------------------------------------------------------------
def _fp_join_cases(sc):
    rng = np.random.default_rng(7)
    pool = [f"k{i}" for i in range(3000)] + POOL
    data = [(words(rng, 6000, pool), rng.integers(0, 1 << 64, 6000, dtype=np.uint64)) for _ in range(3)]
    shs = [side(sc, k, v, 3, 5) for k, v in data]
    check_cogroup(sc, shs, data, 5)
    for mask in (0, 0b111, 0b010):
        check_join(sc, shs, data, 5, mask)


def test_forced_fingerprint_collisions():
    """VEGA_B200_STR_FP_BITS=4 keeps 4 bits of the hash in every fingerprint, so distinct keys share fingerprints all
    the time and the probe must tell them apart by their bytes.  The switch is read once per process: a subprocess."""
    code = r'''
import vega_b200 as vb
from tests.test_gpu_str_join import _fp_join_cases
with vb.Context(0) as sc:
    _fp_join_cases(sc)
print("fp ok")
'''
    env = dict(os.environ, VEGA_B200_STR_FP_BITS="4")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert out.returncode == 0 and "fp ok" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


# ---- limits, rejected arguments, blocking, the lazy index ---------------------------------------------------------------------
def test_two_to_the_63_rows_refused(sc):
    lib = sc._lib
    big = side(sc, ["k"] * 16, np.arange(16, dtype=np.uint64), 1, 1)          # 16 values
    four = side(sc, ["k", "k", "k", "k", "j"], np.arange(5, dtype=np.uint64), 1, 1)
    eight = side(sc, ["k"] * 8, np.arange(8, dtype=np.uint64), 1, 1)
    nr = ctypes.c_uint64()
    L.check(lib.vb_join_n_str_size(_arr([big] * 15), 15, 0, (1 << 15) - 1, ctypes.byref(nr), None, None))
    assert nr.value == 1 << 60
    assert lib.vb_join_n_str_size(_arr([big] * 15 + [eight]), 16, 0, 0, ctypes.byref(nr), None, None) == L.VB_ERR_TOO_LARGE
    # "k" gives 2^62 rows and "j" 2^60, then both 2^62: a partition total of 2^63
    jside = side(sc, ["j"] * 4 + ["k"] * 4, np.arange(8, dtype=np.uint64), 1, 1)
    big_j = side(sc, ["k"] * 16 + ["j"] * 16, np.arange(32, dtype=np.uint64), 1, 1)
    L.check(lib.vb_join_n_str_size(_arr([big_j] * 15 + [four]), 16, 0, 0, ctypes.byref(nr), None, None))
    assert nr.value == (1 << 62) + (1 << 60)
    assert lib.vb_join_n_str_size(_arr([big_j] * 15 + [jside]), 16, 0, 0, ctypes.byref(nr), None, None) == L.VB_ERR_TOO_LARGE


def test_rejected_arguments_leave_the_sides_usable(sc):
    lib = sc._lib
    rng = np.random.default_rng(8)
    data = [(words(rng, 300, POOL), rng.integers(0, 100, 300, dtype=np.uint64)) for _ in range(2)]
    shs = [side(sc, k, v, 2, 3) for k, v in data]
    other_r = side(sc, ["a"], np.zeros(1, dtype=np.uint64), 1, 4)
    red = sc.parallelize(["a", "b"], 1, values=np.ones(2, dtype=np.uint64)).reduce_by_key("sum", 3)._run()
    ish = sc.parallelize((np.arange(4, dtype=np.uint64), np.arange(4, dtype=np.uint64)), 1).group_by_key(3)._run()
    u = ctypes.c_uint64()
    inv = L.VB_ERR_INVALID
    a, b = shs
    cases = [(None, 2, 0), (_arr([a, b]), 0, 0), (_arr([a, b]), 17, 0), ((ctypes.c_void_p * 2)(a._h.value, None), 2, 0),
             (_arr([a, ish]), 2, 0), (_arr([a, red]), 2, 0), (_arr([a, other_r]), 2, 0), (_arr([a, b]), 2, 3)]
    with vb.Context(0) as sc2:
        cases.append((_arr([a, side(sc2, ["a"], np.zeros(1, dtype=np.uint64), 1, 3)]), 2, 0))
        for sides, n, r in cases:
            assert lib.vb_cogroup_n_str_size(sides, n, r, ctypes.byref(u), None, None) == inv
            assert lib.vb_cogroup_n_str(sides, n, r, None, None, None, None, L.VB_HOST) == inv
            assert lib.vb_join_n_str_size(sides, n, r, 0, ctypes.byref(u), None, None) == inv
            assert lib.vb_join_n_str(sides, n, r, 0, None, None, None, None, None, L.VB_HOST) == inv
    assert lib.vb_join_n_str_size(_arr(shs), 2, 0, 0b100, ctypes.byref(u), None, None) == inv      # required bit >= n
    assert lib.vb_join_n_str(_arr(shs), 2, 0, 1 << 31, None, None, None, None, None, L.VB_HOST) == inv
    assert lib.vb_cogroup_n_str(_arr(shs), 2, 0, None, None, None, None, 7) == inv                  # dst_loc
    assert lib.vb_join_n_str(_arr(shs), 2, 0, 0, None, None, None, None, None, 7) == inv
    # the integer entry points still refuse string shuffles
    assert lib.vb_cogroup_n_size(_arr(shs), 2, 0, None, None) == inv
    assert lib.vb_join_n_outer_size(_arr(shs), 2, 0, 0, ctypes.byref(u)) == inv
    check_cogroup(sc, shs, data, 3)
    check_join(sc, shs, data, 3, 0b01)


def test_call_before_seal_blocks_until_sealed(sc):
    a = vb.StrShuffle(sc, 1, 2, L.VB_U64, L.VB_AGG_GROUP)
    b = side(sc, ["x", "y"], np.array([5, 6], dtype=np.uint64), 1, 2)
    a.map(0, vb.rdd._StrCol(["x", "z", "x"]), vb.rdd._Col(np.array([1, 2, 3], dtype=np.uint64), role="value"), 0, 3)
    got = {}

    def work():
        got["keys"] = [cogroup_part(sc, [a, b], r)[0] for r in range(2)]
    t = threading.Thread(target=work)
    t.start()
    time.sleep(0.5)
    assert t.is_alive(), "the cogroup returned before its side was sealed"
    a.seal()
    t.join(120)
    assert not t.is_alive()
    assert sorted(sum(got["keys"], [])) == ["x", "y", "z"]


def _dict_launches(sh):
    n = ctypes.c_uint64()
    L.check(sh._lib.vb_shuffle_kernel_time(sh._h, 1, None, ctypes.byref(n)))
    return n.value


def test_index_built_once_and_only_for_joins(sc):
    rng = np.random.default_rng(9)
    data = [(words(rng, 400, POOL), rng.integers(0, 100, 400, dtype=np.uint64)) for _ in range(2)]
    shs = [side(sc, k, v, 2, 3) for k, v in data]
    sealed = [_dict_launches(s) for s in shs]
    for r in range(3):
        shs[0].reduce_raw(r)                                      # a plain group_by_key read builds no index
    assert [_dict_launches(s) for s in shs] == sealed
    check_join(sc, shs, data, 3, 0b11)
    first = [_dict_launches(s) for s in shs]
    assert first == [x + 1 for x in sealed]                      # one index build per side
    check_join(sc, shs, data, 3, 0b11)
    check_cogroup(sc, shs, data, 3)
    assert [_dict_launches(s) for s in shs] == first


# ---- the mirror -----------------------------------------------------------------------------------------------------
def test_mirror_with_pair_reduce_and_count_parents(sc):
    rng = np.random.default_rng(11)
    ka, kb_, kc = words(rng, 900, POOL), words(rng, 700, POOL[3:]), words(rng, 500, POOL[:60])
    va = rng.integers(0, 1 << 64, len(ka), dtype=np.uint64)
    vb_ = rng.integers(-1000, 1000, len(kb_)).astype(np.int64)
    vc = rng.standard_normal(len(kc))
    pa = sc.parallelize(ka, 3, values=va)
    red = sc.parallelize(kb_, 2, values=vb_).reduce_by_key("min", 5)
    cnt = sc.parallelize(kc, 4, values=vc).count_by_key(3)
    cg = vb.StrCoGroupedRdd([pa, red, cnt], 4)
    mins, counts = {}, {}
    for k, v in zip(kb_, vb_.tolist()):
        mins[k] = min(mins.get(k, v), v)
    for k in kc:
        counts[k] = counts.get(k, 0) + 1
    lists_a = ref_lists([(ka, va)])[0]
    want = {k: [lists_a.get(k, []), [mins[k]] if k in mins else [],
                [counts[k]] if k in counts else []] for k in set(ka) | set(mins) | set(counts)}
    got = cg.collect()
    assert len(got) == len(want)
    for k, ls in got:
        assert [l.tolist() for l in ls] == want[k], k
    k, vs = cg.join_collect()
    rows = sorted(zip(k.tolist(), vs[0].tolist(), vs[1].tolist(), vs[2].tolist()))
    want_rows = sorted((key, a, want[key][1][0], want[key][2][0]) for key in want if all(want[key]) for a in want[key][0])
    assert rows == want_rows
    k, vs = cg.outer_join_collect([1])
    assert isinstance(vs[0], np.ma.MaskedArray) and isinstance(vs[2], np.ma.MaskedArray) and vs[1].dtype == np.int64
    assert sorted(set(k.tolist())) == sorted(mins)
    assert len(k) == sum(max(len(want[key][0]), 1) for key in mins)


# ---- large ----------------------------------------------------------------------------------------------------------
def test_twenty_million_rows_per_side(sc):
    import torch
    n, D = 20_000_000, 1_000_000
    R = 8
    ranks = []
    for j, base in enumerate((0, int(D * 0.98))):                 # 2 % of the keys on both sides
        r = torch.empty(n, dtype=torch.int64, device="cuda")
        sc.gen_pairs(out_keys=r, n=n, mode="uniform", n_distinct=D, seed_k=1 + j * 1_000_000_007)
        ranks.append((r % D) + base)
    vals = [torch.arange(n, dtype=torch.int64, device="cuda") * (j + 3) for j in range(2)]
    torch.cuda.synchronize()
    shs = [sc.parallelize(_device_words(r), 8, values=v).group_by_key(R)._run() for r, v in zip(ranks, vals)]
    ranks = [r.cpu().numpy() for r in ranks]
    vals = [v.cpu().numpy() for v in vals]
    order = [np.argsort(r, kind="stable") for r in ranks]
    ref = [(r[o], v[o]) for r, v, o in zip(ranks, vals, order)]   # (rank, value) triples in list order
    got_k, got_v = [[], []], [[], []]
    for p in range(R):
        keys, lists, ko = cogroup_part(sc, shs, p, dev=True)
        kr = np.array([int(k[1:], 16) for k in keys], dtype=np.int64)
        for j, (o, v) in enumerate(lists):
            check_offsets(o, len(v))
            got_k[j].append(np.repeat(kr, np.diff(o.astype(np.int64))))
            got_v[j].append(v.view(np.int64))
    for j in range(2):
        gk, gv = np.concatenate(got_k[j]), np.concatenate(got_v[j])
        o = np.argsort(gk, kind="stable")
        assert np.array_equal(gk[o], ref[j][0]) and np.array_equal(gv[o], ref[j][1]), j
    # the inner join: per shared key la * lb rows; spot-check 200 keys exactly
    shared = np.intersect1d(ref[0][0], ref[1][0])
    cnt = [dict(zip(*np.unique(r, return_counts=True))) for r in ranks]
    total = 0
    rng = np.random.default_rng(0)
    pick = set(rng.choice(shared, 200, replace=False).tolist())
    for p in range(R):
        keys, ro, vs, _, _, nrows = join_part(sc, shs, p, 0b11, dev=True, valid=False)
        total += nrows
        for i, k in enumerate(keys):
            rk = int(k[1:], 16)
            a, b = int(ro[i]), int(ro[i + 1])
            assert b - a == cnt[0][rk] * cnt[1][rk]
            if rk in pick:
                la, lb = (rv[np.searchsorted(rr, rk):np.searchsorted(rr, rk, side="right")] for rr, rv in ref)
                assert np.array_equal(vs[0][a:b].view(np.int64), np.repeat(la, len(lb)))
                assert np.array_equal(vs[1][a:b].view(np.int64), np.tile(lb, len(la)))
    assert total == sum(cnt[0][k] * cnt[1][k] for k in shared.tolist())


# ---- the C++ example ----------------------------------------------------------------------------------------------------
def test_cpp_example_join_string():
    exe = os.path.join(ROOT, "examples", "_build", "join_string")
    if not os.path.exists(exe):
        pytest.skip("examples not built")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert 'cogroup: [("x", ([1, 2, 3, 4, 5, 6, 7], [10, 11])), ("y", ([1, 2, 3, 4, 5, 6, 7, 8], [30])), ("z", ([], [20]))]' in out.stdout, out.stdout
    assert "join ok" in out.stdout and "left outer join ok" in out.stdout, out.stdout
