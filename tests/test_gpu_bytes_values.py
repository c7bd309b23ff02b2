"""Byte-string values (VB_BYTES) for group_by_key, cogroup, the joins and sort_by_key: the values travel as references
and are gathered back into bytes on the device.

Every check compares against a run of the same keys with the global row index as a u64 value: the index run fixes
which row lands where (checked against tests/group_ref.py), and the bytes run must give values[row] in its place."""
import ctypes
import struct

import numpy as np
import pytest

import vega_b200 as vb
from tests import cogroup_n_ref as CN
from tests import group_ref as G
from tests import join_n_outer_ref as JN
from tests.test_gpu_group_paths import GROUP_CASES, PHI, exact_keys, place, scatter_launches, sliced
from tests.test_oracle_golden import COL1, COL2, JOIN_EXPECTED
from vega_b200 import _lib as L
from vega_b200.rdd import StrCoGroupedRdd, StrKeys, StrSortedRdd

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def bincode_pair(a, b):
    """(String, String) as bincode 1.2.1 encodes it: u64 LE length + bytes, twice."""
    return b"".join(struct.pack("<Q", len(x.encode())) + x.encode() for x in (a, b))


def unbincode_pair(raw):
    n = struct.unpack_from("<Q", raw, 0)[0]
    a = raw[8:8 + n].decode()
    m = struct.unpack_from("<Q", raw, 8 + n)[0]
    return a, raw[16 + n:16 + n + m].decode()


def rand_values(rng, n, big_share=0.01):
    """Mostly 0-64 bytes, about big_share of 1 B-64 KiB, some empty ones, NUL and non-UTF-8 bytes included."""
    lens = rng.integers(0, 65, n)
    big = rng.random(n) < big_share
    lens[big] = rng.integers(1, 65537, int(big.sum()))
    lens[rng.random(n) < 0.05] = 0
    data = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8).tobytes()
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return [data[offs[i]:offs[i + 1]] for i in range(n)]


def grouped_dict(parts):
    """{partition: {key: [values]}} from a list of (keys, offsets, values) partitions."""
    out = {}
    for r, (k, o, v) in enumerate(parts):
        o = o.astype(np.int64)
        out[r] = {int(x): list(v[o[i]:o[i + 1]]) for i, x in enumerate(k.tolist())}
    return out


# -- tests/test_pair_rdd.rs:39-82: col2.join(col1, 4) with its own String and (String, String) values -------------------
def test_join_golden_own_values(sc):
    k2 = np.array([k for k, _ in COL2], dtype=np.int32)
    k1 = np.array([k for k, _ in COL1], dtype=np.int32)
    col2 = sc.parallelize(k2, 4, values=[v for _, v in COL2])
    col1 = sc.parallelize(k1, 4, values=[bincode_pair(*v) for _, v in COL1])
    k, v, w = col2.join(col1, 4).collect()
    got = sorted((int(a), (b, unbincode_pair(c))) for a, b, c in zip(k, v, w))
    assert got == JOIN_EXPECTED
    # the same through vb_join_n at n = 2
    k, (v, w) = vb.CoGroupedRdd([col2, col1], 4).join_collect()
    assert sorted((int(a), (b, unbincode_pair(c))) for a, b, c in zip(k, v, w)) == JOIN_EXPECTED


# -- group_by_key, integer keys ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,R", [(1, 1), (4, 7), (9, 300), (4, 300), (9, 1)])
def test_group_by_key(sc, M, R):
    rng = np.random.default_rng(M * 1000 + R)
    n = 20_000
    keys = rng.integers(0, 3000, n).astype(np.uint64)
    values = rand_values(rng, n)
    values[:3] = [b"", b"\x00\x00", b"\xff\xfe\x80"]
    idx = sc.parallelize(keys, M, values=np.arange(n, dtype=np.uint64)).group_by_key(R)
    idx_sh = idx._run()
    parts_i = [idx_sh.reduce(r) for r in range(R)]
    G.assert_group_equal(parts_i, keys, np.arange(n, dtype=np.uint64), R)
    byt = sc.parallelize(keys, M, values=values).group_by_key(R)
    sh = byt._run()
    parts_b = [sh.reduce(r) for r in range(R)]
    gi, gb = grouped_dict(parts_i), grouped_dict(parts_b)
    assert gb == {r: {k: [values[int(i)] for i in v] for k, v in d.items()} for r, d in gi.items()}


def test_group_by_key_device_in_and_out(sc):
    import torch
    rng = np.random.default_rng(5)
    n, R = 600_000, 7                                    # map tasks of 300 000 rows: more than one thread per row's offset
    keys = rng.integers(0, 500, n).astype(np.int64)
    values = rand_values(rng, n, 0.0005)
    offs = np.concatenate([[0], np.cumsum([len(v) for v in values])]).astype(np.int64)
    data = np.frombuffer(b"".join(values), dtype=np.uint8)
    dk = torch.from_numpy(keys).cuda()
    col = StrKeys(torch.from_numpy(offs).cuda(), torch.from_numpy(data.copy()).cuda())
    sh = sc.parallelize(dk, 2, values=col).group_by_key(R)._run()
    host = sc.parallelize(keys, 2, values=values).group_by_key(R)._run()
    lib = sc._lib
    for r in range(R):
        nk, nv = sh.reduce_size(r)
        ok, oo, ov = (torch.empty(x, dtype=torch.int64, device="cuda") for x in (nk, nk + 1, nv))
        sh.reduce_device(r, out_keys=ok, out_offs=oo, out_vals=ov)
        # references from the device, bytes to the device
        nb = ctypes.c_uint64()
        L.check(lib.vb_shuffle_gather_bytes_size(sh._h, ctypes.c_void_p(ov.data_ptr()), nv, L.VB_DEVICE, ctypes.byref(nb)))
        go = torch.empty(nv + 1, dtype=torch.int64, device="cuda")
        gb = torch.empty(nb.value + 1, dtype=torch.uint8, device="cuda")
        dst = gb[1:]                                      # an output that does not start on a 16-byte boundary
        L.check(lib.vb_shuffle_gather_bytes(sh._h, ctypes.c_void_p(ov.data_ptr()), nv, L.VB_DEVICE, ctypes.c_void_p(go.data_ptr()),
                                            ctypes.c_void_p(dst.data_ptr()), L.VB_DEVICE))
        go, raw = go.cpu().numpy(), dst.cpu().numpy().tobytes()
        dev_vals = [raw[go[i]:go[i + 1]] for i in range(nv)]
        assert dev_vals == [v.encode("utf-8", "surrogateescape") for v in sh.gather(ov.cpu().numpy())]   # refs from the host
        d_dev = {int(k): dev_vals[o0:o1] for k, o0, o1 in zip(ok.cpu().numpy(), oo.cpu().numpy()[:-1], oo.cpu().numpy()[1:])}
        hk, ho, hv = host.reduce(r)
        d_host = {int(k): list(hv[ho[i]:ho[i + 1]]) for i, k in enumerate(hk)}
        assert d_dev == d_host


def test_resubmitted_map_task_replaces_values(sc):
    sh = vb.Shuffle(sc, 2, 3, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP)
    keys = np.array([1, 2, 3], dtype=np.uint64)

    def put(m, vals):
        o = np.concatenate([[0], np.cumsum([len(v) for v in vals])]).astype(np.uint64)
        d = np.frombuffer(b"".join(vals) + b"\0", dtype=np.uint8)
        L.check(sc._lib.vb_shuffle_map_bytes(sh._h, m, keys.ctypes.data, o.ctypes.data, d.ctypes.data, len(d) - 1, 3, L.VB_HOST))
    put(0, [b"old1", b"old2", b"old3"])
    put(1, [b"x", b"", b"z"])
    put(0, [b"new1", b"n2", b""])
    sh.seal()
    sh.as_str = False
    got = {}
    for r in range(3):
        k, o, v = sh.reduce(r)
        got.update({int(x): list(v[o[i]:o[i + 1]]) for i, x in enumerate(k)})
    assert got == {1: [b"new1", b"x"], 2: [b"n2", b""], 3: [b"", b"z"]}


# -- N-way joins: bytes, u64, bytes, and the same shuffle twice ---------------------------------------------------------
def test_cogroup_and_joins_n(sc):
    rng = np.random.default_rng(11)
    R = 5
    ks = [rng.integers(0, hi, n).astype(np.uint64) for n, hi in ((400, 60), (300, 60), (350, 90))]   # keys 60-89: c only
    va = rand_values(rng, 400, 0.0)
    vc = [x.hex() for x in rand_values(rng, 350, 0.0)]
    vc[0] = ""
    a = sc.parallelize(ks[0], 3, values=va)
    b = sc.parallelize(ks[1], 2, values=np.arange(300, dtype=np.uint64) * 7)
    c = sc.parallelize(ks[2], 4, values=vc)
    ai = sc.parallelize(ks[0], 3, values=np.arange(400, dtype=np.uint64))
    ci = sc.parallelize(ks[2], 4, values=np.arange(350, dtype=np.uint64))
    byt = vb.CoGroupedRdd([a, b, c, a], R)
    ind = vb.CoGroupedRdd([ai, b, ci, ai], R)
    # cogroup
    cg = {int(k): lists for k, lists in byt.collect()}
    ci_ = {int(k): lists for k, lists in ind.collect()}
    assert cg.keys() == ci_.keys()
    for k, lists in ci_.items():
        want = [[va[i] for i in lists[0]], list(lists[1]), [vc[i] for i in lists[2]], [va[i] for i in lists[3]]]
        assert [list(x) for x in cg[k]] == want
    # inner and outer joins: same rows in the same order as the index run
    for req in (0b1111, 0b0010, 0):
        kb_, vsb = byt.outer_join_collect(req)
        ki, vsi = ind.outer_join_collect(req)
        assert np.array_equal(kb_, ki)
        for j, table in ((0, va), (2, vc), (3, va)):
            m, d = np.ma.getmaskarray(vsi[j]), np.ma.getdata(vsi[j])
            assert list(vsb[j]) == [None if m[t] else table[int(d[t])] for t in range(len(ki))]
        assert np.array_equal(np.ma.getdata(vsb[1]), np.ma.getdata(vsi[1]))
        assert np.array_equal(np.ma.getmaskarray(vsb[1]), np.ma.getmaskarray(vsi[1]))
    # None differs from the empty value
    kb_, vsb = byt.outer_join_collect(0)
    assert any(v is None for v in vsb[0]) and any(v == "" for v in vsb[2])
    # two sides: vb_join, vb_join_outer and vb_cogroup through the filtered internal shuffles
    for kind in (None, "left", "right", "full"):
        jb = (a.join(c, R) if kind is None else getattr(a, f"{kind}_outer_join")(c, R)).collect()
        ji = (ai.join(ci, R) if kind is None else getattr(ai, f"{kind}_outer_join")(ci, R)).collect()
        assert np.array_equal(jb[0], ji[0])
        for got, idx, table in ((jb[1], ji[1], va), (jb[2], ji[2], vc)):
            m = np.ma.getmaskarray(idx)
            assert list(got) == [None if m[t] else table[int(np.ma.getdata(idx)[t])] for t in range(len(idx))]
    jr = a.join(c, R)
    ir = ai.join(ci, R)
    for r in range(R):
        kb2, (lo, lv), (ro, rv) = jr.cogroup_compute(r)
        ki2, (lo2, lv2), (ro2, rv2) = ir.cogroup_compute(r)
        assert np.array_equal(kb2, ki2) and np.array_equal(lo, lo2) and np.array_equal(ro, ro2)
        assert list(lv) == [va[int(i)] for i in lv2] and list(rv) == [vc[int(i)] for i in rv2]


# -- String keys ---------------------------------------------------------------------------------------------------------
def test_string_keys(sc):
    rng = np.random.default_rng(3)
    R = 6
    words = [f"k{i}" for i in range(40)] + ["", "\x00"]
    ka = [words[i] for i in rng.integers(0, len(words), 500)]
    kc = [words[i] for i in rng.integers(0, len(words), 300)]
    va = rand_values(rng, 500, 0.0)
    vc = [f"v{i}" for i in range(300)]
    a = sc.parallelize(ka, 3, values=va)
    ai = sc.parallelize(ka, 3, values=np.arange(500, dtype=np.uint64))
    b = sc.parallelize(kc, 2, values=np.arange(300, dtype=np.uint64))
    c = sc.parallelize(kc, 2, values=vc)
    ci = b
    # group_by_key
    gb = a.group_by_key(R).collect().to_dict()
    gi = ai.group_by_key(R).collect().to_dict()
    assert {k: list(v) for k, v in gb.items()} == {k: [va[int(i)] for i in v] for k, v in gi.items()}
    # cogroup and joins, mixed with a u64 side
    byt, ind = StrCoGroupedRdd([a, b, c], R), StrCoGroupedRdd([ai, b, ci], R)
    cb = {k: l for k, l in byt.collect()}
    cix = {k: l for k, l in ind.collect()}
    assert cb.keys() == cix.keys()
    for k, l in cix.items():
        assert [list(x) for x in cb[k]] == [[va[int(i)] for i in l[0]], list(l[1]), [vc[int(i)] for i in l[2]]]
    for req in (0b111, 0b001, 0):
        # the order of keys within a partition is unspecified: compare the rows as sorted lists
        kb_, vsb = byt.outer_join_collect(req)
        ki, vsi = ind.outer_join_collect(req)
        side = lambda col, t: None if np.ma.getmaskarray(col)[t] else int(np.ma.getdata(col)[t])
        got = [(kb_[t], vsb[0][t], side(vsb[1], t), vsb[2][t]) for t in range(len(kb_))]
        want = [(ki[t], None if side(vsi[0], t) is None else va[side(vsi[0], t)], side(vsi[1], t),
                 None if side(vsi[2], t) is None else vc[side(vsi[2], t)]) for t in range(len(ki))]
        assert sorted(got, key=repr) == sorted(want, key=repr)


# -- sort_by_key with a bytes payload ------------------------------------------------------------------------------------
def test_sort_by_key_payload(sc):
    rng = np.random.default_rng(8)
    n, R = 30_000, 9
    keys = rng.integers(0, 2000, n).astype(np.uint64)
    values = rand_values(rng, n)
    si = sc.parallelize(keys, 5, values=np.arange(n, dtype=np.uint64)).sort_by_key(R)
    sb = sc.parallelize(keys, 5, values=values).sort_by_key(R)
    for r in range(R):
        ki, vi = si.compute(r)
        kb, vbs = sb.compute(r)
        assert np.array_equal(ki, kb)
        assert list(vbs) == [values[int(i)] for i in vi]
    # equal keys keep input order: the index payload ascends within each key
    k, v = si.collect()
    same = k[1:] == k[:-1]
    assert np.all(v[1:][same] > v[:-1][same])


def test_sort_by_key_payload_string_keys(sc):
    """vb_shuffle_create_str_sort_bytes: keys, key bytes and cuts bit-equal to the u64-payload sort of the same keys, and
    every row carries its own bytes, equal keys in input order."""
    rng = np.random.default_rng(9)
    n, R = 40_000, 9
    words = [f"w{i:04d}" for i in rng.integers(0, 3000, n)] + ["", "\x00", "w"]
    svals = rand_values(rng, len(words))
    ti = StrSortedRdd(sc.parallelize(words, 5, values=np.arange(len(words), dtype=np.uint64)), R)
    tb = StrSortedRdd(sc.parallelize(words, 5, values=svals), R)
    for r in range(R):
        koi, kbi, vi = ti.compute_raw(r)
        kob, kbb, vbs = tb.compute_raw(r)
        assert np.array_equal(koi, kob) and np.array_equal(kbi, kbb)      # same rows, keys and cut in this partition
        assert list(vbs) == [svals[int(i)] for i in vi]
    k, v = ti.collect()
    same = k[1:] == k[:-1]
    assert np.all(v[1:][same] > v[:-1][same])                              # equal keys in input order
    # the byte-string payload does not cross ranks yet
    h = ctypes.c_void_p()
    assert sc._lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 1, 2, L.VB_BYTES, 0, 2, ctypes.byref(h)) == L.VB_ERR_UNSUPPORTED


# -- more than 2^32 value bytes in one partition ------------------------------------------------------------------------
def test_over_4gib_one_partition(sc):
    import torch
    n, size = 70_000, 65_536
    total = n * size
    lib = sc._lib
    offs = torch.arange(0, n + 1, dtype=torch.int64, device="cuda") * size
    tags = torch.arange(n, device="cuda") * size, (torch.arange(n, device="cuda") % 256).to(torch.uint8)

    def pattern():
        d = (torch.arange(size, dtype=torch.int64, device="cuda") % 251).to(torch.uint8).repeat(n)
        d[tags[0]] = tags[1]                              # each value starts with its own tag byte
        return d
    data = pattern()
    keys = torch.zeros(n, dtype=torch.int64, device="cuda")
    sh = vb.Shuffle(sc, 1, 1, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP)
    torch.cuda.synchronize()
    L.check(lib.vb_shuffle_map_bytes(sh._h, 0, ctypes.c_void_p(keys.data_ptr()), ctypes.c_void_p(offs.data_ptr()),
                                     ctypes.c_void_p(data.data_ptr()), total, n, L.VB_DEVICE))
    del data
    sh.seal()
    nk, nv = sh.reduce_size(0)
    assert (nk, nv) == (1, n)
    refs = torch.empty(n, dtype=torch.int64, device="cuda")
    sh.reduce_device(0, out_vals=refs)
    nb = ctypes.c_uint64()
    L.check(lib.vb_shuffle_gather_bytes_size(sh._h, ctypes.c_void_p(refs.data_ptr()), n, L.VB_DEVICE, ctypes.byref(nb)))
    assert nb.value == total > 1 << 32
    go = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    gb = torch.empty(total, dtype=torch.uint8, device="cuda")
    L.check(lib.vb_shuffle_gather_bytes(sh._h, ctypes.c_void_p(refs.data_ptr()), n, L.VB_DEVICE, ctypes.c_void_p(go.data_ptr()),
                                        ctypes.c_void_p(gb.data_ptr()), L.VB_DEVICE))
    assert torch.equal(go, torch.arange(0, n + 1, dtype=torch.int64, device="cuda") * size)   # one map task: input order
    want = pattern()
    assert torch.equal(gb[tags[0]], tags[1])              # sampled values: every value's first byte
    assert int(gb[-size:].to(torch.int64).sum()) == int(want[-size:].to(torch.int64).sum())   # checksum of the last value
    assert torch.equal(gb, want)
    sh.free()


# -- refusals and bad references -----------------------------------------------------------------------------------------
def test_refusals(sc):
    lib, h = sc._lib, ctypes.c_void_p()
    for agg in (L.VB_AGG_SUM, L.VB_AGG_MIN, L.VB_AGG_MAX, L.VB_AGG_COUNT):
        assert lib.vb_shuffle_create(sc._h, 0, 1, 1, L.VB_U64, L.VB_BYTES, agg, 0, ctypes.byref(h)) == L.VB_ERR_UNSUPPORTED
        assert lib.vb_shuffle_create_str(sc._h, 0, 1, 1, L.VB_BYTES, agg, ctypes.byref(h)) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_create(sc._h, 0, 1, 1, L.VB_BYTES, L.VB_U64, L.VB_AGG_GROUP, 0, ctypes.byref(h)) == L.VB_ERR_INVALID
    dts = (ctypes.c_int32 * 1)(L.VB_BYTES)
    spec = (L.vb_agg_col * 1)(L.vb_agg_col(L.VB_AGG_SUM, 0))
    assert lib.vb_shuffle_create_multi(sc._h, 0, 1, 1, L.VB_U64, 1, dts, 1, spec, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_create_str_dist(sc._h, 0, 1, 1, L.VB_BYTES, L.VB_AGG_GROUP, 0, 2, ctypes.byref(h)) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_create_str_sort_dist(sc._h, 0, 1, 1, L.VB_BYTES, 0, 2, ctypes.byref(h)) == L.VB_ERR_UNSUPPORTED
    sh = vb.Shuffle(sc, 1, 2, L.VB_U64, L.VB_BYTES, L.VB_AGG_COGROUP)
    counts = (ctypes.c_uint64 * 2)()
    assert lib.vb_shuffle_set_dist(sh._h, 0, 2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_prepare(sh._h, counts) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_counts(sh._h, counts) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_exchange(sh._h, L.VB_XCHG_AUTO) == L.VB_ERR_UNSUPPORTED
    blob = np.zeros(1, dtype=np.uint64)
    assert lib.vb_shuffle_map_blob(sh._h, 0, blob.ctypes.data, 8, L.VB_HOST) == L.VB_ERR_UNSUPPORTED
    keys = np.array([5, 6], dtype=np.uint64)
    assert lib.vb_shuffle_map_soa(sh._h, 0, keys.ctypes.data, keys.ctypes.data, 2, L.VB_HOST) == L.VB_ERR_INVALID
    other = vb.Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_GROUP)
    offs = np.array([3, 5, 9], dtype=np.uint64)
    data = np.frombuffer(b"...abcdefg", dtype=np.uint8)
    assert lib.vb_shuffle_map_bytes(other._h, 0, keys.ctypes.data, offs.ctypes.data, data.ctypes.data, 10, 2, L.VB_HOST) == L.VB_ERR_INVALID
    # bad offsets, host and device
    bad = np.array([3, 2, 9], dtype=np.uint64)
    assert lib.vb_shuffle_map_bytes(sh._h, 0, keys.ctypes.data, bad.ctypes.data, data.ctypes.data, 10, 2, L.VB_HOST) == L.VB_ERR_INVALID
    beyond = np.array([3, 5, 11], dtype=np.uint64)
    assert lib.vb_shuffle_map_bytes(sh._h, 0, keys.ctypes.data, beyond.ctypes.data, data.ctypes.data, 10, 2, L.VB_HOST) == L.VB_ERR_INVALID
    import torch
    dk, dbad, dd = (torch.from_numpy(x.astype(np.int64) if x.dtype == np.uint64 else x.copy()).cuda() for x in (keys, bad, data))
    torch.cuda.synchronize()
    assert lib.vb_shuffle_map_bytes(sh._h, 0, ctypes.c_void_p(dk.data_ptr()), ctypes.c_void_p(dbad.data_ptr()),
                                    ctypes.c_void_p(dd.data_ptr()), 10, 2, L.VB_DEVICE) == L.VB_ERR_INVALID
    # a good map task (offsets not starting at 0), then bad references
    L.check(lib.vb_shuffle_map_bytes(sh._h, 0, keys.ctypes.data, offs.ctypes.data, data.ctypes.data, 10, 2, L.VB_HOST))
    sh.seal()
    good = np.array([(1 << 32) | 1, 0, 1 << 32], dtype=np.uint64)
    for refs in ([12345], [(2 << 32) | 0], [(1 << 32) | 2], [7]):
        r = np.array(list(good) + refs, dtype=np.uint64)
        o = np.full(len(r) + 1, 77, dtype=np.uint64)
        out = np.full(16, 0xAB, dtype=np.uint8)
        nb = ctypes.c_uint64()
        assert lib.vb_shuffle_gather_bytes_size(sh._h, r.ctypes.data, len(r), L.VB_HOST, ctypes.byref(nb)) == L.VB_ERR_INVALID
        assert lib.vb_shuffle_gather_bytes(sh._h, r.ctypes.data, len(r), L.VB_HOST, o.ctypes.data, out.ctypes.data, L.VB_HOST) == L.VB_ERR_INVALID
        assert np.all(o == 77) and np.all(out == 0xAB)
    sh.as_str = False
    assert list(sh.gather(good)) == [b"cdef", b"", b"ab"]


def test_python_refusals(sc):
    p = sc.parallelize(np.arange(4, dtype=np.uint64), 2, values=["a", "b", "c", "d"])
    for f in (lambda: p.reduce_by_key("sum", 2), lambda: p.count_by_key(2), lambda: p.combine_by_key({"n": ("count", None)}, 2)):
        with pytest.raises(TypeError):
            f()


# -- N-way cogroup and joins against the Python restatement of CoGroupedRdd::compute ----------------------------------
def _py(v):
    return int(v) if isinstance(v, np.integer) else v


def test_n_way_against_python_reference(sc):
    rng = np.random.default_rng(21)
    R = 4
    ka, kb, kc = (rng.integers(0, hi, n).tolist() for n, hi in ((150, 30), (100, 30), (120, 45)))
    va = rand_values(rng, 150, 0.0)
    vb_ = rng.integers(0, 1 << 40, 100).tolist()
    vc = [x.hex() for x in rand_values(rng, 120, 0.0)]
    sides = [(ka, va, 3), (kb, vb_, 2), (kc, vc, 4), (ka, va, 3)]
    parents = [(list(zip(k, v)), ns) for k, v, ns in sides]
    rdds = [sc.parallelize(np.array(k, dtype=np.uint64), ns,
                           values=v if isinstance(v[0], (str, bytes)) else np.array(v, dtype=np.uint64)) for k, v, ns in sides]
    cg = vb.CoGroupedRdd(rdds, R)
    got = {int(k): [[_py(v) for v in l] for l in lists] for k, lists in cg.collect()}
    assert got == {k: [list(l) for l in lists] for k, lists in CN.cogroup_n(parents, R)}
    for req in (0b1111, 0b0101, 0):
        k, cols = cg.outer_join_collect(req)
        rows = [(int(k[t]), [None if np.ma.isMaskedArray(c) and c.mask[t] else _py(np.ma.getdata(c)[t]) for c in cols])
                for t in range(len(k))]
        assert sorted(rows, key=repr) == sorted(JN.join_n_outer(parents, R, req), key=repr)


# -- the grouping paths of tests/test_gpu_group_paths.py with byte-string values -------------------------------------
SOA_CASES = [c for c, spec in GROUP_CASES.items() if spec[2] in ("dev_soa", "dev_soa_misaligned", "host_soa")]
PHI_BITS = int(np.uint64(PHI).view(np.int64))


def _vals_of_rows(rows):
    """Value of row r: the first r % 9 bytes of (r * PHI) little-endian (0 to 8 bytes), as Arrow offsets and bytes."""
    lens = (rows % 9).astype(np.int64)
    words = (rows.astype(np.uint64) * PHI).view(np.uint8).reshape(-1, 8)
    offs = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    keep = np.arange(8)[None, :] < lens[:, None]
    return offs, np.ascontiguousarray(words[keep])


@pytest.mark.parametrize("case", SOA_CASES)
def test_group_paths_bytes(sc, case):
    """Each SoA case of GROUP_CASES (one to four id-sort passes, the misaligned scatters, the two-pass multisplit at 257
    partitions, the hot key whose CSR starts by atomicMin), grouped once with the row index as a value and once with
    byte-string values in the same placement: the same kernels run (rp_scatter launches), the index run matches
    tests/group_ref.py, and key by key the bytes run gives exactly the bytes of the index run's rows, checked on the
    device."""
    import torch
    D, n, where, M, R, hot = GROUP_CASES[case]
    rng = np.random.default_rng([list(GROUP_CASES).index(case), 7])
    keys = exact_keys(rng, n, D, hot=hot)
    rows = np.arange(n, dtype=np.int64)
    kc, ic = place(where, keys, rows)
    offs, data = _vals_of_rows(rows)
    col = StrKeys(offs, data) if where == "host_soa" else StrKeys(torch.from_numpy(offs).cuda(), torch.from_numpy(data).cuda())
    runs = []
    for vals, vcode in ((ic, L.VB_I64), (vb.rdd._BytesCol(col), L.VB_BYTES)):
        maps = sliced(kc, vals, n, M)
        sh = vb.Shuffle(sc, len(maps), R, L.VB_U64, vcode, L.VB_AGG_GROUP)
        for m, (k_, v_, a, b) in enumerate(maps):
            sh.map(m, k_, v_, a, b)
        sh.seal()
        assert sh.stats()["kernels"]["rp_scatter"]["launches"] == scatter_launches(D, R)
        runs.append(sh)
    si, sb = runs
    parts = [si.reduce(r) for r in range(R)]
    G.assert_group_equal(parts, keys, rows, R)
    if hot:
        assert max(int(np.diff(p[1].astype(np.int64)).max(initial=0)) for p in parts) > 0.55 * n
    del parts
    dlens = torch.from_numpy(rows % 9).cuda()
    for r in range(R):
        per = []
        for sh in runs:
            nk, nv = sh.reduce_size(r)
            k_, o_, v_ = (torch.empty(x, dtype=torch.int64, device="cuda") for x in (nk, nk + 1, nv))
            sh.reduce_device(r, out_keys=k_, out_offs=o_, out_vals=v_)
            kv, order = torch.sort(torch.repeat_interleave(k_, torch.diff(o_)), stable=True)   # key by key, lists in order
            per.append((kv, v_[order]))
        (kvi, ri), (kvb, refs) = per
        assert torch.equal(kvi, kvb)
        nv, nb = refs.numel(), ctypes.c_uint64()
        L.check(sc._lib.vb_shuffle_gather_bytes_size(sb._h, ctypes.c_void_p(refs.data_ptr()), nv, L.VB_DEVICE, ctypes.byref(nb)))
        go = torch.empty(nv + 1, dtype=torch.int64, device="cuda")
        gb = torch.empty(max(nb.value, 1), dtype=torch.uint8, device="cuda")
        L.check(sc._lib.vb_shuffle_gather_bytes(sb._h, ctypes.c_void_p(refs.data_ptr()), nv, L.VB_DEVICE,
                                                ctypes.c_void_p(go.data_ptr()), ctypes.c_void_p(gb.data_ptr()), L.VB_DEVICE))
        lens = dlens[ri]
        assert torch.equal(torch.diff(go), lens)
        if nb.value:
            owner = torch.repeat_interleave(torch.arange(nv, device="cuda"), lens)
            pos = torch.arange(nb.value, device="cuda") - go[:-1][owner]
            word = ri[owner] * PHI_BITS                              # wraps as the u64 product does
            assert torch.equal(gb[:nb.value], ((word >> (8 * pos)) & 0xFF).to(torch.uint8))
    for sh in runs:
        sh.free()


def test_gather_null_out_bytes_writes_nothing(sc):
    import torch
    sh = vb.Shuffle(sc, 1, 1, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP)
    keys = np.array([1, 2], dtype=np.uint64)
    offs = np.array([0, 3, 5], dtype=np.uint64)
    data = np.frombuffer(b"abcde", dtype=np.uint8)
    L.check(sc._lib.vb_shuffle_map_bytes(sh._h, 0, keys.ctypes.data, offs.ctypes.data, data.ctypes.data, 5, 2, L.VB_HOST))
    sh.seal()
    refs = torch.tensor([(1 << 32) | 1, 1 << 32], dtype=torch.int64, device="cuda")
    out = torch.full((3,), 77, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    assert sc._lib.vb_shuffle_gather_bytes(sh._h, ctypes.c_void_p(refs.data_ptr()), 2, L.VB_DEVICE, ctypes.c_void_p(out.data_ptr()),
                                           None, L.VB_DEVICE) == L.VB_ERR_INVALID
    assert out.tolist() == [77, 77, 77]
    sh.free()
