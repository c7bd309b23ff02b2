"""sort_by_key over String keys on the device (vb_shuffle_create_str_sort and vb.StrSortedRdd): every partition is
compared row for row with tests/str_sort_ref.py (keys, payload bits, partition sizes), and the large cases with the
integer sort_by_key of the keys' ranks."""
import ctypes
import struct

import numpy as np
import pytest

import vega_b200 as vb
from vega_b200 import _lib as L
from tests import str_sort_ref as SR

pytestmark = pytest.mark.gpu
CODE = {"u64": L.VB_U64, "i64": L.VB_I64, "f64": L.VB_F64}
NP = {"u64": np.uint64, "i64": np.int64, "f64": np.float64}


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


def _column(keys, lead=0):
    """(offsets, bytes) of byte keys; the offsets start at `lead` (a slice of a larger column) over lead filler bytes."""
    lens = np.array([len(k) for k in keys], dtype=np.uint64)
    offs = np.full(len(keys) + 1, lead, dtype=np.uint64)
    np.cumsum(lens, out=offs[1:])
    offs[1:] += np.uint64(lead)
    data = np.frombuffer(b"\xee" * lead + b"".join(keys), dtype=np.uint8)
    return offs, data


def _map(sh, m, keys, vals, loc, lead=0):
    """One map call of byte keys (and values, or None) through the C ABI, from host, device or device-borrowed memory."""
    import torch
    offs, data = _column(keys, lead)
    keep = []
    if loc == L.VB_HOST:
        op, dp = offs.ctypes.data, data.ctypes.data if len(data) else None
        vp = vals.ctypes.data if vals is not None and len(vals) else None
        keep = [offs, data, vals]
    else:
        to = torch.from_numpy(offs.view(np.int64).copy()).cuda()
        td = torch.from_numpy(data.copy()).cuda()
        tv = torch.from_numpy(vals.view(np.int64).copy()).cuda() if vals is not None else None
        torch.cuda.synchronize()
        op, dp = to.data_ptr(), td.data_ptr() if len(data) else None
        vp = tv.data_ptr() if tv is not None and len(vals) else None
        keep = [to, td, tv]
    if vals is not None and not len(vals):
        vp = None
    sh._keepalive.append(keep)
    L.check(sh._lib.vb_shuffle_map_str(sh._h, m, ctypes.c_void_p(op), ctypes.c_void_p(dp) if dp else None, len(data),
                                       ctypes.c_void_p(vp) if vp else None, len(keys), loc))


def _parts(sh):
    out = []
    for r in range(sh.n_reduce):
        ko, kb, v = sh.reduce_raw(r)
        out.append(([kb[int(ko[i]):int(ko[i + 1])].tobytes() for i in range(len(ko) - 1)], v))
    return out


def _check(got, want, vdt):
    assert len(got) == len(want)
    assert [len(g[0]) for g in got] == [len(w[0]) for w in want], "partition sizes"
    for r, ((gk, gv), (wk, wv)) in enumerate(zip(got, want)):
        assert gk == wk, f"keys of partition {r}"
        if wv is None:
            assert gv is None
        else:
            assert gv.dtype == NP[vdt]
            assert gv.view(np.uint64).tolist() == np.asarray(wv, dtype=NP[vdt]).view(np.uint64).tolist(), f"payload of partition {r}"


def _run(sc, maps, R, vdt="u64", loc=L.VB_HOST, lead=0):
    """maps: [(byte keys, values or None)]; every map's values None: key-only.  Returns the partitions and the
    reference's."""
    key_only = all(v is None for _, v in maps)
    sh = vb.StrShuffle(sc, len(maps), R, None if key_only else CODE[vdt], L.VB_AGG_SORT, sort=True)
    for m, (ks, vs) in enumerate(maps):
        _map(sh, m, ks, None if key_only else np.asarray(vs, dtype=NP[vdt]), loc, lead)
    sh.seal()
    keys = [k for ks, _ in maps for k in ks]
    vals = None if key_only else np.concatenate([np.asarray(vs, dtype=NP[vdt]) for _, vs in maps]) if maps else None
    return _parts(sh), SR.partitions(keys, vals, R), sh


def _split(keys, vals, M, rng):
    cuts = sorted(rng.integers(0, len(keys) + 1, M - 1).tolist())
    b = [0] + cuts + [len(keys)]
    return [(keys[b[i]:b[i + 1]], None if vals is None else vals[b[i]:b[i + 1]]) for i in range(M)]


def _edge_keys(rng):
    keys = [b"", b"\x00", b"a", b"a\x00", b"a\x00\x00", b"ab", b"\x7f", b"\x80", b"\xff", b"\xff\x00", b"\x00\xff"]
    for L_ in (7, 8, 9, 15, 16, 17):
        base = bytes(rng.integers(97, 123, L_, dtype=np.uint8))
        keys.append(base)
        for p in (7, 8, 15, 16):
            if p < L_:
                for b in (0x00, 0x41, 0x7F, 0x80, 0xFF):
                    keys.append(base[:p] + bytes([b]) + base[p + 1:])
        keys += [base[:-1], base + b"\x00"]
    prefix = bytes(rng.integers(0, 256, 1000, dtype=np.uint8))    # 1 KB keys sharing 1000 bytes: >= 143 rounds
    keys += [prefix + bytes(rng.integers(0, 256, 24, dtype=np.uint8)) for _ in range(12)]
    keys += [prefix, prefix[:999], prefix + b"\x00", prefix + b"\x00" * 24]
    return keys


@pytest.mark.parametrize("vdt", ["u64", "i64", "f64", None])
def test_word_and_prefix_edges(sc, vdt):
    rng = np.random.default_rng(1)
    pool = _edge_keys(rng)
    keys = [pool[i] for i in rng.integers(0, len(pool), 3 * len(pool))] + pool
    keys = [keys[i] for i in rng.permutation(len(keys))]
    if vdt is None:
        vals = None
    elif vdt == "f64":
        vals = rng.standard_normal(len(keys))
        vals[::7] = np.nan
        vals.view(np.uint64)[::11] = 0x7FF8DEADBEEF0001                  # a NaN with a payload of its own
    else:
        vals = rng.integers(-(1 << 62), 1 << 62, len(keys)).astype(NP[vdt])
    for R in (1, 3, 7):
        got, want, _ = _run(sc, _split(keys, vals, 4, rng), R, vdt or "u64")
        _check(got, want, vdt or "u64")


@pytest.mark.parametrize("dist", ["equal", "distinct", "zipf"])
@pytest.mark.parametrize("R", [1, 3, 300])
def test_key_distributions(sc, dist, R):
    rng = np.random.default_rng(R)
    n = 20_000
    if dist == "equal":
        keys = [b"same key"] * n
    elif dist == "distinct":
        keys = [b"k%x" % i for i in rng.permutation(n)]
    else:
        r = np.minimum(rng.zipf(1.3, n), 5000)
        keys = [b"w%d" % x for x in r]
    vals = np.arange(n, dtype=np.uint64)
    got, want, _ = _run(sc, _split(keys, vals, 5, rng), R)
    _check(got, want, "u64")


@pytest.mark.parametrize("n,R", [(0, 1), (0, 4), (1, 1), (1, 3), (5, 300), (40, 64)])
def test_sizes(sc, n, R):
    rng = np.random.default_rng(n + R)
    keys = [bytes(rng.integers(97, 100, int(rng.integers(0, 4)), dtype=np.uint8)) for _ in range(n)]
    vals = rng.integers(0, 1 << 63, n, dtype=np.uint64)
    got, want, sh = _run(sc, _split(keys, vals, 3, rng), R)
    _check(got, want, "u64")
    sizes = [sh.reduce_size(r) for r in range(R)]
    assert sum(s[0] for s in sizes) == n and all(s[2] == 0 for s in sizes)
    assert sum(s[1] for s in sizes) == sum(len(k) for k in keys)


@pytest.mark.parametrize("loc", [L.VB_HOST, L.VB_DEVICE, L.VB_DEVICE_BORROWED])
@pytest.mark.parametrize("lead", [0, 5])
def test_map_locations_and_offsets(sc, loc, lead):
    rng = np.random.default_rng(loc * 10 + lead)
    keys = [b"k%d" % x for x in rng.integers(0, 300, 5000)] + [b""] * 3
    vals = rng.integers(0, 1 << 63, len(keys), dtype=np.uint64)
    maps = _split(keys, vals, 4, rng)
    maps.insert(2, ([], np.zeros(0, dtype=np.uint64)))                  # an empty map
    got, want, _ = _run(sc, maps, 5, loc=loc, lead=lead)
    _check(got, want, "u64")


@pytest.mark.parametrize("key_only", [False, True])
def test_resubmitted_map_replaces_rows(sc, key_only):
    R = 3
    sh = vb.StrShuffle(sc, 2, R, None if key_only else L.VB_U64, L.VB_AGG_SORT, sort=True)
    v = lambda *x: None if key_only else np.array(x, dtype=np.uint64)
    _map(sh, 0, [b"b", b"gone", b"a"], v(1, 2, 3), L.VB_HOST)
    _map(sh, 1, [b"c", b"a"], v(4, 5), L.VB_HOST)
    _map(sh, 0, [b"b", b"a", b"a"], v(6, 7, 8), L.VB_HOST)             # "gone" only had the replaced rows
    sh.seal()
    want = SR.partitions([b"b", b"a", b"a", b"c", b"a"], None if key_only else np.array([6, 7, 8, 4, 5], dtype=np.uint64), R)
    _check(_parts(sh), want, "u64")


def test_big_endian_u64_keys_match_the_integer_sort(sc):
    rng = np.random.default_rng(7)
    n, M, R = 200_000, 6, 11
    pool = rng.integers(0, 1 << 64, 30_000, dtype=np.uint64)
    pool[:4] = [0, 1, 1 << 63, (1 << 64) - 1]
    ikeys = pool[rng.integers(0, len(pool), n)]
    vals = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    skeys = vb.StrKeys(np.arange(n + 1, dtype=np.uint64) * 8, ikeys.astype(">u8").view(np.uint8))
    s = vb.StrSortedRdd(sc.parallelize(skeys, M, values=vals), R)
    i = sc.parallelize(ikeys, M, values=vals).sort_by_key(R)
    for r in range(R):
        ko, kb, sv = s.compute_raw(r)
        ik, iv = i.compute(r)
        assert len(ko) - 1 == len(ik)
        assert np.array_equal(np.diff(ko.astype(np.int64)), np.full(len(ik), 8))
        assert np.array_equal(kb.view(">u8").astype(np.uint64), ik.view(np.uint64))
        assert np.array_equal(sv.view(np.uint64), iv.view(np.uint64))


def _hex_keys(ranks, width):
    """Fixed-width zero-padded lowercase hex keys of u64 ranks, built on the device: their byte order is the ranks'."""
    import torch
    n = len(ranks)
    shift = 4 * torch.arange(width - 1, -1, -1, device=ranks.device)
    digit = (ranks[:, None] >> shift[None, :]) & 15
    hexc = torch.tensor(list(b"0123456789abcdef"), dtype=torch.uint8, device=ranks.device)
    data = hexc[digit].reshape(-1)
    offs = torch.arange(n + 1, dtype=torch.int64, device=ranks.device) * width
    return vb.StrKeys(offs, data)


def test_fifty_million_rows_match_the_integer_sort_of_the_ranks(sc):
    import torch
    n, D, M, R, W = 50_000_000, 3_000_000, 8, 16, 7
    ranks = torch.empty(n, dtype=torch.int64, device="cuda")
    sc.gen_pairs(out_keys=ranks, n=n, mode="zipf", n_distinct=D, zipf_s=1.1)
    ranks &= (1 << 28) - 1
    vals = torch.arange(n, dtype=torch.int64, device="cuda")
    keys = _hex_keys(ranks, W)
    torch.cuda.synchronize()
    s = vb.StrSortedRdd(sc.parallelize(keys, M, values=vals), R)
    i = sc.parallelize(ranks, M, values=vals).sort_by_key(R)
    ish = i._run()
    sh = s._run()
    for r in range(R):
        nk, nb, _ = sh.reduce_size(r)
        ink, _ = ish.reduce_size(r)
        assert nk == ink and nb == W * nk, r
        ko = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
        kb = torch.empty(nb, dtype=torch.uint8, device="cuda")
        sv = torch.empty(nk, dtype=torch.int64, device="cuda")
        s.compute_device(r, out_key_offsets=ko, out_key_bytes=kb, out_vals=sv)
        ik = torch.empty(nk, dtype=torch.int64, device="cuda")
        iv = torch.empty(nk, dtype=torch.int64, device="cuda")
        ish.reduce_device(r, out_keys=ik, out_comb=iv)
        torch.cuda.synchronize()
        assert torch.equal(ko, torch.arange(nk + 1, dtype=torch.int64, device="cuda") * W)
        assert torch.equal(kb, _hex_keys(ik, W).data)
        assert torch.equal(sv, iv)


def test_error_codes(sc):
    lib = sc._lib
    inv, uns = L.VB_ERR_INVALID, L.VB_ERR_UNSUPPORTED
    out = ctypes.c_void_p()
    for dt in (3, -2, 99):
        assert lib.vb_shuffle_create_str_sort(sc._h, 0, 1, 2, dt, ctypes.byref(out)) == inv
    assert lib.vb_shuffle_create_str_sort(sc._h, 0, 1, 0, L.VB_U64, ctypes.byref(out)) == inv              # n_reduce 0
    assert lib.vb_shuffle_create_str_sort(None, 0, 1, 2, L.VB_U64, ctypes.byref(out)) == inv
    assert lib.vb_shuffle_create_str_sort(sc._h, 0, 1, 2, L.VB_U64, None) == inv
    # the single-aggregate String creates keep refusing SORT
    assert lib.vb_shuffle_create_str(sc._h, 0, 1, 1, L.VB_U64, L.VB_AGG_SORT, ctypes.byref(out)) == uns
    assert lib.vb_shuffle_create_str_dist(sc._h, 0, 1, 1, L.VB_U64, L.VB_AGG_SORT, 0, 2, ctypes.byref(out)) == uns

    sh = vb.StrShuffle(sc, 1, 2, L.VB_I64, L.VB_AGG_SORT, sort=True)
    ko_only = vb.StrShuffle(sc, 1, 2, None, L.VB_AGG_SORT, sort=True)
    h, hk = sh._h, ko_only._h
    offs, data = _column([b"b", b"a"])
    vals = np.array([2, 1], dtype=np.int64)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)
    u = ctypes.c_uint64()
    assert lib.vb_shuffle_map_str(h, 0, p(offs), p(data), 2, None, 2, L.VB_HOST) == inv                     # payload missing
    assert lib.vb_shuffle_map_str(hk, 0, p(offs), p(data), 2, p(vals), 2, L.VB_HOST) == inv                 # key-only with vals
    assert lib.vb_shuffle_map_str(h, 1, p(offs), p(data), 2, p(vals), 2, L.VB_HOST) == inv                  # map id
    # calls that do not apply
    assert lib.vb_shuffle_map_soa(h, 0, p(vals), p(vals), 2, L.VB_HOST) == inv
    assert lib.vb_shuffle_set_key_width(h, 4) == inv
    assert lib.vb_shuffle_map_str_cols(h, 0, p(offs), p(data), 2, None, 2, L.VB_HOST) == inv
    assert lib.vb_shuffle_export_str_cols_prepare(h, ctypes.byref(u), ctypes.byref(u)) == inv
    # not supported yet: across ranks, blobs
    assert lib.vb_shuffle_set_dist(h, 0, 2) == uns
    assert lib.vb_shuffle_export_str_prepare(h, ctypes.byref(u), ctypes.byref(u), ctypes.byref(u)) == uns
    assert lib.vb_shuffle_import_str(h, None, None, None, None, ctypes.byref(u), ctypes.byref(u), ctypes.byref(u)) == uns
    assert lib.vb_shuffle_export_prepare(h, ctypes.byref(u)) == uns
    assert lib.vb_shuffle_exchange(h, L.VB_XCHG_AUTO) == uns
    assert lib.vb_shuffle_map_blob(h, 0, p(vals), 8, L.VB_HOST) == uns
    L.check(lib.vb_shuffle_map_str(h, 0, p(offs), p(data), 2, p(vals), 2, L.VB_HOST))
    L.check(lib.vb_shuffle_map_str(hk, 0, p(offs), p(data), 2, None, 2, L.VB_HOST))
    sh.seal()
    ko_only.seal()
    buf = np.zeros(8, dtype=np.uint64)
    assert lib.vb_shuffle_reduce_size(h, 0, ctypes.byref(u), ctypes.byref(u)) == inv
    assert lib.vb_shuffle_reduce(h, 0, None, None, None, None, L.VB_HOST) == inv
    assert lib.vb_shuffle_reduce_str(h, 0, None, None, None, p(buf), None, L.VB_HOST) == inv                # out_offsets
    assert lib.vb_shuffle_reduce_str(h, 0, None, None, None, None, p(buf), L.VB_HOST) == inv                # out_vals
    assert lib.vb_shuffle_reduce_str(hk, 0, None, None, p(buf), None, None, L.VB_HOST) == inv               # key-only payload
    assert lib.vb_shuffle_reduce_str(h, 2, None, None, None, None, None, L.VB_HOST) == inv                  # reduce id
    assert lib.vb_shuffle_reduce_str_cols(h, 0, None, None, None, L.VB_HOST) == inv
    assert lib.vb_shuffle_reduce_blob_size(h, 0, ctypes.byref(u)) == uns
    sides = (ctypes.c_void_p * 1)(h.value)
    assert lib.vb_cogroup_n_str_size(sides, 1, 0, ctypes.byref(u), ctypes.byref(u), None) == inv
    assert lib.vb_join_n_str_size(sides, 1, 0, 1, ctypes.byref(u), ctypes.byref(u), ctypes.byref(u)) == inv
    assert lib.vb_join_size(h, h, 0, ctypes.byref(u)) == inv
    assert lib.vb_cogroup_n_size(sides, 1, 0, ctypes.byref(u), None) == inv
    assert lib.vb_shuffle_create_narrow(h, 0, ctypes.byref(out)) == inv
    # the shuffles still work after the refused calls
    _check(_parts(sh), SR.partitions([b"b", b"a"], vals, 2), "i64")
    _check(_parts(ko_only), SR.partitions([b"b", b"a"], None, 2), "u64")


def test_python_mirror(sc):
    import torch
    rng = np.random.default_rng(3)
    words = ["", "a", "ab", "é", "日本", "zz\x00", "a\x00"] + ["w%d" % x for x in range(200)]
    keys = [words[i] for i in rng.integers(0, len(words), 3000)]
    vals = rng.standard_normal(len(keys))
    vals[::5] = np.nan
    rdd = vb.StrSortedRdd(sc.parallelize(keys, 4, values=vals), 5)
    k, v = rdd.collect()
    want = sorted(zip(keys, vals.tolist()), key=lambda kv: kv[0].encode())
    assert k.tolist() == [kv[0] for kv in want]
    assert v.view(np.uint64).tolist() == np.array([kv[1] for kv in want]).view(np.uint64).tolist()
    parts = [rdd.compute(r) for r in range(5)]
    assert sum(len(p[0]) for p in parts) == len(keys)
    st = rdd.stats()
    assert st["rows_out"] == len(keys) and "str_order" in st["kernels"]
    # one value column given as a tuple, and the device read
    r2 = vb.StrSortedRdd(sc.parallelize(keys, 3, values=(vals,)), 2)
    sh = r2._run()
    nk, nb, _ = sh.reduce_size(1)
    ko = torch.empty(nk + 1, dtype=torch.int64, device="cuda")
    kb = torch.empty(nb, dtype=torch.uint8, device="cuda")
    tv = torch.empty(nk, dtype=torch.float64, device="cuda")
    r2.compute_device(1, out_key_offsets=ko, out_key_bytes=kb, out_vals=tv)
    hk, hv = r2.compute(1)
    assert vb.StrKeys(ko.cpu().numpy(), kb.cpu().numpy()).to_strs().tolist() == hk.tolist()
    assert tv.cpu().numpy().view(np.uint64).tolist() == hv.view(np.uint64).tolist()
    # key-only: a StrRdd
    ks = vb.StrSortedRdd(sc.parallelize(keys, 4), 3).collect()
    assert ks.tolist() == sorted(keys, key=str.encode)
    assert isinstance(vb.StrSortedRdd(sc.parallelize(keys, 4), 3).compute(0), np.ndarray)
