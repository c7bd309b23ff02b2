"""repartition(n) = coalesce(n, shuffle = true) on the device, one process: every partition's items exactly, in order,
against tests/repartition_ref.py, for every item shape, partition counts on both sides of the one-pass limit (256),
starts that wrap around 2^64, host / device / borrowed sources, host and device destinations, empty maps, n_map 0 and
resubmission; the multiset of each partition against the existing partition_by_key route; and every refusal."""
import ctypes

import numpy as np
import pytest
import torch

import vega_b200 as vb
from tests import repartition_ref as RP
from vega_b200 import _lib as L
from vega_b200.rdd import RepShuffle, StrKeys, _BytesCol, _Col, slice_starts

pytestmark = pytest.mark.gpu

SHAPES = {"u1": (1, False), "u2": (2, False), "b": (0, True), "u1b": (1, True)}


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def make_items(rng, n, shape, big=False):
    n_cols, has_bytes = SHAPES[shape]
    cols = [rng.integers(0, 1 << 63, size=n, dtype=np.int64).view(np.uint64) for _ in range(n_cols)]
    items = None
    if has_bytes:
        lens = rng.integers(0, 21, size=n)
        items = [bytes(rng.integers(0, 256, size=int(k), dtype=np.uint8)) for k in lens]
        if n > 3:
            items[1] = b""
            if big:
                items[2] = bytes(rng.integers(0, 256, size=1 << 20, dtype=np.uint8))
    return cols, items


def as_col(a, src):
    if src == "host":
        return _Col(a, role="value")
    c = _Col(torch.from_numpy(a.view(np.int64)).cuda(), role="value")
    if src == "device":
        c.loc = L.VB_DEVICE                                     # copied by the map call
    c.code = L.VB_U64
    return c


def as_bytes(items, src):
    offs = np.zeros(len(items) + 1, dtype=np.uint64)
    np.cumsum([len(x) for x in items], out=offs[1:])
    data = np.frombuffer(b"".join(items), dtype=np.uint8)
    if src == "host":
        k = StrKeys(offs, data)
    else:
        k = StrKeys(torch.from_numpy(offs.view(np.int64)).cuda(), torch.from_numpy(data.copy()).cuda())
    b = _BytesCol(k)
    b.as_str = False
    return b


def read(sh, r, dst):
    if dst == "host":
        cols, items = sh.reduce(r)
        return [c.tolist() for c in cols], (list(items) if items is not None else None)
    n, nb = sh.reduce_size(r)
    outs = [torch.empty(n, dtype=torch.int64, device="cuda") for _ in sh.codes]
    offs = torch.empty(n + 1, dtype=torch.int64, device="cuda") if sh.has_bytes else None
    data = torch.empty(nb + 3, dtype=torch.uint8, device="cuda")[3:] if sh.has_bytes else None   # an unaligned destination
    sh.reduce_device(r, outs, offs, data)
    cols = [o.cpu().numpy().view(np.uint64).tolist() for o in outs]
    if not sh.has_bytes:
        return cols, None
    o, raw = offs.cpu().tolist(), data.cpu().numpy().tobytes()
    assert o[0] == 0 and o[-1] == nb
    return cols, [raw[o[i]:o[i + 1]] for i in range(n)]


def run(sc, shape, bounds, cols, items, starts, R, src, dst):
    n_cols, has_bytes = SHAPES[shape]
    sh = RepShuffle(sc, len(bounds) - 1, R, [L.VB_U64] * n_cols, has_bytes, as_str=False)
    ccols = [as_col(c, src) for c in cols]
    bcol = as_bytes(items, src) if has_bytes else None
    for m in range(len(bounds) - 1):
        sh.map_items(m, starts[m], ccols, bcol, int(bounds[m]), int(bounds[m + 1]))
    sh.seal()
    got = [read(sh, r, dst) for r in range(R)]
    sh.free()
    return got


def expected(shape, bounds, cols, items, starts, R):
    n_cols, has_bytes = SHAPES[shape]
    rows = list(range(int(bounds[-1])))
    per_map = [rows[int(bounds[m]):int(bounds[m + 1])] for m in range(len(bounds) - 1)]
    parts = RP.repartition(per_map, starts, R)
    return [([[int(c[i]) for i in p] for c in cols], ([items[i] for i in p] if has_bytes else None)) for p in parts]


CASES = [(shape, R, sk) for shape in SHAPES for R in (1, 3, 256, 257, 1000) for sk in ("zero", "r_minus_1", "wrap")]


@pytest.mark.parametrize("shape,R,start_kind", CASES)
def test_exact_order(sc, shape, R, start_kind):
    i = CASES.index((shape, R, start_kind))
    src = ("host", "device", "borrowed")[(i + i // 3) % 3]         # every source meets every start kind
    dst = ("host", "device")[(i // 3 + i // 15) % 2]
    if SHAPES[shape] == (0, True) and src == "borrowed":
        src = "device"                                          # byte strings are always copied
    rng = np.random.default_rng(i)
    n = 3000 if R < 1000 else 6000
    cols, items = make_items(rng, n, shape, big=(R == 3 and start_kind == "zero"))
    bounds = [0, 0, 1000, 1001, 1001, 2200, n]                  # empty maps included
    start = {"zero": 0, "r_minus_1": R - 1, "wrap": (1 << 64) - 3}[start_kind]
    starts = [start, start + 1, start, (1 << 64) - 1, 12345, start]
    assert run(sc, shape, bounds, cols, items, starts, R, src, dst) == expected(shape, bounds, cols, items, starts, R)


def test_large_single_pass(sc):
    """Enough rows for many tiles per part of the multisplit: 5e5 items in 8 maps, R = 64 and R = 300."""
    rng = np.random.default_rng(7)
    n = 500_000
    a = rng.integers(0, 1 << 63, size=n, dtype=np.int64).view(np.uint64)
    bounds = [int(x) for x in slice_starts(n, 8)]
    starts = [int(x) for x in rng.integers(0, 1 << 63, size=8)]
    for R in (64, 300):
        got = run(sc, "u1", bounds, [a], None, starts, R, "borrowed", "host")
        pos = np.concatenate([np.arange(1, bounds[m + 1] - bounds[m] + 1, dtype=np.uint64) + np.uint64(starts[m]) for m in range(8)])
        part = np.array([L.lib().vb_get_partition(int(p), 8, R) for p in pos[:20000]])
        want0 = [a[:20000][part == r].tolist() for r in range(R)]
        for r in range(R):          # the first 20000 rows (maps 0 and part of 1) lead each partition, in order
            assert got[r][0][0][:len(want0[r])] == want0[r]
        assert sum(len(g[0][0]) for g in got) == n


def test_n_map_zero(sc):
    sh = RepShuffle(sc, 0, 5, [L.VB_U64], True)
    sh.seal()
    for r in range(5):
        assert sh.reduce_size(r) == (0, 0)
        cols, items = sh.reduce(r)
        assert cols[0].size == 0 and len(items) == 0
    sh.free()


def test_resubmission_last_wins(sc):
    rng = np.random.default_rng(3)
    a, b = rng.integers(0, 1 << 40, size=500).astype(np.uint64), rng.integers(0, 1 << 40, size=300).astype(np.uint64)
    ia, ib = [bytes([i % 251]) * (i % 7) for i in range(500)], [bytes([i % 13]) * (i % 5 + 1) for i in range(300)]
    sh = RepShuffle(sc, 2, 7, [L.VB_U64], True, as_str=False)
    sh.map_items(0, 10, [_Col(a, role="value")], as_bytes(ia, "host"), 0, 500)
    sh.map_items(1, 20, [_Col(a, role="value")], as_bytes(ia, "host"), 0, 200)
    sh.map_items(0, 30, [_Col(b, role="value")], as_bytes(ib, "host"), 0, 300)    # replaces map 0
    sh.seal()
    want = RP.repartition([list(zip(b.tolist(), ib)), list(zip(a[:200].tolist(), ia[:200]))], [30, 20], 7)
    for r in range(7):
        cols, items = sh.reduce(r)
        assert list(zip(cols[0].tolist(), list(items))) == want[r]
    assert sh.stats()["rows_in"] == 500
    sh.free()


def test_matches_partition_by_key(sc):
    """The existing route vega's users have today: partition_by_key over (position, item) with host positions."""
    rng = np.random.default_rng(11)
    n, M, R = 20_000, 6, 37
    items = rng.integers(0, 1 << 62, size=n).astype(np.uint64)
    bounds = [int(x) for x in slice_starts(n, M)]
    starts = [int(x) for x in rng.integers(0, 1 << 63, size=M)]
    pos = np.concatenate([np.arange(1, bounds[m + 1] - bounds[m] + 1, dtype=np.uint64) + np.uint64(starts[m]) for m in range(M)])
    old = sc.parallelize(pos, M, values=items).partition_by_key(R).glom()
    new = sc.parallelize(items, M).repartition(R, starts=starts).glom()
    assert [sorted(x.view(np.uint64).tolist()) for x in old] == [sorted(x.tolist()) for x in new]


def test_coalesced_shuffle_case(sc):
    """tests/test_rdd.rs:364-385: parallelize(ones(100), 20).repartition(100) -> 100 partitions of the 100 items."""
    parts = sc.parallelize(np.ones(100, dtype=np.uint64), 20).repartition(100).glom()
    assert len(parts) == 100 and sum(len(p) for p in parts) == 100
    want = RP.repartition([[1] * 5 for _ in range(20)], [0] * 20, 100)
    assert [p.tolist() for p in parts] == want


def test_rdd_mirrors(sc):
    keys, vals = np.arange(1000, dtype=np.uint64), np.arange(1000, dtype=np.int64) * -3
    words = [f"w{i % 97}" * (i % 4) for i in range(1000)]
    starts = [5, 9, (1 << 64) - 2, 0]
    bounds = [int(x) for x in slice_starts(1000, 4)]
    per_map = lambda xs: [xs[bounds[m]:bounds[m + 1]] for m in range(4)]
    got = sc.parallelize(keys, 4, values=vals).repartition(9, starts=starts).glom()
    want = RP.repartition(per_map(list(zip(keys.tolist(), vals.tolist()))), starts, 9)
    assert [list(zip(k.tolist(), v.tolist())) for k, v in got] == want
    got = sc.parallelize(keys, 4, values=words).coalesce(9, shuffle=True, starts=starts).glom()
    want = RP.repartition(per_map(list(zip(keys.tolist(), words))), starts, 9)
    assert [list(zip(k.tolist(), list(v))) for k, v in got] == want
    got = sc.parallelize(words, 4).repartition(9, starts=starts).glom()
    assert [list(p) for p in got] == RP.repartition(per_map(words), starts, 9)
    got = sc.parallelize(words, 4, values=vals).repartition(9, starts=starts)
    k, v = got.collect()
    want = [x for p in RP.repartition(per_map(list(zip(words, vals.tolist()))), starts, 9) for x in p]
    assert list(zip(list(k), v.tolist())) == want
    rows = torch.arange(2000, dtype=torch.int64, device="cuda").reshape(1000, 2)
    a, b = sc.parallelize(rows, 4).repartition(9, starts=starts).collect()
    want = [x for p in RP.repartition(per_map([(2 * i, 2 * i + 1) for i in range(1000)]), starts, 9) for x in p]
    assert list(zip(a.tolist(), b.tolist())) == want


def code_of(fn):
    try:
        fn()
    except vb.VegaB200Error as e:
        return e.code
    return L.VB_OK


def test_refusals(sc):
    lib, h = L.lib(), ctypes.c_void_p()
    for n_cols, hb in ((3, 0), (0, 0), (1, 2), (2, -1)):
        assert lib.vb_shuffle_create_repartition(sc._h, 1, 2, 4, n_cols, hb, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_create_repartition(sc._h, 1, 2, 0, 1, 0, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_create_repartition(sc._h, 1, 2, 65537, 1, 0, ctypes.byref(h)) == L.VB_ERR_UNSUPPORTED

    plain = vb.Shuffle(sc, 1, 4, L.VB_U64, L.VB_U64, L.VB_AGG_GROUP)
    a = np.arange(100, dtype=np.uint64)
    ptrs = (ctypes.c_void_p * 1)(a.ctypes.data)
    n, nb = ctypes.c_uint64(), ctypes.c_uint64()
    assert lib.vb_shuffle_map_repartition(plain._h, 0, 0, ptrs, None, None, 0, 100, L.VB_HOST) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_repartition_size(plain._h, 0, ctypes.byref(n), ctypes.byref(nb)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_repartition(plain._h, 0, None, None, None, L.VB_HOST) == L.VB_ERR_INVALID
    plain.free()

    sh = RepShuffle(sc, 1, 4, [L.VB_U64], True)
    s = sh._h
    offs = np.arange(101, dtype=np.uint64)
    data = np.zeros(100, dtype=np.uint8)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    assert lib.vb_shuffle_map_repartition(s, 1, 0, ptrs, p(offs), p(data), 100, 100, L.VB_HOST) == L.VB_ERR_INVALID   # map_id
    assert lib.vb_shuffle_map_repartition(s, 0, 0, None, p(offs), p(data), 100, 100, L.VB_HOST) == L.VB_ERR_INVALID   # no column
    assert lib.vb_shuffle_map_repartition(s, 0, 0, ptrs, None, p(data), 100, 100, L.VB_HOST) == L.VB_ERR_INVALID      # no offsets
    bad = offs.copy(); bad[5] = 1
    assert lib.vb_shuffle_map_repartition(s, 0, 0, ptrs, p(bad), p(data), 100, 100, L.VB_HOST) == L.VB_ERR_INVALID    # decreasing
    assert lib.vb_shuffle_map_repartition(s, 0, 0, ptrs, p(offs), p(data), 99, 100, L.VB_HOST) == L.VB_ERR_INVALID     # past the end
    assert lib.vb_shuffle_map_repartition(s, 0, 0, ptrs, p(offs), p(data), 100, 100, 7) == L.VB_ERR_INVALID
    # every other call on a repartition shuffle, before and after seal
    other = [
        lambda: lib.vb_shuffle_map_soa(s, 0, p(a), p(a), 100, L.VB_HOST),
        lambda: lib.vb_shuffle_map_aos(s, 0, p(a), 50, L.VB_HOST),
        lambda: lib.vb_shuffle_map_bytes(s, 0, p(a), p(offs), p(data), 100, 100, L.VB_HOST),
        lambda: lib.vb_shuffle_map_blob(s, 0, p(data), 8, L.VB_HOST),
        lambda: lib.vb_shuffle_set_key_width(s, 4),
        lambda: lib.vb_shuffle_set_dist(s, 0, 2),
        lambda: lib.vb_shuffle_export_prepare(s, a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))),
    ]
    after = [
        lambda: lib.vb_shuffle_reduce_size(s, 0, ctypes.byref(n), ctypes.byref(nb)),
        lambda: lib.vb_shuffle_reduce(s, 0, None, None, None, None, L.VB_HOST),
        lambda: lib.vb_shuffle_reduce_blob_size(s, 0, ctypes.byref(n)),
        lambda: lib.vb_join_size(s, s, 0, ctypes.byref(n)),
        lambda: lib.vb_shuffle_gather_bytes_size(s, p(a), 1, L.VB_HOST, ctypes.byref(n)),
        lambda: lib.vb_shuffle_create_narrow(s, 0, ctypes.byref(h)),
    ]
    for f in other:
        assert f() == L.VB_ERR_INVALID
    assert lib.vb_shuffle_exchange(s, L.VB_XCHG_AUTO) == L.VB_ERR_STATE               # one process: nothing to exchange
    assert lib.vb_shuffle_exchange(s, L.VB_XCHG_P2P) == L.VB_ERR_UNSUPPORTED
    for rank, world in ((0, 0), (2, 2), (0, 257)):
        assert lib.vb_shuffle_create_repartition_dist(sc._h, 1, 2, 4, 1, 0, rank, world, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_repartition_size(s, 4, ctypes.byref(n), ctypes.byref(nb)) == L.VB_ERR_INVALID
    # still usable
    items = [bytes([i]) * (i % 3) for i in range(100)]
    sh.map_items(0, 41, [_Col(a, role="value")], as_bytes(items, "host"), 0, 100)
    sh.seal()
    for f in other + after:
        assert f() == L.VB_ERR_INVALID
    assert lib.vb_shuffle_reduce_repartition(s, 0, None, None, None, 5) == L.VB_ERR_INVALID
    r0 = RP.repartition([list(zip(a.tolist(), items))], [41], 4)
    big = next(r for r in range(4) if sum(len(x[1]) for x in r0[r]))
    o = np.empty(len(r0[big]) + 1, dtype=np.uint64)
    assert lib.vb_shuffle_reduce_repartition(s, big, None, p(o), None, L.VB_HOST) == L.VB_ERR_INVALID   # bytes, no out_bytes
    sh.as_str = False
    for r in range(4):
        cols, got = sh.reduce(r)
        assert list(zip(cols[0].tolist(), list(got))) == r0[r]
    sh.free()
