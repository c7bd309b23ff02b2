"""Byte-string values across ranks, W ranks of one shuffle in one process (vb_shuffle_create_bytes_dist /
_str_bytes_dist and the bytes export / import calls): every rank's exported columns are swapped with torch.cat, source-
rank major, through the same column bookkeeping as the all-to-all-v of vega_b200/dist.py (_bytes_export / _bytes_import
and the String pair).  Each case asserts that partition r has rows only on rank r % W and that the owners' partitions
equal the one-process bytes shuffle over the same map tasks: the same keys, each with the same values in the same
(map-id) order, byte for byte after the gather through the owning rank's shuffle."""
import ctypes

import numpy as np
import pytest
import torch

import vega_b200 as vb
from tests import multirank as MR
from tests.test_gpu_cogroup_n import abi_cogroup_n
from tests.test_gpu_join_n_outer import abi_outer
from tests.test_gpu_str_join import cogroup_part, join_part
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from vega_b200.rdd import _BytesCol, _Col, _StrCol

pytestmark = pytest.mark.gpu
SHAPES = ("empty", "nul", "small", "4k", "1m")


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


# ---- data -------------------------------------------------------------------------------------------------------------
def values(shape, n, rng):
    """n byte strings: all empty, short ones full of NUL and non-ASCII bytes, uniform 0-64 B, 1 % at 4 KiB among 0-64 B,
    or one value of 1 MiB + 3 among 0-64 B."""
    if shape == "empty":
        return [b""] * n
    hi = {"nul": 13}.get(shape, 65)
    lens = rng.integers(0, hi, n)
    if shape == "4k":
        lens[rng.random(n) < 0.01] = 4096
    if shape == "1m" and n:
        lens[rng.integers(0, n)] = (1 << 20) + 3
    data = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8)
    if shape == "nul":
        data[::3] = 0
        data[1::3] = rng.integers(0x80, 0x100, len(data[1::3]))
    raw, offs = data.tobytes(), np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return [raw[offs[i]:offs[i + 1]] for i in range(n)]


def int_keys(n, distinct, rng):
    return rng.integers(0, distinct, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(3)


def str_keys(n, distinct, rng):
    pool = ["", "k\x00", "é-ключ"] + ["w%05d" % i for i in range(distinct)] + ["L" * 300 + str(i) for i in range(3)]
    return [pool[i] for i in rng.integers(0, len(pool), n)]


# ---- the W-rank harness -----------------------------------------------------------------------------------------------
def one_process(sc, str_keys_, agg, M, R, keys, vals):
    """The one-process bytes shuffle over the M map tasks."""
    starts = vb.slice_starts(len(vals), M)
    if str_keys_:
        sh = vb.StrShuffle(sc, M, R, L.VB_BYTES, L.VB_AGG_SORT if agg == L.VB_AGG_SORT else L.VB_AGG_GROUP,
                           sort=agg == L.VB_AGG_SORT)
        kc = _StrCol(vb.StrKeys.from_strs(keys))
    else:
        sh = vb.Shuffle(sc, M, R, L.VB_U64, L.VB_BYTES, agg)
        kc = _Col(keys)
    vc = _BytesCol(vals)
    for m in range(M):
        sh.map(m, kc, vc, int(starts[m]), int(starts[m + 1]))
    sh.seal()
    sh.as_str = False
    return sh


def ranks(sc, str_keys_, agg, W, M, R, keys, vals):
    """The same map tasks on W ranks: map, export, swap, import, seal.  Returns the sealed shuffles by rank."""
    eng = vdist.StrBytesCudaEngine(sc) if str_keys_ else vdist.BytesCudaEngine(sc)
    starts = vb.slice_starts(len(vals), M)
    shs = [eng.create(M, R, L.VB_BYTES, agg, r, W) if str_keys_ else eng.create(M, R, L.VB_U64, L.VB_BYTES, agg, r, W)
           for r in range(W)]
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        for m in range(lo, hi):
            eng.map(sh, m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]])
    if W > 1:
        export, import_ = (vdist._str_bytes_export, vdist._str_bytes_import) if str_keys_ else (vdist._bytes_export, vdist._bytes_import)
        recv = MR.swap_columns([export(eng, sh, W) for sh in shs])
        for sh, (cols, splits) in zip(shs, recv):
            import_(eng, sh, cols, splits)
    for sh in shs:
        eng.seal(sh)
        sh.as_str = False
    return shs


def group_part(sh, r, str_keys_):
    """{key: [values, in order]} of one partition, the values gathered through sh."""
    if str_keys_:
        ko, kb, o, v = sh.reduce_raw(r)
        ks = [bytes(kb[int(ko[i]):int(ko[i + 1])]) for i in range(len(ko) - 1)]
    else:
        k, o, v = sh.reduce(r)
        ks = np.asarray(k).view(np.uint64).tolist()
    o = np.asarray(o).astype(np.int64)
    assert o[0] == 0 and o[-1] == len(v), "offsets do not start at 0 or end at the value count"
    d = {kk: list(v[o[i]:o[i + 1]]) for i, kk in enumerate(ks)}
    assert len(d) == len(ks), "a key appears twice in one partition"
    return d


def check_groups(one, shs, R, str_keys_):
    W = len(shs)
    for r in range(R):
        want = group_part(one, r, str_keys_)
        for d, sh in enumerate(shs):
            if r % W == d:
                assert group_part(sh, r, str_keys_) == want, f"partition {r} on rank {d}"
            else:
                assert sh.reduce_size(r)[0] == 0, f"rank {d} holds keys of partition {r}, owned by rank {r % W}"


# ---- GROUP and COGROUP, integer and String keys -----------------------------------------------------------------------
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("kind", ["group", "cogroup", "str_group"])
def test_groups_match_one_process(sc, kind, W, shape):
    rng = np.random.default_rng(W * 100 + SHAPES.index(shape))
    n, M, R = 6000, 11, 13
    s = kind == "str_group"
    keys = str_keys(n, 500, rng) if s else int_keys(n, 700, rng)
    vals = values(shape, n, rng)
    agg = L.VB_AGG_COGROUP if kind == "cogroup" else L.VB_AGG_GROUP
    check_groups(one_process(sc, s, agg, M, R, keys, vals), ranks(sc, s, agg, W, M, R, keys, vals), R, s)


@pytest.mark.parametrize("shape", ["small", "1m"])
@pytest.mark.parametrize("kind", ["group", "cogroup", "str_group"])
def test_256_ranks(sc, kind, shape):
    rng = np.random.default_rng(256 + SHAPES.index(shape))
    n, M, R = 20_000, 300, 300
    s = kind == "str_group"
    keys = str_keys(n, 3000, rng) if s else int_keys(n, 5000, rng)
    vals = values(shape, n, rng)
    agg = L.VB_AGG_COGROUP if kind == "cogroup" else L.VB_AGG_GROUP
    check_groups(one_process(sc, s, agg, M, R, keys, vals), ranks(sc, s, agg, 256, M, R, keys, vals), R, s)


@pytest.mark.parametrize("kind", ["group", "cogroup", "str_group"])
@pytest.mark.parametrize("M,R", [(2, 5), (7, 2), (1, 1)])
def test_ranks_that_map_or_receive_nothing(sc, kind, M, R):
    """W = 3: with M = 2 rank 0 maps nothing, with R = 2 rank 2 owns no partition, with M = R = 1 both."""
    rng = np.random.default_rng(M * 10 + R)
    n = 3000
    s = kind == "str_group"
    keys = str_keys(n, 200, rng) if s else int_keys(n, 300, rng)
    vals = values("nul", n, rng)
    agg = L.VB_AGG_COGROUP if kind == "cogroup" else L.VB_AGG_GROUP
    check_groups(one_process(sc, s, agg, M, R, keys, vals), ranks(sc, s, agg, 3, M, R, keys, vals), R, s)


def test_world_one_is_the_one_process_shuffle(sc):
    rng = np.random.default_rng(1)
    keys, vals = int_keys(2000, 100, rng), values("small", 2000, rng)
    check_groups(one_process(sc, False, L.VB_AGG_GROUP, 4, 5, keys, vals), ranks(sc, False, L.VB_AGG_GROUP, 1, 4, 5, keys, vals), 5, False)


# ---- cogroup and joins of dist bytes shuffles ---------------------------------------------------------------------------
def _gather(sh, refs, valid=None):
    """Values of a side: gathered bytes for a bytes side (None where invalid), the u64 itself for a u64 side."""
    if sh.vcode == L.VB_BYTES:
        return list(sh.gather(refs, valid))
    v = np.asarray(refs).view(np.uint64).tolist()
    return v if valid is None else [x if ok else None for x, ok in zip(v, np.asarray(valid).tolist())]


def _u64_side(sc, s, agg, W, M, R, keys, vals):
    """A dist shuffle of u64 values through the same harness (CudaEngine's or StrCudaEngine's export / import), and its
    one-process twin."""
    eng = vdist.StrCudaEngine(sc) if s else vdist.CudaEngine(sc)
    export, import_ = (vdist._str_export, vdist._str_import) if s else (vdist._rows_export, vdist._rows_import)
    starts = vb.slice_starts(len(vals), M)
    shs = [eng.create(M, R, L.VB_U64, agg, r, W) if s else eng.create(M, R, L.VB_U64, L.VB_U64, agg, r, W) for r in range(W)]
    for r, sh in enumerate(shs):
        lo, hi = vdist.map_block(r, W, M)
        for m in range(lo, hi):
            eng.map(sh, m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]])
    recv = MR.swap_columns([export(eng, sh, W) for sh in shs])
    for sh, (cols, splits) in zip(shs, recv):
        import_(eng, sh, cols, splits)
    for sh in shs:
        eng.seal(sh)
    if s:
        one, kc = vb.StrShuffle(sc, M, R, L.VB_U64, agg), _StrCol(vb.StrKeys.from_strs(keys))
    else:
        one, kc = vb.Shuffle(sc, M, R, L.VB_U64, L.VB_U64, agg), _Col(keys)
    for m in range(M):
        one.map(m, kc, _Col(vals, role="value"), int(starts[m]), int(starts[m + 1]))
    one.seal()
    return one, shs


def _sides(sc, s, W, specs, R):
    """specs: per side (keys, values, is_bytes) -> (one-process sides, per rank the dist sides)."""
    agg = L.VB_AGG_GROUP if s else L.VB_AGG_COGROUP
    ones, dists = [], []
    for j, (keys, vals, is_bytes) in enumerate(specs):
        M = 3 + 2 * j
        if is_bytes:
            ones.append(one_process(sc, s, agg, M, R, keys, vals))
            dists.append(ranks(sc, s, agg, W, M, R, keys, vals))
        else:
            o, d = _u64_side(sc, s, agg, W, M, R, keys, vals)
            ones.append(o)
            dists.append(d)
    return ones, [[d[r] for d in dists] for r in range(W)]


def _cogroup(sc, shs, r, s):
    if s:
        ks, sides, _ = cogroup_part(sc, shs, r)
        ks = [k.encode("utf-8", "surrogateescape") for k in ks]
    else:
        k, offs, vals = abi_cogroup_n(sc, shs, r)
        ks = k.tolist()
        sides = list(zip(offs, vals))
    out = {}
    for i, key in enumerate(ks):
        out[key] = tuple(tuple(_gather(sh, v[int(o[i]):int(o[i + 1])])) for sh, (o, v) in zip(shs, sides))
    return out


def _join(sc, shs, r, mask, s):
    if s:
        ks, ro, vs, oks, _, _ = join_part(sc, shs, r, mask)
        ro = np.asarray(ro).astype(np.int64)
        keys = [k.encode("utf-8", "surrogateescape") for i, k in enumerate(ks) for _ in range(ro[i + 1] - ro[i])]
    else:
        k, vs, oks = abi_outer(sc, shs, r, mask)
        keys = k.tolist()
    cols = [_gather(sh, v, ok) for sh, v, ok in zip(shs, vs, oks)]
    return sorted(zip(keys, *cols), key=repr)


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("s", [False, True], ids=["int", "str"])
@pytest.mark.parametrize("n_sides,mixed", [(2, False), (3, False), (2, True), (3, True)])
def test_cogroup_and_joins_match_one_process(sc, W, s, n_sides, mixed):
    """N-way cogroup, inner, left, right and full outer joins of dist bytes sides (with mixed, side 1 holds u64
    values), every rank against the one-process sides.  Sides overlap in part, so outer joins have None slots."""
    rng = np.random.default_rng(W * 7 + n_sides + 100 * mixed + 1000 * s)
    R = 6
    specs = []
    for j in range(n_sides):
        n = 1500 + 500 * j
        keys = str_keys(n, 300 + 150 * j, rng) if s else int_keys(n, 300 + 150 * j, rng)
        is_bytes = not (mixed and j == 1)
        specs.append((keys, values("nul" if j % 2 else "small", n, rng) if is_bytes else rng.integers(0, 1 << 63, n).astype(np.uint64),
                      is_bytes))
    ones, per_rank = _sides(sc, s, W, specs, R)
    full = (1 << n_sides) - 1
    masks = [full, 1, 2, 0] if n_sides == 2 else [full, 1, 0, 5]
    for r in range(R):
        shs = per_rank[r % W]
        assert _cogroup(sc, shs, r, s) == _cogroup(sc, ones, r, s), f"cogroup of partition {r}"
        for mask in masks:
            assert _join(sc, shs, r, mask, s) == _join(sc, ones, r, mask, s), f"join of partition {r}, required {mask:#x}"
        for d in range(W):
            if d != r % W:
                assert not _cogroup(sc, per_rank[d], r, s), f"rank {d} holds partition {r}"


# ---- errors and references ----------------------------------------------------------------------------------------------
def _maps(eng, sh, W, M, keys, vals):
    starts = vb.slice_starts(len(vals), M)
    lo, hi = vdist.map_block(sh.rank, W, M)
    for m in range(lo, hi):
        eng.map(sh, m, keys[starts[m]:starts[m + 1]], vals[starts[m]:starts[m + 1]])


def test_error_codes(sc):
    lib, h = sc._lib, ctypes.c_void_p()
    for agg in (L.VB_AGG_SUM, L.VB_AGG_MIN, L.VB_AGG_MAX, L.VB_AGG_COUNT):
        assert lib.vb_shuffle_create_bytes_dist(sc._h, 0, 2, 2, L.VB_U64, agg, 0, 0, 2, ctypes.byref(h)) == L.VB_ERR_UNSUPPORTED
    for rank, world in ((2, 2), (0, 0), (0, 257)):
        assert lib.vb_shuffle_create_bytes_dist(sc._h, 0, 2, 2, L.VB_U64, L.VB_AGG_GROUP, 0, rank, world, ctypes.byref(h)) == L.VB_ERR_INVALID
        assert lib.vb_shuffle_create_str_bytes_dist(sc._h, 0, 2, 2, rank, world, ctypes.byref(h)) == L.VB_ERR_INVALID
        assert lib.vb_shuffle_create_str_sort_bytes_dist(sc._h, 0, 2, 2, rank, world, ctypes.byref(h)) == L.VB_ERR_INVALID
    rng = np.random.default_rng(5)
    keys, vals = int_keys(400, 50, rng), values("small", 400, rng)
    eng = vdist.BytesCudaEngine(sc)
    W, M, R = 2, 4, 3
    cnt, nvb = (ctypes.c_uint64 * W)(), (ctypes.c_uint64 * W)()
    p = ctypes.c_void_p()
    # world 1, a sort, and a plain bytes shuffle
    one = eng.create(M, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, 0, 1)
    assert lib.vb_shuffle_export_bytes_prepare(one._h, cnt, nvb) == L.VB_ERR_STATE
    srt = eng.create(M, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_SORT, 0, W)
    assert lib.vb_shuffle_export_bytes_prepare(srt._h, cnt, nvb) == L.VB_ERR_UNSUPPORTED
    plain = vb.Shuffle(sc, M, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP)
    assert lib.vb_shuffle_export_bytes_prepare(plain._h, cnt, nvb) == L.VB_ERR_INVALID
    strsh = vdist.StrBytesCudaEngine(sc).create(M, R, L.VB_BYTES, L.VB_AGG_GROUP, 0, W)
    assert lib.vb_shuffle_export_bytes_prepare(strsh._h, cnt, nvb) == L.VB_ERR_INVALID
    # the calls that stay refused on a bytes dist shuffle
    shs = [eng.create(M, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_COGROUP, r, W) for r in range(W)]
    a = shs[0]
    assert lib.vb_shuffle_exchange(a._h, L.VB_XCHG_P2P) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_exchange(a._h, L.VB_XCHG_AUTO) == L.VB_ERR_STATE            # no communicator
    assert lib.vb_shuffle_set_dist(a._h, 0, 2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_prepare(a._h, cnt) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_counts(a._h, cnt) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_direct(a._h, cnt, cnt) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_import_arena(a._h, cnt) == L.VB_ERR_UNSUPPORTED
    blob = np.zeros(1, dtype=np.uint64)
    assert lib.vb_shuffle_map_blob(a._h, 0, blob.ctypes.data, 8, L.VB_HOST) == L.VB_ERR_UNSUPPORTED
    # import before export, seal without import
    zero = (ctypes.c_uint64 * W)()
    assert lib.vb_shuffle_import_bytes(a._h, None, None, None, zero, zero) == L.VB_ERR_STATE
    for sh in shs:
        _maps(eng, sh, W, M, keys, vals)
    exports = [vdist._bytes_export(eng, sh, W) for sh in shs]
    assert lib.vb_shuffle_seal(a._h) == L.VB_ERR_STATE
    # map after export
    offs = np.array([0, 1], dtype=np.uint64)
    one_key, one_byte = np.array([1], dtype=np.uint64), np.frombuffer(b"x", dtype=np.uint8)
    assert lib.vb_shuffle_map_bytes(a._h, 0, one_key.ctypes.data, offs.ctypes.data, one_byte.ctypes.data, 1, 1, L.VB_HOST) == L.VB_ERR_STATE
    recv = MR.swap_columns(exports)
    (k, ln, by), (c0, _, b0) = recv[0]
    arr = lambda xs: (ctypes.c_uint64 * W)(*xs)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    torch.cuda.synchronize()
    # too many rows, NULL columns, lengths that do not add up: refused, nothing kept
    assert lib.vb_shuffle_import_bytes(a._h, None, None, None, arr([0xFFFFFFFE, 0]), zero) == L.VB_ERR_TOO_LARGE
    assert sum(c0) and sum(b0)
    assert lib.vb_shuffle_import_bytes(a._h, None, ptr(ln), ptr(by), arr(c0), arr(b0)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_import_bytes(a._h, ptr(k), ptr(ln), None, arr(c0), arr(b0)) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_import_bytes(a._h, ptr(k), ptr(ln), ptr(by), arr(c0), arr([b0[0] + 1, b0[1]])) == L.VB_ERR_INVALID
    bad = ln.clone()
    bad[0] += 1
    torch.cuda.synchronize()
    assert lib.vb_shuffle_import_bytes(a._h, ptr(k), ptr(bad), ptr(by), arr(c0), arr(b0)) == L.VB_ERR_INVALID
    # the correct import still succeeds; a second one is refused
    vdist._bytes_import(eng, a, *recv[0])
    assert lib.vb_shuffle_import_bytes(a._h, ptr(k), ptr(ln), ptr(by), arr(c0), arr(b0)) == L.VB_ERR_STATE
    vdist._bytes_import(eng, shs[1], *recv[1])
    for sh in shs:
        eng.seal(sh)
        sh.as_str = False
    assert lib.vb_shuffle_import_bytes(shs[1]._h, None, None, None, zero, zero) == L.VB_ERR_STATE   # after seal
    check_groups(one_process(sc, False, L.VB_AGG_COGROUP, M, R, keys, vals), shs, R, False)
    # references: map-time ones are refused after the exchange, received ones gather
    nb = ctypes.c_uint64()
    for sh in shs:
        mapped = np.array([(vdist.map_block(sh.rank, W, M)[0] + 1) << 32], dtype=np.uint64)
        assert lib.vb_shuffle_gather_bytes_size(sh._h, mapped.ctypes.data, 1, L.VB_HOST, ctypes.byref(nb)) == L.VB_ERR_INVALID
        got = np.array([(M + 1) << 32], dtype=np.uint64)
        L.check(lib.vb_shuffle_gather_bytes_size(sh._h, got.ctypes.data, 1, L.VB_HOST, ctypes.byref(nb)))


def test_str_error_codes(sc):
    lib = sc._lib
    rng = np.random.default_rng(6)
    keys, vals = str_keys(500, 60, rng), values("nul", 500, rng)
    eng = vdist.StrBytesCudaEngine(sc)
    W, M, R = 2, 3, 4
    cs = [(ctypes.c_uint64 * W)() for _ in range(4)]
    one = eng.create(M, R, L.VB_BYTES, L.VB_AGG_GROUP, 0, 1)
    assert lib.vb_shuffle_export_str_bytes_prepare(one._h, *cs) == L.VB_ERR_STATE
    srt = eng.create(M, R, L.VB_BYTES, L.VB_AGG_SORT, 0, W)
    assert lib.vb_shuffle_export_str_bytes_prepare(srt._h, *cs) == L.VB_ERR_UNSUPPORTED
    intsh = vdist.BytesCudaEngine(sc).create(M, R, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, 0, W)
    assert lib.vb_shuffle_export_str_bytes_prepare(intsh._h, *cs) == L.VB_ERR_INVALID
    shs = [eng.create(M, R, L.VB_BYTES, L.VB_AGG_GROUP, r, W) for r in range(W)]
    a = shs[0]
    zero = (ctypes.c_uint64 * W)()
    assert lib.vb_shuffle_import_str_bytes(a._h, None, None, None, None, None, zero, zero, zero, zero) == L.VB_ERR_STATE
    assert lib.vb_shuffle_exchange(a._h, L.VB_XCHG_P2P) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_str_prepare(a._h, *cs[:3]) == L.VB_ERR_UNSUPPORTED
    for sh in shs:
        _maps(eng, sh, W, M, keys, vals)
    recv = MR.swap_columns([vdist._str_bytes_export(eng, sh, W) for sh in shs])
    assert lib.vb_shuffle_seal(a._h) == L.VB_ERR_STATE
    cols, splits = recv[0]
    arr = lambda xs: (ctypes.c_uint64 * W)(*xs)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    ns = [arr(splits[i]) for i in (0, 1, 3, 4)]
    assert sum(splits[3]) and sum(splits[4])
    bad = cols[3].clone()
    bad[-1] += 2
    torch.cuda.synchronize()
    assert lib.vb_shuffle_import_str_bytes(a._h, *[ptr(c) for c in cols[:3]], ptr(cols[3]), None, *ns) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_import_str_bytes(a._h, *[ptr(c) for c in cols[:3]], ptr(bad), ptr(cols[4]), *ns) == L.VB_ERR_INVALID
    vdist._str_bytes_import(eng, a, cols, splits)
    assert lib.vb_shuffle_import_str_bytes(a._h, *[ptr(c) for c in cols], *ns) == L.VB_ERR_STATE
    vdist._str_bytes_import(eng, shs[1], *recv[1])
    for sh in shs:
        eng.seal(sh)
        sh.as_str = False
    check_groups(one_process(sc, True, L.VB_AGG_GROUP, M, R, keys, vals), shs, R, True)


def test_received_store_beyond_4_gib(sc):
    """W = 2, one key and one partition: rank 0 receives every value, 4.4 GB in all, into one store whose 64-bit offsets
    must gather the values back exactly, in map-id order."""
    lib = sc._lib
    n, M, W = 4200, 6, 2
    lens = torch.full((n,), 1 << 20, dtype=torch.int64, device="cuda") + (torch.arange(n, device="cuda") * 37) % 1000
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    total = int(offs[-1])
    assert total > 1 << 32
    data = torch.randint(0, 256, (total,), dtype=torch.uint8, device="cuda")
    keys = torch.full((n,), 42, dtype=torch.int64, device="cuda")
    eng = vdist.BytesCudaEngine(sc)
    shs = [eng.create(M, 1, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, r, W) for r in range(W)]
    starts = vb.slice_starts(n, M)
    for sh in shs:
        lo, hi = vdist.map_block(sh.rank, W, M)
        for m in range(lo, hi):
            a, b = int(starts[m]), int(starts[m + 1])
            col = vb.StrKeys(offs[a:b + 1], data)
            sh.map(m, _Col(keys[a:b]), _BytesCol(col), 0, b - a)
    recv = MR.swap_columns([vdist._bytes_export(eng, sh, W) for sh in shs])
    for sh, (cols, splits) in zip(shs, recv):
        vdist._bytes_import(eng, sh, cols, splits)
        del cols
    del recv
    for sh in shs:
        eng.seal(sh)
    nk, nv = shs[0].reduce_size(0)
    assert (nk, nv) == (1, n) and shs[1].reduce_size(0) == (0, 0)
    k, o, refs = np.empty(1, dtype=np.uint64), np.empty(2, dtype=np.uint64), np.empty(n, dtype=np.uint64)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    L.check(lib.vb_shuffle_reduce(shs[0]._h, 0, p(k), None, p(o), p(refs), L.VB_HOST))
    nb = ctypes.c_uint64()
    L.check(lib.vb_shuffle_gather_bytes_size(shs[0]._h, p(refs), n, L.VB_HOST, ctypes.byref(nb)))
    assert nb.value == total
    go = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    gb = torch.empty(total, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    L.check(lib.vb_shuffle_gather_bytes(shs[0]._h, p(refs), n, L.VB_HOST, ctypes.c_void_p(go.data_ptr()),
                                        ctypes.c_void_p(gb.data_ptr()), L.VB_DEVICE))
    assert torch.equal(go, offs) and torch.equal(gb, data)
