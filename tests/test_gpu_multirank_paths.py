"""The multi-rank shuffle (set_dist, export_prepare / export_buffers, import, seal) at 2 to 256 ranks in one process.

Every rank is its own shuffle in one context; tests/multirank.py swaps the exported slices with torch.cat (source-rank
major, as the all-to-all-v does) and seals every rank.  So the seal-side code runs on real device buffers: the export
merge of every map-side path and the split by destination rank, then the seal's merge of imported accumulators (K_MERGE
over order-transformed values) or its grouping of imported rows.  Each case checks that partition r has rows only on
rank r % W and that the owners' union equals the single-process oracle for the same map tasks: the answer must not
depend on W.  Integer ops, COUNT and f64 MIN/MAX are compared bit for bit, f64 SUM with tests/util.py:assert_f64_sums
(bit-exact in the exact and subnormal modes), group value lists in order.  Path cases assert the statistic that proves
the path ran, read after the export and before the seal, whose import merge adds launches of its own."""
import ctypes

import numpy as np
import pytest

import vega_b200 as vb
from tests import cogroup_n_ref as CN
from tests import join_n_outer_ref as JO
from tests.multirank import all_to_all_v, group_dict, maps_by_rank, owned_parts, run_ranks
from tests.test_gpu_cogroup import abi_cogroup, part_dict
from tests.test_gpu_cogroup_n import abi_cogroup_n, abi_join_n, join_by_key, part_dict_n
from tests.test_gpu_join_n_outer import abi_outer, rows_by_key
from tests.test_gpu_outer_join import abi_rows, by_key
from tests.test_gpu_reduce_paths import AGG, CODE, OP_IDS, OPS, _col, _dev, check_reduce
from tests.util import assert_parts_equal, oracle_group, rand_pairs
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from vega_b200.rdd import Shuffle, StrShuffle

pytestmark = pytest.mark.gpu
AGG = dict(AGG, group=L.VB_AGG_GROUP)


@pytest.fixture(scope="module")
def eng():
    sc = vb.Context(0)
    yield vdist.CudaEngine(sc)
    sc.close()


# ---- map task placement: place(map_id, lo, hi) -> (keys, vals) for CudaEngine.map -------------------------------------
def host(keys, vals, vcode=None):
    return lambda m, lo, hi: (keys[lo:hi], None if vals is None else vals[lo:hi])


def device(keys, vals, vcode):
    """Each map task its own (16-byte aligned) torch CUDA columns: borrowed by the library."""
    return lambda m, lo, hi: (_col(_dev(keys[lo:hi]), L.VB_U64), None if vals is None else _col(_dev(vals[lo:hi]), vcode))


def aos(keys, vals, vcode):
    """Each map task its own device (n, 2) rows; COUNT rows carry their value column anyway."""
    v = np.zeros(len(keys), np.uint64) if vals is None else np.ascontiguousarray(vals).view(np.uint64)
    return lambda m, lo, hi: (_col(_dev(np.stack([keys[lo:hi], v[lo:hi]], axis=1)), vcode, rows=True), None)


PLACE = {"host": host, "device": device, "aos": aos}


def shuffle_ranks(eng, W, op, vdt, keys, vals, M, R, place="host", key_width=8, hint=0, maps=None):
    """One shuffle over W ranks -> (owners' partitions, stats after export, stats after seal) of every rank."""
    vcode = CODE[vdt]
    if maps is None:
        maps = maps_by_rank(len(keys), M, W, PLACE[place](keys, None if op == "count" else vals, vcode))
    shs, pre = run_ranks(eng, W, AGG[op], maps, R, L.VB_U64, vcode, key_width=key_width, hint=hint, n_map=M)
    try:
        parts = owned_parts(eng, shs, R)
        post = [sh.stats() for sh in shs]
    finally:
        for sh in shs:
            sh.free()
    return parts, pre, post


def check(parts, op, vdt, mode, keys, vals, M, R, key_width=8):
    if len(keys) == 0:
        assert all(len(p[0]) == 0 for p in parts)
    elif op == "group":
        assert_parts_equal([group_dict(*p) for p in parts], oracle_group(keys, vals, M, R, key_width=key_width))
    else:
        check_reduce(parts, op, vdt, mode, keys, vals, R, key_width=key_width)


# ---- 1. every reduce op on every map-side path, at three ranks ---------------------------------------------------------
# name: (rows, keys, hot-key share, R, M, placement, hint); every rank runs the path on its block of M / 3 map tasks
PATHS = {
    "register_small": (150_000, 20_000, 0.0, 7, 3, "host", 0),          # one host task of 50k rows per rank: below 65,536
    "bulk_soa_tail": (3 * 102_979, 50_000, 0.0, 7, 3, "device", 0),     # one device task per rank, n % 1024 = 579
    "bulk_aos": (6 * 70_001, 50_000, 0.0, 5, 6, "aos", 0),              # two device AoS tasks per rank
    "hot_key_cache": (3_000_000, 100_000, 0.12, 7, 3, "device", 0),     # one task of 1M rows per rank, top key 12 %
    "per_map_merge": (400_000, 100_000, 0.0, 7, 12, "host", 0),         # four host tasks per rank: per-map tables merged
    "shared_borrowed": (12 * 70_001, 100_000, 0.0, 7, 12, "device", 0),  # four device tasks per rank: one shared table
    "restart_per_map": (300_000, 120_000, 0.0, 7, 6, "host", 100),      # hint=100: per-map tables and the import restart
    "restart_shared": (300_000, 120_000, 0.0, 7, 12, "device", 100),    # hint=100: the shared table and the import restart
}


def _assert_path(path, pre, post):
    for st, after in zip(pre, post):
        if path == "register_small":
            assert st["hot_kernel_variant"] == 0
        elif path in ("bulk_soa_tail", "bulk_aos", "hot_key_cache"):
            assert st["hot_kernel_variant"] == 1
        elif path == "per_map_merge":
            assert st["kernels"]["merge"]["launches"] >= 1
        elif path == "shared_borrowed":
            assert st["hot_kernel_variant"] == 1 and st["kernels"]["merge"]["launches"] == 0
        else:
            assert st["table_restarts"] >= 1
            assert after["table_restarts"] > st["table_restarts"], "the import merge did not restart"


@pytest.mark.parametrize("i_op", range(len(OPS)), ids=OP_IDS)
@pytest.mark.parametrize("path", list(PATHS))
def test_reduce_path_across_three_ranks(eng, path, i_op):
    op, vdt, mode = OPS[i_op]
    n, nkeys, hot, R, M, place, hint = PATHS[path]
    rng = np.random.default_rng([list(PATHS).index(path), i_op, 3])
    keys, vals = rand_pairs(rng, n, nkeys, vdt or "u64", values=mode, hot=hot)
    parts, pre, post = shuffle_ranks(eng, 3, op, vdt, keys, vals, M, R, place, hint=hint)
    _assert_path(path, pre, post)
    check(parts, op, vdt, mode, keys, vals, M, R)


@pytest.mark.parametrize("i_op", range(len(OPS)), ids=OP_IDS)
def test_partition_first_on_one_of_two_ranks(eng, i_op):
    """Rank 0 maps (1<<22)+5 device rows with hint=3e6 (the partition-first build of a 2^23-slot table), rank 1 a small
    host slice."""
    op, vdt, mode = OPS[i_op]
    big, small = (1 << 22) + 5, 20_000
    rng = np.random.default_rng([i_op, 22])
    keys, vals = rand_pairs(rng, big + small, 300_000, vdt or "u64", values=mode)
    v = None if op == "count" else vals
    maps = [[(0, *device(keys, v, CODE[vdt])(0, 0, big))], [(1, *host(keys, v)(1, big, big + small))]]
    parts, pre, _ = shuffle_ranks(eng, 2, op, vdt, keys, vals, 2, 7, hint=3_000_000, maps=maps)
    assert pre[0]["table_slots"] >= 1 << 23
    check(parts, op, vdt, mode, keys, vals, 2, 7)


# ---- 2. world shapes -----------------------------------------------------------------------------------------------------
WOPS = [("sum", "u64", "full"), ("min", "f64", "special"), ("sum", "f64", "cancel"), ("count", None, "full"),
        ("group", "u64", "full")]
WOP_IDS = [f"{op}-{vdt or 'keys'}-{mode}" for op, vdt, mode in WOPS]
# name: (W, M, R, rows, keys)
SHAPES = {
    "w2": (2, 4, 7, 60_000, 8000),
    "w5_m7": (5, 7, 11, 60_000, 8000),           # M not a multiple of W
    "w8": (8, 16, 13, 60_000, 8000),
    "w256": (256, 300, 300, 120_000, 20_000),     # the largest world set_dist takes; some ranks map two tasks
    "m_lt_w": (8, 3, 13, 30_000, 4000),           # ranks without a map task export nothing
    "r_lt_w": (8, 8, 3, 30_000, 4000),            # ranks 3..7 own no partition and import zero rows (NULL buffers)
    "r1": (3, 4, 1, 40_000, 6000),                # R <= 256: the unordered table split of the finalize
    "r255": (3, 4, 255, 40_000, 6000),
    "r256": (3, 4, 256, 40_000, 6000),
    "r257": (3, 4, 257, 40_000, 6000),            # R > 256: the ordered two-pass split
    "r1000": (3, 4, 1000, 40_000, 6000),
    "key_width_4": (3, 5, 7, 40_000, 3000),       # i32 keys widened to 64 bits: destination from the 4-byte hash
    "one_key": (4, 6, 5, 40_000, 1),              # every row one key
    "empty": (3, 2, 5, 0, 0),                     # no rows at all
}


def _shape_data(shape, i_op):
    W, M, R, n, nkeys = SHAPES[shape]
    op, vdt, mode = WOPS[i_op]
    rng = np.random.default_rng([list(SHAPES).index(shape), i_op, 5])
    keys, vals = rand_pairs(rng, n, nkeys, vdt or "u64", values=mode)
    key_width = 8
    if shape == "key_width_4":
        k32 = rng.integers(-nkeys, nkeys, n).astype(np.int32)
        k32[rng.choice(n, 400, replace=False)] = np.resize(np.array([-1, -(1 << 31), (1 << 31) - 1, 0], np.int32), 400)
        keys, key_width = k32.astype(np.int64).view(np.uint64), 4
    elif shape == "one_key":
        keys[:] = keys[0]
    return W, M, R, keys, vals, key_width


@pytest.mark.parametrize("i_op", range(len(WOPS)), ids=WOP_IDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_world_shapes(eng, shape, i_op):
    op, vdt, mode = WOPS[i_op]
    W, M, R, keys, vals, key_width = _shape_data(shape, i_op)
    parts, pre, _ = shuffle_ranks(eng, W, op, vdt, keys, vals, M, R, key_width=key_width)
    for r, st in enumerate(pre):
        lo, hi = vdist.map_block(r, W, M)
        assert (st["rows_in"] == 0) == (lo == hi or len(keys) == 0)
    check(parts, op, vdt, mode, keys, vals, M, R, key_width=key_width)


def test_world_above_256_is_refused(eng):
    sh = Shuffle(eng.sc, 1, 4, L.VB_U64, L.VB_U64, L.VB_AGG_SUM)
    for rank, world in ((0, 257), (256, 256), (0, 0), (0, (1 << 32) - 1)):
        assert eng.sc._lib.vb_shuffle_set_dist(sh._h, rank, world) == L.VB_ERR_INVALID, (rank, world)
    assert eng.sc._lib.vb_shuffle_set_dist(sh._h, 255, 256) == L.VB_OK
    sh.free()


# ---- 3. group_by_key over imported rows ----------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [3, 8])
def test_group_device_rows_on_some_ranks_host_rows_on_others(eng, W):
    rng = np.random.default_rng(W)
    n, M, R = 200_000, 2 * W + 1, 9
    keys, vals = rand_pairs(rng, n, 30_000, values="full")
    dev_rows, host_cols = aos(keys, vals, L.VB_U64), host(keys, vals)
    owner = lambda m: next(r for r in range(W) if m < vdist.map_block(r, W, M)[1])
    maps = maps_by_rank(n, M, W, lambda m, lo, hi: (dev_rows if owner(m) % 2 else host_cols)(m, lo, hi))
    parts, _, _ = shuffle_ranks(eng, W, "group", "u64", keys, vals, M, R, maps=maps)
    check(parts, "group", "u64", "full", keys, vals, M, R)


def test_group_dictionary_of_imported_rows_restarts(eng):
    rng = np.random.default_rng(11)
    n, M, R = 150_000, 5, 6
    keys, vals = rand_pairs(rng, n, 60_000, values="full")
    parts, pre, post = shuffle_ranks(eng, 3, "group", "u64", keys, vals, M, R, place="device", hint=1)
    assert all(b["table_restarts"] > a["table_restarts"] for a, b in zip(pre, post))
    check(parts, "group", "u64", "full", keys, vals, M, R)


# ---- 4. cogroup and joins of imported sides -------------------------------------------------------------------------------
def cogroup_ranks(eng, W, sides, R):
    """One COGROUP shuffle per side [(keys, vals, M)] over W ranks -> shs[rank] = [the rank's shuffle of every side]."""
    per_side = []
    for j, (k, v, M) in enumerate(sides):
        place = (host if j % 2 else device)(k, v, L.VB_U64)
        shs, _ = run_ranks(eng, W, L.VB_AGG_COGROUP, maps_by_rank(len(k), M, W, place), R, L.VB_U64, L.VB_U64, n_map=M)
        per_side.append(shs)
    return [list(x) for x in zip(*per_side)]


def across_ranks(W, R, call):
    """call(rank, r) -> {key: ...} of partition r on that rank: keys only on the owner r % W; returns the owners'."""
    out = []
    for r in range(R):
        for d in range(W):
            got = call(d, r)
            if d == r % W:
                out.append(got)
            else:
                assert got == {}, f"rank {d} has {len(got)} keys of partition {r}, owned by rank {r % W}"
    return out


@pytest.mark.parametrize("empty_side", [False, True])
def test_cogroup_and_joins_of_imported_sides(eng, empty_side):
    W, R = 3, 7
    rng = np.random.default_rng(int(empty_side))
    sides = []
    for j, (rows, M) in enumerate(((9000, 4), (6000, 3), (4500, 5))):
        k, v = rand_pairs(rng, rows, 3000, values="full")        # keys 0 and 2^64-1 among them
        keep = (k >> np.uint64(7)) % np.uint64(4) != np.uint64(j)  # a quarter of the keys lack side j
        k, v = k[keep], v[keep]
        if empty_side and j == 1:
            k, v = k[:0], v[:0]
        sides.append((k, v, M))
    sc = eng.sc
    shs = cogroup_ranks(eng, W, sides, R)
    try:
        ref3, ref2 = CN.ref_parts_n(sides, R), CN.ref_parts_n(sides[:2], R)
        got = across_ranks(W, R, lambda d, r: part_dict(*abi_cogroup(sc, *shs[d][:2], r), r, R))
        assert_parts_equal(got, ref2)
        for mask, kind in ((0b11, None), (0b01, "left"), (0b10, "right"), (0b00, "full")):
            got = across_ranks(W, R, lambda d, r: by_key(*abi_rows(sc, *shs[d][:2], r, kind)))
            assert_parts_equal(got, JO.outer_of_parts(ref2, mask))
        got = across_ranks(W, R, lambda d, r: part_dict_n(*abi_cogroup_n(sc, shs[d], r), r, R))
        assert_parts_equal(got, ref3)
        got = across_ranks(W, R, lambda d, r: join_by_key(*abi_join_n(sc, shs[d], r)))
        assert_parts_equal(got, CN.join_of_parts(ref3))
        for mask in range(8):
            got = across_ranks(W, R, lambda d, r: rows_by_key(*abi_outer(sc, shs[d], r, mask)))
            assert_parts_equal(got, JO.outer_of_parts(ref3, mask))
        assert sum(len(d) for d in JO.outer_of_parts(ref3, 0)) > 0
    finally:
        for rank in shs:
            for sh in rank:
                sh.free()


# ---- 5. a resubmitted map task -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i_op", [0, 8, 11], ids=[OP_IDS[i] for i in (0, 8, 11)])
def test_resubmitted_borrowed_map_task(eng, i_op):
    """Rank 1 first submits its first map task with other rows, then the real ones: the stale rows are already in
    the rank's shared table, which the export has to rebuild from the final inputs."""
    op, vdt, mode = OPS[i_op]
    W, M, R, n = 3, 6, 7, 240_000
    rng = np.random.default_rng([i_op, 9])
    keys, vals = rand_pairs(rng, n, 40_000, vdt or "u64", values=mode)
    sk, sv = rand_pairs(rng, 30_000, 5000, vdt or "u64", values=mode)
    v, stale_v = (None, None) if op == "count" else (vals, sv)
    maps = maps_by_rank(n, M, W, device(keys, v, CODE[vdt]))
    maps[1].insert(0, (maps[1][0][0], *device(sk, stale_v, CODE[vdt])(0, 0, len(sk))))
    parts, _, _ = shuffle_ranks(eng, W, op, vdt, keys, vals, M, R, maps=maps)
    check(parts, op, vdt, mode, keys, vals, M, R)


# ---- 6. phase errors -----------------------------------------------------------------------------------------------------
def _code(fn):
    with pytest.raises(vb.VegaB200Error) as e:
        fn()
    return e.value.code, str(e.value)


def test_phase_errors(eng):
    """Each out-of-order call returns its code and leaves the shuffle usable: the run then completes correctly."""
    sc, lib = eng.sc, eng.sc._lib
    rng = np.random.default_rng(12)
    keys, vals = rand_pairs(rng, 20_000, 3000, values="full")
    counts = (ctypes.c_uint64 * 2)()
    # export at world 1
    sh = Shuffle(sc, 1, 3, L.VB_U64, L.VB_U64, L.VB_AGG_SUM)
    eng.map(sh, 0, keys, vals)
    assert lib.vb_shuffle_export_prepare(sh._h, counts) == L.VB_ERR_STATE
    assert lib.vb_shuffle_export_counts(sh._h, counts) == L.VB_ERR_STATE
    sh.seal()
    check([sh.reduce(r) for r in range(3)], "sum", "u64", "full", keys, vals, 1, 3)
    sh.free()
    # two ranks of a GROUP shuffle, one call out of order at every phase
    W, M, R = 2, 4, 5
    maps = maps_by_rank(len(keys), M, W, host(keys, vals))
    shs = [eng.create(M, R, L.VB_U64, L.VB_U64, L.VB_AGG_GROUP, r, W) for r in range(W)]
    for r in range(W):
        for m, k, v in maps[r]:
            eng.map(shs[r], m, k, v)
    assert lib.vb_shuffle_import(shs[0]._h, None, None, (ctypes.c_uint64 * 2)()) == L.VB_ERR_STATE
    assert _code(lambda: shs[0].exchange())[0] == L.VB_ERR_STATE             # no communicator in this context
    assert _code(lambda: shs[0].seal())[0] == L.VB_ERR_STATE                  # seal before export
    exports = [eng.export(sh, W) for sh in shs]
    assert lib.vb_shuffle_export_prepare(shs[0]._h, counts) == L.VB_ERR_STATE    # export twice
    assert lib.vb_shuffle_export_counts(shs[0]._h, counts) == L.VB_ERR_STATE
    assert _code(lambda: eng.map(shs[1], maps[1][0][0], *maps[1][0][1:]))[0] == L.VB_ERR_STATE   # map after export
    recv = all_to_all_v(exports)
    assert _code(lambda: shs[1].seal())[0] == L.VB_ERR_STATE                  # seal without import
    for sh, rv in zip(shs, recv):
        eng.import_(sh, *rv)
    for sh in shs:
        eng.seal(sh)
    parts = owned_parts(eng, shs, R)
    check(parts, "group", "u64", "full", keys, vals, M, R)
    for sh in shs:
        sh.free()
    # shuffles the multi-rank exchange does not carry: several aggregates, string keys, sort_by_key
    multi = ([L.VB_U64], [(L.VB_AGG_SUM, 0), (L.VB_AGG_MAX, 0)])
    assert _code(lambda: Shuffle(sc, 1, 3, L.VB_U64, L.VB_U64, 0, multi=multi, rank=0, world=2))[0] == L.VB_ERR_UNSUPPORTED
    ssh = StrShuffle(sc, 1, 3, L.VB_U64, L.VB_AGG_SUM)
    assert lib.vb_shuffle_set_dist(ssh._h, 0, 2) == L.VB_ERR_UNSUPPORTED
    ssh.free()
    for fn in ("vb_shuffle_export_prepare", "vb_shuffle_export_counts"):
        sh = Shuffle(sc, 2, 3, L.VB_U64, L.VB_U64, L.VB_AGG_SORT, rank=0, world=2)
        eng.map(sh, 0, keys, vals)
        code, msg = _code(lambda: L.check(getattr(lib, fn)(sh._h, counts)))
        assert code == L.VB_ERR_UNSUPPORTED, fn
        if fn == "vb_shuffle_export_prepare":
            assert "vb_shuffle_exchange" in msg
        sh.free()
    # the context still runs a whole multi-rank shuffle
    parts, _, _ = shuffle_ranks(eng, 3, "sum", "u64", keys, vals, 4, 5)
    check(parts, "sum", "u64", "full", keys, vals, 4, 5)
