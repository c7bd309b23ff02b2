"""The integer hash table under keys built to collide (tests/slot_hash_ref.py), through every op that builds or probes it,
against the same exact references as the path tests.

Ordinary rand_pairs rows carry families of crafted keys: a chain of 512 keys that share one home bucket (128 full
buckets: half the HA_MAX_PROBE limit, because a probe round lost to a concurrent insert's CAS re-reads its bucket and
counts against the limit too), a chain homed in the last bucket that wraps to bucket 0 (where key 0 lives), three hot
keys at 5 % of the rows each whose two hot-key-cache slots are the same, and on the partition-first path keys homed in
the last bucket of every table region.  Joins probe the tables with absent keys that share a family's home bucket and
must walk the whole chain to miss.  So a probe that only works on well-spread keys fails here.

The random keys whose slot hash falls on or just before the chain at 2^16 slots are moved away (carve), so that the
chain needs exactly 128 buckets at every table size from 2^16 slots up.  Keys that need more than 256 buckets (1025 and
more sharing one home) must still fit in a table that cannot grow: those cases end the file."""
import numpy as np
import pytest

import vega_b200 as vb
from tests import group_ref as G
from tests import slot_hash_ref as S
from tests import test_gpu_combine as C
from tests import test_gpu_combine_multirank as CM
from tests import test_gpu_reduce_paths as RP
from tests.multirank import maps_by_rank, owned_parts, run_ranks
from tests.test_gpu_cogroup_n import shuffles
from tests.test_gpu_group_paths import check_join, cogroup_pair, exact_keys, full_i64, gpu_cogroup, place, run_group, sliced
from tests.test_gpu_narrow import check_sides, parent, result_rows, view
from tests.test_gpu_reduce_paths import _col, _dev, check_reduce, run_reduce
from tests.util import EMPTY_KEY, rand_pairs
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from vega_b200.rdd import _Col

pytestmark = pytest.mark.gpu

SAME_TOP = 0x0_AAAA_AAAA          # the chain's home: a third of the way into every table, away from region edges
CLASH_LOW = 0x3C5A7               # low 20 slot-hash bits of the cache-clash keys
CARVE_LOG = 16                    # the 512-key chain needs exactly 128 buckets at this table size and above
OPS = [("sum", "u64", "full"), ("min", "i64", "full"), ("max", "i64", "full"), ("min", "f64", "special"),
       ("max", "f64", "special")]
OP_IDS = [f"{op}-{vdt}" for op, vdt, _ in OPS]
TWO = ([("u64", "full"), ("f64", "special")], [("sum", 0), ("max", 0), ("min", 1), ("max", 1), ("count", 0)])


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def on_chain(keys):
    """Keys whose slot hash lies on the chain's 320 buckets at 2^16 slots, or 16 buckets before it (2^64-1 never:
    it takes the special slot)."""
    home = SAME_TOP >> (S.TOP - (CARVE_LOG - 2))
    sh = 64 - (CARVE_LOG - 2)
    h = S.slot_hash(keys)
    return (h >= np.uint64((home - 16) << sh)) & (h < np.uint64((home + 320) << sh)) & (keys != np.uint64(EMPTY_KEY))


def carve(keys):
    """keys with every key on_chain moved elsewhere."""
    keys = keys.copy()
    for salt in range(1, 64):
        bad = on_chain(keys)
        if not bad.any():
            return keys
        keys[bad] ^= np.uint64(0x5DEECE66D * salt)
    raise AssertionError("carve did not converge")


def families(rng, exclude, chain=512, region_log=None):
    """The crafted keys: {name: keys}."""
    f = {"chain": S.same_home(rng, chain, SAME_TOP, exclude)}
    f["wrap"] = S.wrap(rng, 64, np.concatenate([exclude, f["chain"]]))
    clash = S.cache_clash(rng, 8, CLASH_LOW, np.concatenate([exclude] + list(f.values())))
    f["clash"] = clash[~on_chain(clash)][:3]
    if region_log:
        f["edge"] = S.region_edge(rng, 16, region_log, np.concatenate([exclude] + list(f.values())))
    assert not any(on_chain(f[k]).any() for k in f if k != "chain")
    return f


def colliding(rng, keys, chain=512, region_log=None, hot_share=0.05, copies=3):
    """rand_pairs keys carved, then overwritten at random rows by the families: each cache-clash key on hot_share of
    the rows, every other family key on `copies` rows; keys 0 and 2^64-1 on two rows each."""
    keys = carve(keys)
    n = len(keys)
    fam = families(rng, keys, chain, region_log)
    pos = rng.permutation(n)
    at = 0
    for name, ks in fam.items():
        for k in ks.tolist():
            m = int(hot_share * n) if name == "clash" else copies
            keys[pos[at:at + m]] = np.uint64(k)
            at += m
    keys[pos[at:at + 4]] = np.array([0, 0, EMPTY_KEY, EMPTY_KEY], dtype=np.uint64)
    assert at + 4 <= n
    return keys, fam


# ---- the device hash is the numpy one ------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["same_home_1025", "same_home_256", "spread_1025"])
def test_device_hash_pins_the_chain_limit(sc, family):
    """1025 keys of one home bucket need a 257th bucket: the first table (2^12 slots, below the largest size 2^14)
    gives up and restarts at its largest size, where chains may run on.  256 such keys (64 buckets) and 1025 keys of
    random homes fit the first table.  If the numpy slot hash drifted from the device's, the same-home keys would
    spread and nothing would restart; if the limit shrank below about 64 buckets, the short chain would restart.  A
    longer short chain (the 1024 keys of a full 256-bucket chain) cannot be pinned: below the largest size a probe
    round lost to a concurrent CAS also counts against the 256-round limit, so such a chain may restart under
    contention."""
    rng = np.random.default_rng(len(family))
    n_same = int(family.rsplit("_", 1)[1])
    fam = S.same_home(rng, n_same, SAME_TOP) if family.startswith("same") else rng.integers(1, 1 << 63, n_same, dtype=np.uint64)
    keys = rng.permutation(np.concatenate([np.repeat(fam, 4), np.array([0, 0, EMPTY_KEY, EMPTY_KEY], np.uint64)]))
    vals = rng.integers(0, 1 << 64, len(keys), dtype=np.uint64)
    assert S.chain_model(np.concatenate([fam, np.zeros(1, np.uint64)]), 12)[0] == (family == "same_home_1025")
    parts, st = run_reduce(sc, "sum", "u64", _Col(keys), _Col(vals, role="value"), len(keys), 1, 7, hint=1000)
    if family == "same_home_1025":
        assert st["table_restarts"] >= 1 and st["table_slots"] == 1 << 14
    else:
        assert st["table_restarts"] == 0 and st["table_slots"] == 1 << 12
    check_reduce(parts, "sum", "u64", "full", keys, vals, 7)


# ---- reduce_by_key on every hash-aggregate path ---------------------------------------------------------------------
@pytest.mark.parametrize("i_op", range(len(OPS)), ids=OP_IDS)
@pytest.mark.parametrize("path", list(RP.PATHS))
def test_reduce_paths_with_colliding_keys(sc, path, i_op):
    op, vdt, mode = OPS[i_op]
    data = "hot_key_cache" if path == "register_hot" else path
    n, nkeys, hot, R = RP.PATHS[data]
    rng = np.random.default_rng([list(RP.PATHS).index(data), i_op, 51])
    keys, vals = rand_pairs(rng, n, nkeys, vdt, values=mode, hot=hot)
    region_log = 23 if path == "partition_first" else None
    # the hot paths' rows already have two hot keys: their cache-clash keys take 1 % of the rows each.  register_hot
    # gets no long chain: its register-staged kernel keeps the hot-key cache on, every CTA's cache holds chain keys, and
    # the CTAs' flushes at exit race on the chain's buckets until the shared table (which can still grow) gives up
    # and is rebuilt partition-first, off the path this case asserts
    keys, fam = colliding(rng, keys, chain=0 if path == "register_hot" else 512, region_log=region_log,
                          hot_share=0.01 if hot else 0.05)
    parts, st = RP._run_path(sc, path, op, vdt, keys, vals, n, R)
    if path == "partition_first":     # region edges at 2^23 slots stay region edges at 2^24, the size after a restart
        assert st["table_slots"] >= 1 << region_log
    check_reduce(parts, op, vdt, mode, keys, vals, R)


# ---- combine_by_key: the "four" spec and a two-column spec (NV = 2, register and bulk kernels) ----------------------
def _combine_data(rng, spec, n, nkeys, hot):
    dts = C.spec_of(spec)[0]
    lead = next(i for i, (d, _) in enumerate(dts) if d == "f64")
    keys, lead_vals = rand_pairs(rng, n, nkeys, dts[lead][0], values=dts[lead][1], hot=hot)
    cols = [lead_vals if i == lead else rand_pairs(rng, n, nkeys, d, values=m)[1] for i, (d, m) in enumerate(dts)]
    keys, _ = colliding(rng, keys)
    return keys, cols


@pytest.mark.parametrize("spec", ["four", "two"])
@pytest.mark.parametrize("path", list(C.PATHS))
def test_combine_paths_with_colliding_keys(sc, path, spec):
    sp = C.SPECS[spec] if spec == "four" else TWO
    data = "hot_key_cache" if path == "register_hot" else path
    n, nkeys, hot, _ = C.PATHS[data]
    rng = np.random.default_rng([list(C.PATHS).index(data), len(spec), 52])
    keys, cols = _combine_data(rng, sp, n, nkeys, hot)
    parts, R = C._run_path(sc, path, sp, keys, cols)
    C.check_combine(parts, sp, keys, cols, R)


# ---- group_by_key: the OPK_DICT dictionary, lists in map order -------------------------------------------------------
@pytest.mark.parametrize("where", ["host_soa", "dev_soa", "dev_soa_misaligned"])
def test_group_dictionary_with_colliding_keys(sc, where):
    rng = np.random.default_rng([len(where), 53])
    keys, _ = rand_pairs(rng, 300_000, 60_000)
    keys, _ = colliding(rng, keys, hot_share=0.01)
    vals = full_i64(rng, len(keys))
    M, R = (3, 7) if where == "host_soa" else (1, 7)
    kc, vc = place(where, keys, vals)
    parts, _ = run_group(sc, sliced(kc, vc, len(keys), M), R)
    G.assert_group_equal(parts, keys, vals, R)


# ---- joins and cogroup: table_find over full chains ------------------------------------------------------------------
def _join_sides(rng):
    """Right: random keys with the wrapped chain and the 512-key chain.  Left: random keys (half of them on the right),
    absent neighbours of both chains (miss after the whole chain), and 150 chain keys (some at its far end)."""
    kb = exact_keys(rng, 80_000, 50_000)
    kb, fam = colliding(rng, kb, hot_share=0.0)
    ka = exact_keys(rng, 90_000, 40_000, first_rank=25_000)
    ka = carve(ka)
    absent = np.concatenate([S.same_home(rng, 200, SAME_TOP, fam["chain"]), S.wrap(rng, 100, fam["wrap"])])
    far = rng.choice(fam["chain"], 150, replace=False)
    pos = rng.permutation(len(ka))
    ka[pos[:600]] = np.repeat(absent, 2)
    ka[pos[600:900]] = np.repeat(far, 2)
    assert not np.isin(absent, kb).any()
    return ka, full_i64(rng, len(ka)), kb, full_i64(rng, len(kb))


@pytest.mark.parametrize("order", ["lazy", "grouped"])
@pytest.mark.parametrize("kind", ["inner", "left", "full", "cogroup"])
def test_joins_probe_colliding_chains(sc, kind, order):
    """lazy inner / left: the left rows are filtered through a dictionary of the right keys (semi_probe_kernel);
    grouped: both sides are read first, and the join probes each side's own dictionary."""
    rng = np.random.default_rng([len(kind), len(order), 54])
    ka, va, kb, vb_ = _join_sides(rng)
    R = 7
    sa, sb = cogroup_pair(sc, ka, va, kb, vb_, R)
    try:
        if order == "grouped":
            for s_, k, v in ((sa, ka, va), (sb, kb, vb_)):
                G.assert_group_equal([s_.reduce(r) for r in range(R)], k, v, R)
        if kind == "cogroup":
            G.assert_cogroup_equal(gpu_cogroup(sc, sa, sb, R), ka, va, kb, vb_, R)
        else:
            check_join(sc, sa, sb, kind, ka, va, kb, vb_, R)
        if order == "lazy" and kind in ("inner", "left"):
            assert sa.stats()["kernels"]["join"]["launches"] >= 1
    finally:
        sa.free()
        sb.free()


# ---- narrow views: a reduce result with a 128-bucket chain as a join side (narrow_dict_kernel) ------------------------
def test_narrow_view_with_colliding_keys(sc):
    rng = np.random.default_rng(55)
    R = 1                                                     # one dictionary over every result key
    ka, va = rand_pairs(rng, 60_000, 30_000, values="full")
    ka, fam = colliding(rng, ka, hot_share=0.0)
    kc, vc = rand_pairs(rng, 20_000, 8000, values="full")
    kc = carve(kc)
    kc[:600] = np.repeat(np.concatenate([fam["chain"][-150:], S.same_home(rng, 150, SAME_TOP, fam["chain"])]), 2)
    pa = parent(sc, ka, va, 3, R, "sum")
    v = view(pa)
    check_sides(sc, [v, shuffles(sc, [(kc, vc, 2)], R)[0]], [(*result_rows(pa, R), 1), (kc, vc, 2)], R)
    assert v.stats()["table_slots"] >= 1 << CARVE_LOG


# ---- across ranks: the import merge builds a table from colliding keys ------------------------------------------------
@pytest.fixture(scope="module")
def eng(sc):
    return vdist.CudaEngine(sc)


@pytest.mark.parametrize("W", [2, 3])
def test_reduce_import_merge_with_colliding_keys(eng, W):
    rng = np.random.default_rng([W, 56])
    keys, vals = rand_pairs(rng, 200_000, 60_000, "i64", values="full")
    keys, _ = colliding(rng, keys)
    M, R = 4, 2 * W + 1
    for op in ("sum", "max"):
        maps = maps_by_rank(len(keys), M, W, lambda m, lo, hi: (keys[lo:hi], vals[lo:hi]))
        shs, _ = run_ranks(eng, W, RP.AGG[op], maps, R, L.VB_U64, L.VB_I64, n_map=M)
        try:
            parts = owned_parts(eng, shs, R)
        finally:
            for sh in shs:
                sh.free()
        check_reduce(parts, op, "i64", "full", keys, vals, R)


@pytest.mark.parametrize("W", [2, 3])
def test_combine_import_merge_with_colliding_keys(sc, W):
    rng = np.random.default_rng([W, 57])
    keys, cols = _combine_data(rng, C.SPECS["four"], 200_000, 60_000, 0.0)
    R = 2 * W + 1
    parts, shs, _, _ = CM.run_ranks(sc, W, "four", keys, cols, 4, R)
    CM.free_all(shs)
    C.check_combine(parts, "four", keys, cols, R)


# ---- 4-byte keys: one home bucket at the table size the hint fixes ---------------------------------------------------
def test_four_byte_keys_share_a_home_bucket(sc):
    rng = np.random.default_rng(58)
    log_cap, hint = 13, 2000                                  # ceil_log2(2.5 * hint) = 13
    fam = S.i32_same_home(rng, 200, log_cap)
    n = 120_000
    keys = rng.integers(-1500, 1500, n).astype(np.int32)
    keys[rng.choice(n, 4 * len(fam), replace=False)] = np.repeat(fam, 4)
    keys[:4] = [-1, -(1 << 31), (1 << 31) - 1, 0]
    wide = keys.astype(np.int64).view(np.uint64)
    aborts, longest = S.chain_model(wide, log_cap)
    assert not aborts and longest > 50
    _, vals = rand_pairs(rng, n, 1, "i64", values="full")
    kc = _Col(keys)
    assert kc.key_width == 4
    parts, st = run_reduce(sc, "sum", "i64", kc, _Col(vals, role="value"), n, 1, 7, key_width=4, hint=hint)
    assert st["table_slots"] >= 1 << log_cap
    check_reduce(parts, "sum", "i64", "full", wide, vals, 7, key_width=4)


# ---- more than 1024 keys of one home bucket: a table that cannot grow lets the chain run on ---------------------------
BIG_CASES = ["reduce_host_restart", "reduce_host_max_log", "shared_borrowed", "combine", "group", "narrow", "inner_join"]


def _same_home_rows(rng, n_same, extra_keys=2000, copies=4):
    """Every key of an n_same-key one-home family on `copies` rows, plus rows of extra_keys random keys, 0 and 2^64-1."""
    fam = S.same_home(rng, n_same, SAME_TOP)
    other, _ = rand_pairs(rng, 3 * extra_keys, extra_keys)
    keys = rng.permutation(np.concatenate([np.repeat(fam, copies), other, np.array([0, EMPTY_KEY] * 2, np.uint64)]))
    return keys, fam


@pytest.mark.parametrize("case", BIG_CASES)
@pytest.mark.parametrize("n_same", [1025, 3000])
def test_more_than_1024_keys_of_one_home_bucket(sc, n_same, case):
    rng = np.random.default_rng([n_same, BIG_CASES.index(case), 59])
    keys, fam = _same_home_rows(rng, n_same)
    n, R = len(keys), 5
    vals = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
    if case in ("reduce_host_restart", "reduce_host_max_log"):
        hint = 100 if case == "reduce_host_restart" else 0        # no hint: the first table is already the largest
        parts, st = run_reduce(sc, "max", "i64", _Col(keys), _Col(vals, role="value"), n, 2, R, hint=hint)
        assert st["table_restarts"] >= 1
        check_reduce(parts, "max", "i64", "full", keys, vals, R)
    elif case == "shared_borrowed":
        kc, vc = _col(_dev(keys), L.VB_U64), _col(_dev(vals), L.VB_I64)
        parts, st = run_reduce(sc, "sum", "i64", kc, vc, n, 4, R)
        assert st["kernels"]["merge"]["launches"] == 0 and st["table_restarts"] >= 1
        check_reduce(parts, "sum", "i64", "full", keys, vals, R)
    elif case == "combine":
        cols = [rand_pairs(rng, n, 1, d, values=m)[1] for d, m in C.SPECS["four"][0]]
        kc, vcs = C._cols(keys, cols, "four", device=False)
        parts, _ = C.run_combine(sc, "four", kc, vcs, n, 2, R)
        C.check_combine(parts, "four", keys, cols, R)
    elif case == "group":
        kc, vc = place("dev_soa", keys, vals)
        parts, _ = run_group(sc, sliced(kc, vc, n, 2), R)
        G.assert_group_equal(parts, keys, vals, R)
    elif case == "narrow":
        pa = parent(sc, keys, vals.view(np.uint64), 2, 1, "sum")
        kc = np.concatenate([fam[::3], S.same_home(rng, 300, SAME_TOP, fam), np.array([0, EMPTY_KEY], np.uint64)])
        vc = rng.integers(0, 1 << 64, len(kc), dtype=np.uint64)
        check_sides(sc, [view(pa), shuffles(sc, [(kc, vc, 2)], 1)[0]], [(*result_rows(pa, 1), 1), (kc, vc, 2)], 1,
                    masks=False)
    else:                                                         # the right side holds the family: table_find past bucket 256
        ka = np.concatenate([fam[::2], S.same_home(rng, 500, SAME_TOP, fam), rand_pairs(rng, 3000, 1500)[0]])
        va = full_i64(rng, len(ka))
        sa, sb = cogroup_pair(sc, ka, va, keys, vals, R)
        try:
            check_join(sc, sa, sb, "inner", ka, va, keys, vals, R)
        finally:
            sa.free()
            sb.free()


# ---- a dense one-home input: every key on one chain, one row each, at the largest table size -------------------------
DENSE_CASES = ["reduce_host", "reduce_device", "group", "narrow"]


@pytest.mark.parametrize("case", DENSE_CASES)
def test_dense_one_home_input_at_the_largest_size(sc, case):
    """2^14 distinct keys of one home bucket, one row each, no hint: the table starts at (or restarts to) its largest
    size, 2^15 slots, where the chain is 4096 of its 8192 buckets and every key's insert races every other's.  A
    narrow view inserts them with one thread per key.  Inserts there have no round limit, so no lost CAS can make a
    table that cannot grow give up."""
    rng = np.random.default_rng([DENSE_CASES.index(case), 60])
    fam = S.same_home(rng, 1 << 14, SAME_TOP)
    keys = rng.permutation(fam)
    n, R = len(keys), 5
    vals = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
    assert S.chain_model(keys, 15, limit=1 << 13) == (False, 1 << 12)
    if case == "reduce_host":
        parts, st = run_reduce(sc, "max", "i64", _Col(keys), _Col(vals, role="value"), n, 1, R)
        assert st["table_slots"] >= 1 << 15
        check_reduce(parts, "max", "i64", "full", keys, vals, R)
    elif case == "reduce_device":
        parts, st = run_reduce(sc, "sum", "i64", _col(_dev(keys), L.VB_U64), _col(_dev(vals), L.VB_I64), n, 2, R)
        assert st["table_slots"] >= 1 << 15
        check_reduce(parts, "sum", "i64", "full", keys, vals, R)
    elif case == "group":
        kc, vc = place("dev_soa", keys, vals)
        parts, st = run_group(sc, sliced(kc, vc, n, 1), R)
        assert st["table_slots"] >= 1 << 15
        G.assert_group_equal(parts, keys, vals, R)
    else:
        pa = parent(sc, keys, vals.view(np.uint64), 2, 1, "sum")
        v = view(pa)
        kc = np.concatenate([fam[::8], S.same_home(rng, 500, SAME_TOP, fam), rand_pairs(rng, 2000, 1000)[0]])
        vc = rng.integers(0, 1 << 64, len(kc), dtype=np.uint64)
        check_sides(sc, [v, shuffles(sc, [(kc, vc, 2)], 1)[0]], [(*result_rows(pa, 1), 1), (kc, vc, 2)], 1, masks=False)
        assert v.stats()["table_slots"] == 1 << 15
