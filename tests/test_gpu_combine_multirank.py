"""combine_by_key across ranks, W ranks in one process and one context (vb_shuffle_create_multi_dist and the _cols
export / import calls): every rank's exported key column and [n_acc][rows] accumulator block are swapped with
torch.cat, source-rank major, as the all-to-all-v of vega_b200/dist.py would deliver them.

Every case asserts that partition r has keys only on rank r % W and that the owners' partitions equal the one-process
vb_shuffle_create_multi shuffle over the same map tasks: integer SUM / MIN / MAX, COUNT, integer MEAN and f64 MIN / MAX
bit for bit (NaNs compared as NaN; the all-NaN keys' NaN bit for bit where the case says so), f64 SUM and MEAN against
the exact sums within the bound of any summation order (tests/util.py:assert_f64_sums through check_combine)."""
import ctypes

import numpy as np
import pytest
import torch

import vega_b200 as vb
from tests import cogroup_n_ref as CN
from tests import multirank as MR
from tests.test_gpu_cogroup_n import abi_parts_n, join_parts_n
from tests.test_gpu_combine import AGG, CODE, SPECS, check_combine, make_data, out_dtype, run_combine, spec_of
from tests.util import EMPTY_KEY, assert_parts_equal, bits_dict, rand_pairs
from vega_b200 import _lib as L
from vega_b200.dist import CudaEngine
from vega_b200.rdd import Shuffle, _Col

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


def multi_of(spec):
    dts, aggs = spec_of(spec)
    return [CODE[d] for d, _ in dts], [(AGG[o], c) for o, c in aggs]


def n_acc_of(spec):
    ops = [o for o, _ in SPECS[spec][1]]
    return len(ops) + ("mean" in ops and "count" not in ops)


# ---- the W-rank harness ---------------------------------------------------------------------------------------------
def swap(exports):
    """exports[src] = (counts[dst], keys[rows], accs[n_acc][rows]), destination-major -> per destination (keys, accs,
    counts[src]) with the sources concatenated in ascending order.  New tensors: the exported ones die with the seal."""
    recv = MR.swap_columns([([k, a.t()], [c, c]) for c, k, a in exports])
    return [(k, a.t().contiguous(), n[0]) for (k, a), n in recv]


def placer(keys, cols, loc):
    """place(map_id, lo, hi) -> (key _Col, value _Cols) of rows [lo, hi) on the host, on the device copied in the map
    call (VB_DEVICE) or borrowed until seal (VB_DEVICE_BORROWED: the shared-table path)."""
    if loc == "host":
        return lambda m, lo, hi: (_Col(keys[lo:hi]), tuple(_Col(c[lo:hi], role="value") for c in cols))
    tk = torch.from_numpy(np.ascontiguousarray(keys).view(np.int64)).cuda()
    tcs = [torch.from_numpy(np.ascontiguousarray(c).view(np.int64)).cuda() for c in cols]

    def place(m, lo, hi):
        kc, vcs = _Col(tk[lo:hi]), tuple(_Col(t[lo:hi], role="value") for t in tcs)
        for c in (kc,) + vcs:
            c.code = L.VB_U64
            if loc == "device":
                c.loc = L.VB_DEVICE
        return kc, vcs
    return place


def run_ranks(sc, W, spec, keys, cols, M, R, loc="host", hint=0, key_width=8, resubmit=False, keep_exports=False,
              out_loc=L.VB_HOST):
    """One combine shuffle on W ranks: map, export, swap, import, seal; every partition of every rank is read.
    Returns (the owners' partitions as (keys, [column per aggregate]), shuffles, map-side stats, exports if kept)."""
    multi = multi_of(spec)
    place = placer(keys if key_width == 8 else keys.astype(np.int32), cols, loc)
    maps = MR.maps_by_rank(len(keys), M, W, place)
    shs = [Shuffle.combine_dist(sc, M, R, L.VB_U64, multi, r, W, key_width=key_width, hint=hint) for r in range(W)]
    for r in range(W):
        for m, kc, vcs in maps[r]:
            assert kc.key_width == key_width
            if resubmit:                      # a first attempt with other rows, overwritten by the real one
                other = place(m, 0, min(len(keys), kc.n + 7))
                shs[r].map_cols(m, other[0], other[1], 0, other[0].n)
            shs[r].map_cols(m, kc, vcs, 0, kc.n)
    exports = snaps = None
    if W == 1:
        shs[0].seal()
    else:
        exports = [sh.export_cols() for sh in shs]
        snaps = [sh.stats() for sh in shs]
        kept = [(c, k.clone(), a.clone()) for c, k, a in exports] if keep_exports else None
        for sh, (k, a, c) in zip(shs, swap(exports)):
            sh.import_cols(k, a, c)
        for sh in shs:
            sh.seal()
        exports = kept
    outs = [out_dtype(spec, a) for a in range(len(spec_of(spec)[1]))]
    parts = [None] * R
    for d, sh in enumerate(shs):
        for r in range(R):
            if out_loc == L.VB_HOST:
                p = sh.reduce_cols(r, outs)
            else:
                nk, _ = sh.reduce_size(r)
                tk = torch.empty(nk, dtype=torch.int64, device="cuda")
                ta = [torch.empty(nk, dtype=torch.int64, device="cuda") for _ in outs]
                sh.reduce_cols(r, outs, L.VB_DEVICE, tk, ta)
                p = (tk.cpu().numpy().view(np.uint64), [t.cpu().numpy().view(dt) for t, dt in zip(ta, outs)])
            if r % W == d:
                parts[r] = p
            else:
                assert len(p[0]) == 0, f"rank {d} holds keys of partition {r}, owned by rank {r % W}"
    return parts, shs, snaps, exports


def free_all(shs):
    for sh in shs:
        sh.free()


def one_process(sc, spec, keys, cols, M, R, key_width=8):
    kc = _Col(keys if key_width == 8 else keys.astype(np.int32))
    parts, _ = run_combine(sc, spec, kc, tuple(_Col(c, role="value") for c in cols), len(keys), M, R, key_width=key_width)
    return parts


def assert_equals_one_process(parts, want, spec):
    """Every column but f64 SUM / MEAN bit for bit (NaN as NaN), and the same keys in every partition."""
    dts, aggs = SPECS[spec]
    for a, (op, c) in enumerate(aggs):
        if op in ("sum", "mean") and dts[c][0] == "f64":
            assert_parts_equal([set(k.view(np.uint64).tolist()) for k, _ in parts], [set(k.view(np.uint64).tolist()) for k, _ in want])
            continue
        assert_parts_equal([bits_dict(k, o[a]) for k, o in parts], [bits_dict(k, o[a]) for k, o in want])


def check_all(sc, parts, spec, keys, cols, M, R, key_width=8):
    assert_equals_one_process(parts, one_process(sc, spec, keys, cols, M, R, key_width), spec)
    if key_width == 8:
        check_combine(parts, spec, keys, cols, R)


# ---- 1. the three specs of test_gpu_combine.py on 1 to 256 ranks ------------------------------------------------------
@pytest.mark.parametrize("W", [1, 2, 3, 8, 256])
@pytest.mark.parametrize("spec", list(SPECS))
def test_specs_across_ranks(sc, spec, W):
    """M = 6 map tasks: at W = 8 and 256 most ranks have none and only receive."""
    keys, cols = make_data([W, sorted(SPECS).index(spec), 21], spec, 60_000, 8_000)
    R = 2 * W + 1
    parts, shs, _, _ = run_ranks(sc, W, spec, keys, cols, 6, R)
    free_all(shs)
    check_all(sc, parts, spec, keys, cols, 6, R)


@pytest.mark.parametrize("W,R", [(3, 1), (4, 10), (3, 300)])
def test_partition_counts(sc, W, R):
    """R = 1 (one owner), R not a multiple of W, and R > 256 (the radix split of the finalize)."""
    keys, cols = make_data([W, R, 22], "mixed", 80_000, 20_000)
    parts, shs, _, _ = run_ranks(sc, W, "mixed", keys, cols, 5, R)
    free_all(shs)
    check_all(sc, parts, "mixed", keys, cols, 5, R)


# ---- 2. input locations, resubmission, empty shuffles ------------------------------------------------------------------
@pytest.mark.parametrize("loc", ["host", "device", "borrowed"])
def test_input_locations_and_resubmission(sc, loc):
    keys, cols = make_data([23, ["host", "device", "borrowed"].index(loc)], "four", 150_000, 30_000)
    for resubmit in (False, True):
        parts, shs, snaps, _ = run_ranks(sc, 3, "four", keys, cols, 6, 7, loc=loc, resubmit=resubmit)
        free_all(shs)
        if loc == "borrowed":                 # one shared table per rank: no map-side merge
            assert all(s["kernels"]["merge"]["launches"] == 0 for s in snaps)
        else:
            assert all(s["kernels"]["merge"]["launches"] >= 1 for s in snaps)
        check_all(sc, parts, "four", keys, cols, 6, 7)


def test_empty_shuffles(sc):
    for spec in SPECS:
        keys, cols = make_data(24, spec, 3, 2)
        for loc in ("host", "borrowed"):
            parts, shs, _, _ = run_ranks(sc, 4, spec, keys, cols, 3, 5, loc=loc)     # 3 rows, 3 map tasks, 4 ranks
            free_all(shs)
            check_all(sc, parts, spec, keys, cols, 3, 5)
        parts, shs, snaps, _ = run_ranks(sc, 3, spec, keys[:0], [c[:0] for c in cols], 3, 4)
        assert all(len(k) == 0 for k, _ in parts)
        assert all(sh.stats()["rows_out"] == 0 for sh in shs)
        free_all(shs)


# ---- 3. full value range, special keys, 4-byte keys ----------------------------------------------------------------------
def test_special_values_and_keys_across_ranks(sc):
    """u64 / i64 at full range, f64 NaN payloads, +-0 and +-inf ("four": columns full, full, exact, special); keys 0 and
    2^64 - 1 on every rank; a key whose column-3 values are all NaN on rank 0's map task only, and one all NaN
    everywhere: its MIN / MAX NaN is the one-process NaN bit for bit."""
    W, M, R = 3, 3, 7
    keys, cols = make_data(25, "four", 90_000, 6_000)
    starts = vb.slice_starts(len(keys), M)
    for m in range(M):
        lo = int(starts[m])
        keys[lo:lo + 40:2] = 0
        keys[lo + 1:lo + 40:2] = EMPTY_KEY
        keys[lo + 40:lo + 60] = 0xABCDEF                      # NaN on map 0 only
        keys[lo + 60:lo + 80] = 0x123456                      # NaN on every map
        bits = cols[3].view(np.uint64)
        bits[lo + 60:lo + 80] = [0x7FF8000000000000 + i for i in range(20)]
        if m == 0:
            bits[lo + 40:lo + 60] = [0xFFF8000000000001 + i for i in range(20)]
    parts, shs, _, _ = run_ranks(sc, W, "four", keys, cols, M, R)
    free_all(shs)
    check_all(sc, parts, "four", keys, cols, M, R)
    want = one_process(sc, "four", keys, cols, M, R)
    raw = lambda ps, a: {k: v for kk, o in ps for k, v in zip(kk.view(np.uint64).tolist(), o[a].view(np.uint64).tolist())}
    for a in (6, 7):                                          # min(3), max(3)
        g, w = raw(parts, a), raw(want, a)
        assert np.isnan(np.uint64(g[0x123456]).view(np.float64)) and g[0x123456] == w[0x123456]
        assert not np.isnan(np.uint64(g[0xABCDEF]).view(np.float64)) and g[0xABCDEF] == w[0xABCDEF]
        assert g[0] == w[0] and g[EMPTY_KEY] == w[EMPTY_KEY]


def test_four_byte_keys(sc):
    rng = np.random.default_rng(26)
    n = 100_000
    k32 = rng.integers(-3000, 3000, n).astype(np.int32)
    k32[:4] = [-1, -(1 << 31), (1 << 31) - 1, 0]
    keys = k32.astype(np.int64)
    _, cols = make_data(26, "four", n, 3000)
    parts, shs, _, _ = run_ranks(sc, 3, "four", keys, cols, 4, 11, key_width=4)
    free_all(shs)
    for r, (k, _) in enumerate(parts):
        assert all(vb.lib().vb_get_partition(int(x), 4, 11) == r for x in k.view(np.uint64).tolist())
    assert_equals_one_process(parts, one_process(sc, "four", keys, cols, 4, 11, key_width=4), "four")


# ---- 4. table restarts, device output ------------------------------------------------------------------------------------
@pytest.mark.parametrize("loc", ["host", "borrowed"])
def test_table_restarts_on_map_side_and_import_merge(sc, loc):
    """hint = 1: the per-map (host) or shared (borrowed) tables overflow and restart, and so does the import merge."""
    keys, cols = make_data([27, int(loc == "host")], "mixed", 200_000, 60_000)
    parts, shs, snaps, _ = run_ranks(sc, 2, "mixed", keys, cols, 4, 5, loc=loc, hint=1)
    assert all(s["table_restarts"] >= 1 for s in snaps)
    assert all(sh.stats()["table_restarts"] > s["table_restarts"] for sh, s in zip(shs, snaps))
    free_all(shs)
    check_all(sc, parts, "mixed", keys, cols, 4, 5)


def test_device_output_equals_host_output(sc):
    keys, cols = make_data(28, "four", 120_000, 20_000)
    host, shs, _, _ = run_ranks(sc, 3, "four", keys, cols, 4, 7, loc="borrowed")
    free_all(shs)
    dev, shs, _, _ = run_ranks(sc, 3, "four", keys, cols, 4, 7, loc="borrowed", out_loc=L.VB_DEVICE)
    free_all(shs)
    for (hk, ho), (dk, do) in zip(host, dev):
        oh, od = np.argsort(hk.view(np.uint64)), np.argsort(dk.view(np.uint64))
        assert np.array_equal(hk.view(np.uint64)[oh], dk.view(np.uint64)[od])
        for a, b in zip(ho, do):
            assert np.array_equal(a.view(np.uint64)[oh], b.view(np.uint64)[od])


# ---- 5. the wire format -----------------------------------------------------------------------------------------------------
def rank_partials(keys, cols, spec, rows):
    """(distinct keys, [partial of every accumulator per key]) of one rank's rows, in plain value form, from numpy."""
    dts, aggs = SPECS[spec]
    k = keys[rows].view(np.uint64)
    uk, inv = np.unique(k, return_inverse=True)
    accs = []
    specs = list(aggs) + ([("count", 0)] if n_acc_of(spec) > len(aggs) else [])
    for op, c in specs:
        d = dts[c][0]
        v = cols[c][rows]
        if op == "count":
            x = np.zeros(len(uk), np.uint64)
            np.add.at(x, inv, np.uint64(1))
        elif op in ("sum", "mean"):
            x = np.zeros(len(uk), np.float64 if d == "f64" else np.uint64)
            np.add.at(x, inv, v if d == "f64" else v.view(np.uint64))
        else:
            if d == "f64":
                x = np.full(len(uk), np.nan)
                (np.fmin if op == "min" else np.fmax).at(x, inv, v)
            else:
                dt = np.int64 if d == "i64" else np.uint64
                x = np.full(len(uk), np.iinfo(dt).max if op == "min" else np.iinfo(dt).min, dtype=dt)
                (np.minimum if op == "min" else np.maximum).at(x, inv, v.astype(dt))
        accs.append(x)
    return uk, accs


def test_wire_format_decodes_to_per_rank_partials(sc):
    """Each rank's export: one row per distinct key it holds, in the destination block of the key's owner, with the
    partial of every accumulator (the spec's COUNT, each SUM, a MEAN's sum, MIN / MAX in the column's dtype, f64 NaN
    when all the rank's values were NaN).  "mixed" adds the internal COUNT after its 7 aggregates."""
    W, M, R = 3, 5, 7
    for spec in ("four", "mixed"):
        keys, cols = make_data(29, spec, 50_000, 4_000)
        if spec == "mixed":
            cols[2] = np.ldexp(np.round(cols[2] * 8), -3)            # exact f64 sums in any order
        parts, shs, _, exports = run_ranks(sc, W, spec, keys, cols, M, R, keep_exports=True)
        free_all(shs)
        starts = vb.slice_starts(len(keys), M)
        for r, (counts, k, a) in enumerate(exports):
            assert a.shape == (n_acc_of(spec), sum(counts)) and k.shape == (sum(counts),)
            lo, hi = vb.dist.map_block(r, W, M)
            uk, want = rank_partials(keys, cols, spec, np.arange(int(starts[lo]), int(starts[hi])))
            ku = k.cpu().numpy().view(np.uint64)
            off = np.cumsum([0] + counts)
            for d in range(W):
                assert all(vb.lib().vb_get_partition(int(x), 8, R) % W == d for x in ku[off[d]:off[d + 1]].tolist())
            order = np.argsort(ku)
            assert np.array_equal(ku[order], uk), "not one row per distinct key of the rank"
            got = a.cpu().numpy()[:, order]
            for j, w in enumerate(want):
                if w.dtype == np.float64:      # NaN where all the rank's values were NaN; +-0 compare equal
                    assert np.array_equal(got[j].view(np.float64), w, equal_nan=True), (spec, j)
                else:
                    assert np.array_equal(got[j].view(np.uint64), w.view(np.uint64)), (spec, j)
        check_all(sc, parts, spec, keys, cols, M, R)


# ---- 6. a column of a multi-rank combine as a join side -----------------------------------------------------------------
@pytest.mark.parametrize("W", [2, 3])
def test_narrow_view_joined_with_multirank_cogroup(sc, W):
    rng = np.random.default_rng(30 + W)
    R, M = 2 * W + 1, 2 * W
    keys, cols = make_data(30 + W, "four", 20_000, 3_000)
    kb, vb_ = rand_pairs(rng, 12_000, 3000, values="full")
    kb[: len(kb) // 2] = keys[: len(kb) // 2]                  # half of the right keys are left keys
    tb, tvb = (torch.from_numpy(x.view(np.int64)).cuda() for x in (kb, vb_))
    _, combs, _, _ = run_ranks(sc, W, "four", keys, cols, M, R, loc="borrowed")
    cogs, _ = MR.run_ranks(CudaEngine(sc), W, L.VB_AGG_COGROUP,
                           MR.maps_by_rank(len(kb), M, W, lambda m, lo, hi: (tb[lo:hi], tvb[lo:hi])), R, L.VB_U64, L.VB_U64)
    uk, cnt = np.unique(keys.view(np.uint64), return_counts=True)
    want = CN.ref_parts_n([(uk, cnt.astype(np.uint64), 1), (kb, vb_, M)], R)
    got, got_j = [dict() for _ in range(R)], [dict() for _ in range(R)]
    for d in range(W):
        v = Shuffle.narrow(combs[d], 0, L.VB_U64)              # column 0: the spec's COUNT
        parts, joins = abi_parts_n(sc, [v, cogs[d]], R), join_parts_n(sc, [v, cogs[d]], R)
        for r in range(R):
            if r % W == d:
                got[r], got_j[r] = parts[r], joins[r]
            else:
                assert not parts[r] and not joins[r], f"rank {d} has keys of partition {r}"
    assert_parts_equal(got, want)
    assert_parts_equal(got_j, CN.join_of_parts(want))
    free_all(combs + cogs)


# ---- 7. errors ----------------------------------------------------------------------------------------------------------------
def _code(fn):
    try:
        fn()
    except vb.VegaB200Error as e:
        return e.code
    return L.VB_OK


def test_errors(sc):
    lib = vb.lib()
    codes, aggs = multi_of("four")
    dts = (ctypes.c_int32 * len(codes))(*codes)
    spec = (L.vb_agg_col * len(aggs))(*[L.vb_agg_col(a, c) for a, c in aggs])
    h = ctypes.c_void_p()
    for rank, world in ((0, 0), (0, 257), (2, 2), (5, 3)):
        assert lib.vb_shuffle_create_multi_dist(sc._h, 0, 1, 2, L.VB_U64, 4, dts, 8, spec, rank, world, ctypes.byref(h)) == L.VB_ERR_INVALID
    assert _code(lambda: Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, multi=(codes, aggs), world=2)) == L.VB_ERR_UNSUPPORTED
    keys = np.arange(100, dtype=np.uint64)
    kc, vcs = _Col(keys), tuple(_Col(keys.view(np.int64) if d != L.VB_F64 else keys.astype(np.float64), role="value") for d in codes)
    cnt2 = (ctypes.c_uint64 * 2)()
    p = ctypes.c_void_p(keys.ctypes.data)
    kp, ap, na = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint32()
    # a single-column shuffle: VB_ERR_INVALID; a multi shuffle of world 1: VB_ERR_STATE
    single = Shuffle(sc, 1, 2, L.VB_U64, L.VB_U64, L.VB_AGG_SUM, rank=0, world=2)
    one = Shuffle.combine_dist(sc, 1, 2, L.VB_U64, (codes, aggs), 0, 1)
    for s_, want in ((single, L.VB_ERR_INVALID), (one, L.VB_ERR_STATE)):
        assert lib.vb_shuffle_export_cols_prepare(s_._h, cnt2) == want
        assert lib.vb_shuffle_export_cols_buffers(s_._h, ctypes.byref(kp), ctypes.byref(ap), ctypes.byref(na)) == want
        assert lib.vb_shuffle_import_cols(s_._h, p, p, 8, cnt2) == want
    assert lib.vb_shuffle_exchange(one._h, L.VB_XCHG_AUTO) == L.VB_ERR_UNSUPPORTED
    single.free()
    one.free()
    sh = Shuffle.combine_dist(sc, 1, 2, L.VB_U64, (codes, aggs), 0, 2)
    h = sh._h
    # the single-column, P2P and set_dist calls stay unsupported on a multi shuffle
    assert lib.vb_shuffle_set_dist(h, 0, 2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_set_dist(h, 0, 1) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_prepare(h, cnt2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_counts(h, cnt2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_buffers(h, ctypes.byref(kp), ctypes.byref(ap)) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_import(h, None, None, cnt2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_export_direct(h, cnt2, cnt2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_import_arena(h, cnt2) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_exchange(h, L.VB_XCHG_P2P) == L.VB_ERR_UNSUPPORTED
    assert lib.vb_shuffle_exchange(h, L.VB_XCHG_NCCL) == L.VB_ERR_STATE            # no communicator
    # phase errors
    assert lib.vb_shuffle_import_cols(h, p, p, 8, cnt2) == L.VB_ERR_STATE            # before export
    assert lib.vb_shuffle_export_cols_buffers(h, ctypes.byref(kp), ctypes.byref(ap), ctypes.byref(na)) == L.VB_ERR_STATE
    sh.map_cols(0, kc, vcs, 0, 100)
    assert lib.vb_shuffle_seal(h) == L.VB_ERR_STATE                                   # no export, no import
    counts, k, a = sh.export_cols()
    assert sum(counts) == 100 and a.shape == (8, 100)
    assert lib.vb_shuffle_export_cols_prepare(h, cnt2) == L.VB_ERR_STATE              # twice
    assert _code(lambda: sh.map_cols(0, kc, vcs, 0, 100)) == L.VB_ERR_STATE          # map after export
    assert lib.vb_shuffle_seal(h) == L.VB_ERR_STATE                                   # no import
    big = (ctypes.c_uint64 * 2)(0xFFFFFFFE, 0)
    nz = (ctypes.c_uint64 * 2)(1, 0)
    assert lib.vb_shuffle_import_cols(h, p, p, 8, big) == L.VB_ERR_TOO_LARGE
    assert lib.vb_shuffle_import_cols(h, None, p, 8, nz) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_import_cols(h, p, None, 8, nz) == L.VB_ERR_INVALID
    assert lib.vb_shuffle_import_cols(h, p, p, 7, nz) == L.VB_ERR_INVALID
    with pytest.raises(ValueError):
        sh.import_cols(k, a[:, :3], counts)                                          # caught by the mirror
    kk, aa = k.clone(), a.clone()
    sh.import_cols(kk, aa, counts)
    assert lib.vb_shuffle_import_cols(h, p, p, 8, nz) == L.VB_ERR_STATE              # twice
    sh.seal()
    assert lib.vb_shuffle_import_cols(h, p, p, 8, nz) == L.VB_ERR_STATE              # after seal
    assert lib.vb_shuffle_export_cols_buffers(h, ctypes.byref(kp), ctypes.byref(ap), ctypes.byref(na)) == L.VB_ERR_STATE
    assert sum(len(sh.reduce_cols(r, [out_dtype("four", i) for i in range(8)])[0]) for r in range(2)) == 100
    sh.free()
