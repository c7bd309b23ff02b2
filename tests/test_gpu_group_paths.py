"""group_by_key, the cogroup and every join kind through each path of the grouping pipeline (seal_group), against the
exact references of tests/group_ref.py: every key, its partition, and its value list element for element.

seal_group builds a key -> slot dictionary (one slot id per row), numbers the keys bucket-major, sorts the
(u32 id, u64 value) pairs with a stable LSD sort of ceil(ceil_log2(max(D, 2)) / 8) passes of 8 bits, and turns the
sorted ids into CSR offsets.  Which kernels run depends on the number of distinct keys D, the row count, the
alignment of the rows, the loader and table restarts.  Each case places its input so that one path must run and
asserts the statistic that proves it; where no statistic tells two kernels apart, it asserts the input property that
selects the kernel and names the kernel in a comment:
  * rp_scatter launches = id-sort passes + 1 (R <= 256) or + 2 (R > 256): the multisplit of the dictionary by
    partition is one pass, or two 8-bit passes over the 16-bit bucket id;
  * the gather sweep (rp_gsweep_kernel) runs a pass only on 16-byte aligned rows with n >= 4 sweep tiles; otherwise
    rp_scatter_kernel does; the last pass records the CSR itself (rp_gsweep_kernel<CSR>) only when it is a gather
    sweep over SoA (id, value) rows, otherwise csr_bounds_kernel computes it;
  * the dictionary restarts 4x larger on overflow and rewrites every row's slot id (table_restarts).
Values are full-range i64, compared bit for bit; keys 0 and 2^64-1 (the table's empty marker) are in every case with
at least 3 keys."""
import numpy as np
import pytest

import vega_b200 as vb
from tests import group_ref as G
from tests.test_gpu_cogroup import abi_cogroup
from tests.test_gpu_outer_join import abi_rows
from tests.test_gpu_reduce_paths import _col, _dev
from tests.util import EMPTY_KEY
from vega_b200 import _lib as L
from vega_b200.rdd import Shuffle, _Col

pytestmark = pytest.mark.gpu

# gather-sweep tile of the (u32 id, u64 value) passes, GsPlan<u32, true, LDM>::T in gsweep.cuh: 1024 threads x K rows
GS_TILE_SOA = 1024 * 11         # LD_KEY32_VAL_SOA
GS_TILE_AOS = 1024 * 7          # LD_KEY32_VAL_AOS (values inside 16-byte rows)
PHI = np.uint64(0x9E3779B97F4A7C15)
BIG = (1 << 24) + (1 << 21)     # rows of the 2^24-key cases


@pytest.fixture(scope="module")
def sc():
    c = vb.Context(0)
    yield c
    c.close()


def passes(D):
    """Id-sort passes of seal_group for D distinct keys."""
    bits = (max(D, 2) - 1).bit_length()
    return max(1, (bits + 7) // 8)


def scatter_launches(D, R):
    return passes(D) + (1 if R <= 256 else 2)


def exact_keys(rng, n, D, hot=0.0, first_rank=0):
    """n keys with exactly D distinct values: ranks first_rank + a permutation of 0..D-1 plus n - D random draws,
    shuffled, through rand_pairs' bijection; for D >= 3 ranks first_rank and first_rank + 1 become the keys 0 and
    2^64-1.  hot > 0: about that share of the rows has rank first_rank + 2."""
    extra = rng.integers(0, D, n - D)
    if hot:
        extra[rng.random(n - D) < hot * n / (n - D)] = 2
    ranks = rng.permutation(np.concatenate([np.arange(D), extra])).astype(np.uint64) + np.uint64(first_rank)
    keys = ranks * PHI + np.uint64(12345)
    if D >= 3:
        keys[ranks == np.uint64(first_rank)] = 0
        keys[ranks == np.uint64(first_rank + 1)] = EMPTY_KEY
    return keys


def full_i64(rng, n):
    return rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)


def place(where, keys, vals):
    """(key column or rows, value column or None) as the library receives them."""
    if where == "host_soa":
        return _Col(keys), _Col(vals, role="value")
    if where in ("dev_soa", "dev_soa_misaligned"):
        mis = where.endswith("misaligned")
        kc, vc = _col(_dev(keys, misalign=mis), L.VB_U64), _col(_dev(vals, misalign=mis), L.VB_I64)
        assert kc.ptr % 16 == vc.ptr % 16 == (8 if mis else 0)
        return kc, vc
    rows = np.stack([keys, vals.view(np.uint64)], axis=1)
    if where == "dev_aos":
        return _col(_dev(rows), L.VB_I64, rows=True), None
    assert where == "host_aos", where
    return _Col(rows, allow_rows=True), None


def run_group(sc, maps, R, hint=0):
    """One GROUP shuffle; maps[m] = (key column or rows, value column, start, stop).  Returns every partition and the
    statistics."""
    sh = Shuffle(sc, len(maps), R, L.VB_U64, L.VB_I64, L.VB_AGG_GROUP, hint=hint)
    try:
        for m, (kc, vc, a, b) in enumerate(maps):
            sh.map(m, kc, vc, a, b)
        sh.seal()
        parts = [sh.reduce(r) for r in range(R)]
        st = sh.stats()
    finally:
        sh.free()
    return parts, st


def sliced(kc, vc, n, M):
    s = vb.slice_starts(n, M)
    return [(kc, vc, int(s[m]), int(s[m + 1])) for m in range(len(s) - 1)]


# ---- group_by_key: the path matrix --------------------------------------------------------------------------------
# name: (D, rows, placement, map tasks, R, hot-key share)
GROUP_CASES = {
    "one_key": (1, 3_000_000, "dev_soa", 4, 7, 0.0),             # one value run across every part and tile
    "d256_aos": (256, 2_000_000, "dev_aos", 3, 7, 0.0),          # AoS loader (zero-copy: the 3 maps are adjacent rows)
    "d256_misaligned": (256, 2_000_000, "dev_soa_misaligned", 1, 7, 0.0),
    "d257": (257, 2_000_000, "host_soa", 3, 7, 0.0),             # first 2-pass D
    "d65536": (1 << 16, 3_000_000, "dev_soa", 1, 7, 0.0),        # last 2-pass D
    "d65537": ((1 << 16) + 1, 3_000_000, "dev_soa_misaligned", 1, 7, 0.0),
    "d2^24": (1 << 24, BIG, "dev_soa", 4, 7, 0.0),               # last 3-pass D
    "d2^24+1": ((1 << 24) + 1, BIG, "dev_soa", 4, 257, 0.0),     # 4 passes, two-pass multisplit of the dictionary
    "d2^24+1_host_aos": ((1 << 24) + 1, BIG, "host_aos", 3, 7, 0.0),
    "small_n": (3000, 5000, "dev_soa", 1, 7, 0.0),
    "hot": (100_000, 8_000_000, "dev_soa", 1, 7, 0.6),           # one run across many parts: CSR starts by atomicMin
}


@pytest.mark.parametrize("case", list(GROUP_CASES))
def test_group_path_matches_exact_reference(sc, case):
    D, n, where, M, R, hot = GROUP_CASES[case]
    rng = np.random.default_rng([list(GROUP_CASES).index(case), 7])
    keys, vals = exact_keys(rng, n, D, hot=hot), full_i64(rng, n)
    kc, vc = place(where, keys, vals)
    aligned = kc.ptr % 16 == 0
    if case == "d256_misaligned":
        # one borrowed map is grouped in place: the register-staged hash_agg_kernel<OPK_DICT> builds the dictionary
        # (the bulk kernel needs 16-byte aligned keys) and the only pass, rp_scatter_kernel<u32, true,
        # LD_KEY32_VAL_SOA, DG_BITS>, reads the caller's misaligned values; csr_bounds_kernel computes the CSR
        assert not aligned and M == 1
    elif case == "d65537":
        # pass 1 reads the caller's misaligned values (rp_scatter_kernel), passes 2 and 3 the library's own aligned
        # buffers (rp_gsweep_kernel, the last one rp_gsweep_kernel<CSR>)
        assert not aligned and M == 1 and n >= 4 * GS_TILE_SOA
    elif case == "small_n":
        # n < 4 sweep tiles: rp_scatter_kernel on both passes, csr_bounds_kernel
        assert n < 4 * GS_TILE_SOA
    elif case == "d256_aos":
        # the one pass reads values inside the rows (LD_KEY32_VAL_AOS): csr_bounds_kernel computes the CSR
        assert aligned and kc.rows and n >= 4 * GS_TILE_AOS
    else:
        assert aligned and n >= 4 * GS_TILE_SOA
    parts, st = run_group(sc, sliced(kc, vc, n, M), R)
    assert st["kernels"]["rp_scatter"]["launches"] == scatter_launches(D, R)
    assert sum(len(p[0]) for p in parts) == D
    if hot:
        assert max(int(np.diff(p[1].astype(np.int64)).max(initial=0)) for p in parts) > 0.55 * n
    G.assert_group_equal(parts, keys, vals, R)


@pytest.mark.parametrize("case", ["restart", "restart_misaligned"])
def test_group_dictionary_restarts(sc, case):
    """hint=1: the dictionary starts at 16 slots and restarts 4x larger until 120k keys fit; every restart rewrites
    the slot id of every row, across every input.  restart: maps on the host, copied from the device, empty and
    borrowed (gathered into one owned input); restart_misaligned: one borrowed misaligned map, grouped in place by
    the register-staged dictionary kernel."""
    rng = np.random.default_rng(len(case))
    D, n, R = 120_000, 300_000, 7
    keys, vals = exact_keys(rng, n, D), full_i64(rng, n)
    if case == "restart":
        a, b = n // 3, 2 * n // 3
        dev = [_col(_dev(keys), L.VB_U64), _col(_dev(vals), L.VB_I64)]
        for c in dev:
            c.loc = L.VB_DEVICE                       # copied by the library before the map call returns
        borrowed = (_col(_dev(keys), L.VB_U64), _col(_dev(vals), L.VB_I64))
        maps = [(_Col(keys), _Col(vals, role="value"), 0, a), (dev[0], dev[1], a, b), (borrowed[0], borrowed[1], b, b),
                (borrowed[0], borrowed[1], b, n)]
    else:
        kc, vc = place("dev_soa_misaligned", keys, vals)
        maps = [(kc, vc, 0, n)]
    parts, st = run_group(sc, maps, R, hint=1)
    assert st["table_restarts"] >= 2
    assert st["kernels"]["rp_scatter"]["launches"] == scatter_launches(D, R)
    G.assert_group_equal(parts, keys, vals, R)


# ---- cogroup and joins --------------------------------------------------------------------------------------------
# A lazy COGROUP seal copies the rows into owned aligned buffers, so alignment is no axis here: pass count, restarts
# and size are.  While both sides are lazy, a join groups internal shuffles: a side the kind keeps whole is grouped
# whole, the other only over the rows whose key is on both sides (filtered through a dictionary of the right keys,
# built with the right side's hint and counted on the left shuffle).  Their kernel launches count on the left shuffle.
def cogroup_pair(sc, ka, va, kb, vb_, R, Ma=3, Mb=2, hint_b=0):
    out = []
    for k, v, M, hint in ((ka, va, Ma, 0), (kb, vb_, Mb, hint_b)):
        maps = sliced(_Col(k), _Col(v, role="value"), len(k), M)
        sh = Shuffle(sc, len(maps), R, L.VB_U64, L.VB_I64, L.VB_AGG_COGROUP, hint=hint)
        for m, (kc, vc, a, b) in enumerate(maps):
            sh.map(m, kc, vc, a, b)
        sh.seal()
        out.append(sh)
    return out


def gpu_join(sc, sa, sb, kind, R):
    return G.join_output_rows([abi_rows(sc, sa, sb, r, None if kind == "inner" else kind) for r in range(R)], R)


def gpu_cogroup(sc, sa, sb, R):
    parts = []
    for r in range(R):
        k, lo, lv, ro, rv = abi_cogroup(sc, sa, sb, r)
        parts.append((k, (lo, lv), (ro, rv)))
    return parts


def check_join(sc, sa, sb, kind, ka, va, kb, vb_, R):
    G.assert_rows_equal(gpu_join(sc, sa, sb, kind, R), G.join_rows(kind, ka, va, kb, vb_), G.JOIN_COLS)


def _free(*shs):
    for s in shs:
        s.free()


def test_cogroup_and_full_join_four_passes_per_side(sc):
    """Both sides with 2^24 + 1 distinct keys, half of them shared: the FULL pair groups each side whole, 4 passes
    each; the cogroup reads the same pair."""
    rng = np.random.default_rng(24)
    D, R = (1 << 24) + 1, 7
    ka, kb = exact_keys(rng, D + (1 << 20), D), exact_keys(rng, D + (1 << 19), D, first_rank=D // 2)
    va, vb_ = full_i64(rng, len(ka)), full_i64(rng, len(kb))
    sa, sb = cogroup_pair(sc, ka, va, kb, vb_, R)
    try:
        check_join(sc, sa, sb, "full", ka, va, kb, vb_, R)
        G.assert_cogroup_equal(gpu_cogroup(sc, sa, sb, R), ka, va, kb, vb_, R)
        assert sa.stats()["kernels"]["rp_scatter"]["launches"] == 2 * scatter_launches(D, R)
    finally:
        _free(sa, sb)


def test_inner_join_four_passes(sc):
    """2^24 + 1 keys on both sides, every key shared, a few hundred of them with 2-3 rows on each side (nesting
    order): each filtered side sorts in 4 passes."""
    rng = np.random.default_rng(25)
    D, R = (1 << 24) + 1, 7
    ka, kb = exact_keys(rng, D + 400, D), exact_keys(rng, D + 500, D)
    va, vb_ = full_i64(rng, len(ka)), full_i64(rng, len(kb))
    sa, sb = cogroup_pair(sc, ka, va, kb, vb_, R)
    try:
        check_join(sc, sa, sb, "inner", ka, va, kb, vb_, R)
        assert sa.stats()["kernels"]["rp_scatter"]["launches"] == 2 * scatter_launches(D, R)
    finally:
        _free(sa, sb)


def test_left_join_four_passes(sc):
    """2^24 + 1 left keys, 2 % of them on the right too (plus keys on the right only): the left side is grouped
    whole in 4 passes, the right only over its matching rows."""
    rng = np.random.default_rng(26)
    D, R = (1 << 24) + 1, 7
    ka = exact_keys(rng, D + (1 << 20), D)
    shared = rng.choice(np.unique(ka), D // 50, replace=False)
    kb = np.concatenate([np.repeat(shared, 2), exact_keys(rng, 200_000, 100_000, first_rank=D)])
    kb = rng.permutation(kb)
    va, vb_ = full_i64(rng, len(ka)), full_i64(rng, len(kb))
    n_matched = len(np.intersect1d(ka, kb))                 # the shared draws, and keys 0 and 2^64-1
    sa, sb = cogroup_pair(sc, ka, va, kb, vb_, R)
    try:
        check_join(sc, sa, sb, "left", ka, va, kb, vb_, R)
        assert sa.stats()["kernels"]["rp_scatter"]["launches"] == scatter_launches(D, R) + scatter_launches(n_matched, R)
    finally:
        _free(sa, sb)


@pytest.mark.parametrize("order", ["lazy", "grouped"])
@pytest.mark.parametrize("kind", ["inner", "left", "right", "full", "cogroup"])
def test_right_side_hint_restarts(sc, kind, order):
    """The right side created with hint=1.  lazy: inner / left / right filter the rows through a dictionary of the
    right keys built with that hint, which restarts (counted on the left shuffle); full and the cogroup keep both
    sides whole and build no such dictionary.  grouped: every partition of both sides is read first
    (vb_shuffle_reduce), so the right side's own dictionary restarts, and the join reads the grouped sides."""
    rng = np.random.default_rng([len(kind), len(order)])
    R = 7
    ka, kb = exact_keys(rng, 90_000, 40_000), exact_keys(rng, 80_000, 50_000, first_rank=25_000)
    ka[:300], kb[:300] = ka[300:600], ka[300:600]          # a few keys with 2+ rows on each side
    va, vb_ = full_i64(rng, len(ka)), full_i64(rng, len(kb))
    sa, sb = cogroup_pair(sc, ka, va, kb, vb_, R, hint_b=1)
    try:
        if order == "grouped":
            for s_, k, v in ((sa, ka, va), (sb, kb, vb_)):
                G.assert_group_equal([s_.reduce(r) for r in range(R)], k, v, R)
            assert sb.stats()["table_restarts"] >= 1
        if kind == "cogroup":
            G.assert_cogroup_equal(gpu_cogroup(sc, sa, sb, R), ka, va, kb, vb_, R)
        else:
            check_join(sc, sa, sb, kind, ka, va, kb, vb_, R)
        if order == "lazy" and kind in ("inner", "left", "right"):
            assert sa.stats()["table_restarts"] >= 1
    finally:
        _free(sa, sb)


@pytest.mark.parametrize("kind", ["inner", "left", "right", "full", "cogroup"])
def test_sides_smaller_than_one_tile(sc, kind):
    """Sides of 3000 and 700 rows (one radix tile is 4096 rows): every id-sort pass is rp_scatter_kernel."""
    rng = np.random.default_rng(len(kind) + 40)
    R = 5
    ka, kb = exact_keys(rng, 3000, 1200), exact_keys(rng, 700, 500, first_rank=900)
    va, vb_ = full_i64(rng, len(ka)), full_i64(rng, len(kb))
    assert len(ka) < 4096 and len(kb) < 4096
    sa, sb = cogroup_pair(sc, ka, va, kb, vb_, R)
    try:
        if kind == "cogroup":
            G.assert_cogroup_equal(gpu_cogroup(sc, sa, sb, R), ka, va, kb, vb_, R)
        else:
            check_join(sc, sa, sb, kind, ka, va, kb, vb_, R)
    finally:
        _free(sa, sb)
