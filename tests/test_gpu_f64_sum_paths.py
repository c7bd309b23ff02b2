"""f64 SUM and MEAN at NaN, +-inf, overflow and -0.0 on every aggregate path, against tests/f64_sum_ref.py.

The sum of a key's values may come out of any summation order (atomics, hot-key caches, per-map tables, other ranks'
partials, CPU-produced blob partials), so each key is checked against the set of results some order can produce: NaN
as a class, infinities, the exact sum bit for bit where every partial sum is representable (the sign of a zero
included: all -0.0 sums to -0.0, any other zero to +0.0), the order-independent error bound otherwise.  Only the
few keys whose partial sums can overflow may take more than one outcome class.

sharp_pairs places the cases where the kernels branch: an all -0.0 key on key 0 and on 2^64-1 (the table's empty
marker, which takes the special slot), the hot key of the hot-key-cache paths all -0.0 and the second hot key with a
NaN, keys spread over every map task (so over every rank of a multi-rank run) whose per-rank partials are -0.0 on every
rank, NaN on one rank only, and +inf on one rank with -inf on another; and for String keys, warps full of one key, so
that the match-any leader fold meets -0.0 and NaN.  Each path asserts the statistic that proves it ran (the runners of
test_gpu_reduce_paths.py and test_gpu_combine.py)."""
import numpy as np
import pytest

import vega_b200 as vb
from tests import f64_sum_ref as F
from tests import str_blob_ref as B
from tests import test_gpu_combine as CB
from tests import test_gpu_reduce_paths as RP
from tests.test_gpu_combine_multirank import free_all, run_ranks as combine_ranks
from tests.test_gpu_multirank_paths import shuffle_ranks
from tests.test_gpu_str_blob import combined_blob, str_pairs
from tests.test_gpu_str_combine import decode
from tests.test_gpu_str_combine_multirank import owned as str_combine_owned, run_world
from tests.test_gpu_str_multirank import columns, owned as str_owned, run_ranks as str_ranks
from tests.util import EMPTY_KEY, NAN_BITS, assert_f64_sums
from vega_b200 import _lib as L
from vega_b200 import dist as vdist
from vega_b200.rdd import StrShuffle, _Col

pytestmark = pytest.mark.gpu

GOLD = np.uint64(0x9E3779B97F4A7C15)
# key classes, by rank
NEGZ, ZEROS, CANCEL, NAN, PINF, NINF, BOTHINF, INF_FIN, EXACT, SUB, OVF = range(11)


@pytest.fixture(scope="module")
def sc():
    with vb.Context(0) as c:
        yield c


def key_class(ranks):
    """Rank r's class: r % 11, except that only one in 8 of the overflow-prone ranks stays so (the rest are exact),
    rank 0 (the hot key) is all -0.0 and rank 1 (the second hot key) holds a NaN."""
    c = (ranks % np.uint64(11)).astype(np.int64)
    c[(c == OVF) & ((ranks // np.uint64(11)) % np.uint64(8) != 0)] = EXACT
    c[ranks == 0] = NEGZ
    c[ranks == 1] = NAN
    return c


def sharp_pairs(rng, n, n_keys, hot=0.0, wide=True, runs=False):
    """n f64 rows over about n_keys keys -> (keys u64, values, class of each row).

    Values by class: all -0.0; a mix of +-0.0; -0.0 with exact values that cancel to zero (the key's last row takes
    the negated sum of the others); exact values k * 2^-30 with a NaN (both signs, own payloads) on the key's first
    row; +inf only; -inf only; exact values with +inf first and -inf last; exact values with +inf first; exact
    values; subnormals k * 2^-1074; +-1.5e308 (overflow-prone).  hot: as rand_pairs (rank 0 all -0.0, rank 1 with a
    NaN).  wide: keys spread over 64 bits, plus rows on key 0 and on 2^64-1, all -0.0; else the key is the rank.  runs:
    the first 512 rows are 8 warps of rank 0 and 8 of rank 1.  Three more keys have about 32 rows each spread evenly
    over the rows: all -0.0; exact values with a NaN on its first row; exact values with +inf on its first row and
    -inf on its last."""
    ranks = rng.integers(0, max(n_keys, 1), n).astype(np.uint64)
    if hot:
        u = rng.random(n)
        ranks[u < 1.5 * hot] = np.uint64(1)
        ranks[u < hot] = np.uint64(0)
    if runs:
        ranks[:256], ranks[256:512] = 0, 1
    spread = np.uint64(n_keys) + np.arange(3, dtype=np.uint64)
    pos = np.arange(512 if runs else 0, n, max(n // 96, 1))
    for i in range(3):
        ranks[pos[i::3]] = spread[i]
    keys = ranks * GOLD + np.uint64(12345) if wide else ranks.copy()
    cls = key_class(ranks)
    cls[ranks == spread[0]], cls[ranks == spread[1]], cls[ranks == spread[2]] = NEGZ, NAN, BOTHINF
    if wide and n >= 2:
        at = rng.choice(np.setdiff1d(np.arange(n), pos), size=max(2, n // 4096), replace=False)
        keys[at[0::2]], keys[at[1::2]] = np.uint64(0), np.uint64(EMPTY_KEY)
        cls[at] = NEGZ
    ints = rng.integers(-(1 << 20), 1 << 20, n, endpoint=True)
    vals = np.ldexp(ints.astype(np.float64), -30)
    vals[cls == NEGZ] = -0.0
    z = cls == ZEROS
    vals[z] = np.where(rng.random(int(z.sum())) < 0.5, 0.0, -0.0)
    c = (cls == CANCEL) & (rng.random(n) < 0.3)
    vals[c], ints[c] = -0.0, 0
    vals[cls == PINF] = np.inf
    vals[cls == NINF] = -np.inf
    s = cls == SUB
    vals[s] = np.ldexp(ints[s].astype(np.float64), -1074)
    o = cls == OVF
    vals[o] = np.where(rng.random(int(o.sum())) < 0.5, 1.5e308, -1.5e308)
    # per-key fix-ups on each key's first and last row (in row order)
    order = np.argsort(keys, kind="stable")
    starts = np.flatnonzero(np.r_[True, keys[order][1:] != keys[order][:-1]])
    ends = np.r_[starts[1:], n]
    first, last = order[starts], order[ends - 1]
    kc = cls[first]
    sel = kc == CANCEL
    tot = np.add.reduceat(np.where(cls[order] == CANCEL, ints[order], 0), starts)[sel]
    lr = last[sel]
    vals[lr] = -np.ldexp((tot - ints[lr]).astype(np.float64), -30)
    f = first[kc == NAN]
    vals.view(np.uint64)[f] = rng.choice(np.array(NAN_BITS, dtype=np.uint64), len(f))
    vals[first[(kc == BOTHINF) | (kc == INF_FIN)]] = np.inf
    vals[last[kc == BOTHINF]] = -np.inf
    return keys, vals, cls


def lenient(keys, cls):
    return set(np.ascontiguousarray(keys).view(np.uint64)[cls == OVF].tolist())


def sums_of(parts):
    return [dict(zip(np.ascontiguousarray(k).view(np.uint64).tolist(), np.asarray(c).tolist())) for k, c in parts]


def assert_sharp_keys(got_parts, keys, cls):
    """The cases the file is about are in the input and came out as the reference pins them (assert_f64_sums checks
    every key; this names the first failure by case)."""
    got = {k: v for d in got_parts for k, v in d.items()}
    k = np.ascontiguousarray(keys).view(np.uint64)
    negz = set(k[cls == NEGZ].tolist())
    assert negz and (cls == NAN).any()
    wrong = [hex(x) for x in negz if np.float64(got[x]).view(np.uint64) != np.uint64(1 << 63)]
    assert not wrong, f"{len(wrong)} all -0.0 keys do not sum to -0.0: {wrong[:5]}"


# ---- integer reduce_by_key SUM over every hash-aggregate path ---------------------------------------------------------
@pytest.mark.parametrize("path", list(RP.PATHS))
def test_reduce_paths(sc, path):
    data = "hot_key_cache" if path == "register_hot" else path
    n, nkeys, hot, R = RP.PATHS[data]
    rng = np.random.default_rng([sorted(set(RP.PATHS) - {"register_hot"}).index(data), 71])
    keys, vals, cls = sharp_pairs(rng, n, nkeys, hot)
    assert {0, EMPTY_KEY} <= set(keys[cls == NEGZ].tolist())
    if hot:
        u, cnt = np.unique(keys, return_counts=True)
        assert cls[keys == u[np.argmax(cnt)]][0] == NEGZ and cnt.max() > 0.05 * n
    parts, _ = RP._run_path(sc, path, "sum", "f64", keys, vals, n, R)
    got = sums_of(parts)
    assert_sharp_keys(got, keys, cls)
    assert_f64_sums(got, keys, vals, R, lenient=lenient(keys, cls))


@pytest.mark.parametrize("R", [1, 257, 65536])
def test_reduce_partition_counts(sc, R):
    rng = np.random.default_rng([R, 72])
    keys, vals, cls = sharp_pairs(rng, 200_000, 60_000)
    parts, _ = RP.run_reduce(sc, "sum", "f64", _Col(keys), _Col(vals, role="value"), len(keys), 3, R)
    got = sums_of(parts)
    assert_sharp_keys(got, keys, cls)
    assert_f64_sums(got, keys, vals, R, lenient=lenient(keys, cls))


@pytest.mark.parametrize("R", [7, 300])
def test_reduce_four_byte_keys(sc, R):
    """i32 keys: rank 0 is -1, widened to the empty marker (the special slot), all -0.0."""
    rng = np.random.default_rng([R, 73])
    ranks, vals, cls = sharp_pairs(rng, 120_000, 3000, wide=False)
    k32 = (ranks.astype(np.int64) - 1).astype(np.int32)
    wide = k32.astype(np.int64).view(np.uint64)
    assert EMPTY_KEY in set(wide[cls == NEGZ].tolist())
    kc = _Col(k32)
    assert kc.key_width == 4
    parts, _ = RP.run_reduce(sc, "sum", "f64", kc, _Col(vals, role="value"), len(k32), 3, R, key_width=4)
    got = sums_of(parts)
    assert_sharp_keys(got, wide, cls)
    assert_f64_sums(got, wide, vals, R, key_width=4, lenient=lenient(wide, cls))


# ---- combine_by_key: SUM, MEAN, MIN and MAX of the sharp column next to an exact column ---------------------------------
SPEC = ([("f64", "exact"), ("f64", "sharp")],
        [("sum", 1), ("mean", 1), ("min", 1), ("max", 1), ("sum", 0), ("mean", 0)])


def sharp_cols(rng, n, nkeys, hot=0.0):
    keys, vals, cls = sharp_pairs(rng, n, nkeys, hot)
    exact = np.ldexp(rng.integers(-(1 << 20), 1 << 20, n, endpoint=True).astype(np.float64), -30)
    return keys, [exact, vals], cls


@pytest.mark.parametrize("path", list(CB.PATHS))
def test_combine_paths(sc, path):
    """SUM and MEAN against the reference (bit for bit where it pins one value), MIN and MAX bit for bit against the
    oracle's single-column shuffle."""
    data = "hot_key_cache" if path == "register_hot" else path
    n, nkeys, hot, _ = CB.PATHS[data]
    keys, cols, cls = sharp_cols(np.random.default_rng([sorted(CB.PATHS).index(data), 74]), n, nkeys, hot)
    parts, R = CB._run_path(sc, path, SPEC, keys, cols)
    assert_sharp_keys([dict(zip(k.view(np.uint64).tolist(), o[0].tolist())) for k, o in parts], keys, cls)
    CB.check_combine(parts, SPEC, keys, cols, R, lenient=lenient(keys, cls))


# ---- across ranks, in one process ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [2, 3, 8])
def test_reduce_across_ranks(sc, W):
    """12 map tasks; the spread keys' partials: -0.0 on every rank, NaN on rank 0 only, +inf on rank 0 and -inf on
    the last rank."""
    rng = np.random.default_rng([W, 75])
    keys, vals, cls = sharp_pairs(rng, 300_000, 50_000)
    M, R = 12, 2 * W + 1
    parts, _, _ = shuffle_ranks(vdist.CudaEngine(sc), W, "sum", "f64", keys, vals, M, R,
                                place="device" if W == 3 else "host")
    got = sums_of(parts)
    assert_sharp_keys(got, keys, cls)
    assert_f64_sums(got, keys, vals, R, lenient=lenient(keys, cls))


@pytest.mark.parametrize("W", [2, 3, 8])
def test_combine_across_ranks(sc, W):
    keys, cols, cls = sharp_cols(np.random.default_rng([W, 76]), 300_000, 50_000)
    M, R = 12, 2 * W + 1
    parts, shs, _, _ = combine_ranks(sc, W, SPEC, keys, cols, M, R, loc="device" if W == 3 else "host")
    free_all(shs)
    CB.check_combine(parts, SPEC, keys, cols, R, lenient=lenient(keys, cls))


# ---- String keys ----------------------------------------------------------------------------------------------------
def str_data(seed, n=120_000, n_keys=8000):
    """sharp_pairs over String keys "f<rank>" with warps of one key at the start: (names per row, values, classes,
    rank of each row)."""
    ranks, vals, cls = sharp_pairs(np.random.default_rng(seed), n, n_keys, hot=0.1, wide=False, runs=True)
    names = [f"f{r}" for r in ranks.tolist()]
    return names, vals, cls, ranks


def by_rank(parts, a=None):
    """[{String key: value or tuple}] -> [{rank: value}] (keys are "f<rank>")."""
    return [{int(k[1:]): (v if a is None else v[a]) for k, v in p.items()} for p in parts]


def check_str(got_parts, ranks, vals, cls, mean=False):
    got = {k: v for d in got_parts for k, v in d.items()}
    wrong = [k for k in set(ranks[cls == NEGZ].tolist()) if np.float64(got[k]).view(np.uint64) != np.uint64(1 << 63)]
    assert not wrong, f"{len(wrong)} all -0.0 keys do not {'average' if mean else 'sum'} to -0.0: {wrong[:5]}"
    F.assert_outcomes(got, F.key_outcomes(ranks, vals, mean=mean), "f64 means" if mean else "f64 sums",
                      lenient=lenient(ranks, cls))


@pytest.mark.parametrize("W", [1, 2, 3, 8])
def test_str_reduce(sc, W):
    """reduce_by_key SUM over String keys (W = 1: one process; else export, import and seal on W ranks)."""
    names, vals, cls, ranks = str_data([W, 77])
    M, R = 12, 2 * W + 1
    shs = str_ranks(sc, W, "sum", "f64", names, vals, M, R, where="device" if W == 3 else "host")
    got = by_rank(str_owned(shs, "sum", R))
    free_all(shs)
    check_str(got, ranks, vals, cls)


STR_MULTI = ([L.VB_F64, L.VB_F64], [(L.VB_AGG_SUM, 1), (L.VB_AGG_MEAN, 1), (L.VB_AGG_MIN, 1), (L.VB_AGG_SUM, 0)])
STR_OUTS = [np.float64] * 4


def test_str_combine_one_process(sc):
    """The String combine with five accumulators (the MEAN's COUNT included): SUM and MEAN of the sharp column."""
    names, vals, cls, ranks = str_data(78)
    exact = np.ldexp(np.random.default_rng(79).integers(-(1 << 20), 1 << 20, len(vals)).astype(np.float64), -30)
    M, R = 4, 5
    kc, _ = columns(names, None, "host")
    vcs = (_Col(exact, role="value"), _Col(vals, role="value"))
    starts = vb.slice_starts(len(names), M)
    sh = StrShuffle(sc, M, R, L.VB_U64, L.VB_AGG_SUM, multi=STR_MULTI)
    try:
        for m in range(M):
            sh.map_cols(m, kc, vcs, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        parts = [decode(sh.reduce_cols(r, STR_OUTS)) for r in range(R)]
    finally:
        sh.free()
    check_str(by_rank(parts, 0), ranks, vals, cls)
    check_str(by_rank(parts, 1), ranks, vals, cls, mean=True)
    F.assert_outcomes({k: v for d in by_rank(parts, 3) for k, v in d.items()}, F.key_outcomes(ranks, exact), exact=True)


@pytest.mark.parametrize("W", [2, 3, 8])
def test_str_combine_across_ranks(sc, W):
    names, vals, cls, ranks = str_data([W, 80])
    exact = np.ldexp(np.random.default_rng([W, 81]).integers(-(1 << 20), 1 << 20, len(vals)).astype(np.float64), -30)
    M, R = 12, 2 * W + 1
    shs, _ = run_world(sc, W, STR_MULTI, names, [exact, vals], M, R, where="device" if W == 3 else "host")
    parts = str_combine_owned(shs, R, STR_OUTS)
    free_all(shs)
    check_str(by_rank(parts, 0), ranks, vals, cls)
    check_str(by_rank(parts, 1), ranks, vals, cls, mean=True)


# ---- blobs: CPU-encoded buckets of f64 SUM partials, mixed with row map tasks ------------------------------------------
def test_blob_partials(sc):
    """Maps 0 and 2 as rows, 1 and 3 as CPU-encoded buckets whose partials (each key's values of the map folded from
    the first, as vega's combiner does) include -0.0, NaN and +-inf.  The reduce is checked against the reference
    over the row values and the partials; vb_shuffle_reduce_blob re-encodes every partition byte for byte."""
    names, vals, cls, ranks = str_data(82, n=40_000, n_keys=3000)
    M, R = 4, 5
    starts = vb.slice_starts(len(names), M)
    kc, vc = columns(names, vals, "host")
    sh = StrShuffle(sc, M, R, L.VB_F64, L.VB_AGG_SUM)
    ref_k, ref_v = [], []
    try:
        for m in range(M):
            lo, hi = int(starts[m]), int(starts[m + 1])
            if m % 2 == 0:
                sh.map(m, kc, vc, lo, hi)
                ref_k.append(ranks[lo:hi])
                ref_v.append(vals[lo:hi])
            else:
                blob = combined_blob(names[lo:hi], vals[lo:hi], "sum", "f64")
                pairs = B.decode_str_pairs(blob)
                ref_k.append(np.array([int(k[1:]) for k, _ in pairs], dtype=np.uint64))
                ref_v.append(np.array([c for _, c in pairs], dtype=np.uint64).view(np.float64))
                sh.map_blob(m, blob)
        sh.seal()
        partial = np.concatenate(ref_v)
        assert np.isnan(partial).any() and np.isinf(partial).any()
        assert (partial.view(np.uint64) == np.uint64(1 << 63)).any()
        parts = [dict(zip(*[x.tolist() for x in sh.reduce(r)[:2]])) for r in range(R)]
        for r in range(R):
            assert sh.reduce_blob(r) == B.encode_str_pairs(str_pairs(sh, r)), r
    finally:
        sh.free()
    rk = np.concatenate(ref_k)
    oc = F.key_outcomes(rk, partial)
    got = {k: v for d in by_rank(parts) for k, v in d.items()}
    wrong = [k for k in set(ranks[cls == NEGZ].tolist()) if np.float64(got[k]).view(np.uint64) != np.uint64(1 << 63)]
    assert not wrong, f"{len(wrong)} all -0.0 keys do not sum to -0.0: {wrong[:5]}"
    F.assert_outcomes(got, oc, lenient=lenient(ranks, cls))
