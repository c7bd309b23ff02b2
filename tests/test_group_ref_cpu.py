"""tests/group_ref.py against what the suite already trusts: the C oracle's group shuffle and inner join, the outer
joins of tests/outer_join_ref.py, oracle/pyref.py's cogroup, and the oracle's HashPartitioner.  Small random inputs
with duplicated keys, keys 0 and 2^64-1, several map tasks and R in {1, 7, 300}."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import pyref as P
from tests import group_ref as G
from tests.outer_join_ref import outer_join_parts
from tests.util import EMPTY_KEY

R_VALUES = [1, 7, 300]


def _pairs(rng, n, n_keys):
    """n rows over n_keys keys (0 and 2^64-1 among them), full-range i64 values."""
    pool = rng.integers(0, 1 << 64, n_keys, dtype=np.uint64)
    pool[:2] = [0, EMPTY_KEY]
    keys = pool[rng.integers(0, n_keys, n)]
    keys[rng.choice(n, 2, replace=False)] = pool[:2]
    vals = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
    return keys, vals


def _oracle_group_parts(keys, vals, M, R):
    return [(p["keys"], p["offsets"], p["vals"]) for p in O.shuffle("group", keys, vals.view(np.uint64), M, R)]


@pytest.mark.parametrize("R", R_VALUES)
@pytest.mark.parametrize("M", [1, 3])
def test_group_matches_oracle(R, M):
    rng = np.random.default_rng([R, M])
    keys, vals = _pairs(rng, 3000, 400)
    G.assert_group_equal(_oracle_group_parts(keys, vals, M, R), keys, vals, R)


def test_group_mismatches_are_caught():
    """A swapped pair of values inside one list, a key moved to another partition and a list split in two all fail."""
    rng = np.random.default_rng(9)
    keys, vals = _pairs(rng, 2000, 50)
    R = 7
    parts = _oracle_group_parts(keys, vals, 2, R)
    k, o, v = parts[0]
    swapped = v.copy()
    swapped[[0, 1]] = swapped[[1, 0]]
    assert o[1] >= 2 and swapped[0] != swapped[1]
    with pytest.raises(AssertionError):
        G.assert_group_equal([(k, o, swapped)] + parts[1:], keys, vals, R)
    with pytest.raises(AssertionError, match="hash elsewhere"):
        G.assert_group_equal([parts[1]] + [parts[0]] + parts[2:], keys, vals, R)
    split = (np.r_[k[:1], k], np.r_[o[:1], o[:1] + 1, o[1:]], v)       # key 0's list as two lists
    with pytest.raises(AssertionError):
        G.assert_group_equal([split] + parts[1:], keys, vals, R)


def _oracle_inner(ka, va, Ma, kb, vb, Mb, R):
    return [(k, v, w, np.ones(len(k), np.uint8), np.ones(len(k), np.uint8))
            for k, v, w in O.join(ka, va.view(np.uint64), Ma, kb, vb.view(np.uint64), Mb, R)]


def _join_inputs(R):
    rng = np.random.default_rng([R, 2])
    ka, va = _pairs(rng, 1500, 300)
    kb, vb = _pairs(rng, 1200, 300)
    kb[:] = rng.choice(np.unique(ka), len(kb))            # shared keys with several rows on each side
    only_r = rng.random(len(kb)) < 0.2
    kb[only_r] = rng.integers(0, 1 << 64, int(only_r.sum()), dtype=np.uint64)      # keys on the right only
    kb[rng.random(len(kb)) < 0.05] = np.uint64(12345)     # and one of them with many rows
    keep = kb % np.uint64(4) != 1                         # about a quarter of the left keys on the left only
    return ka, va, kb[keep], vb[keep]


@pytest.mark.parametrize("R", R_VALUES)
def test_inner_join_matches_oracle(R):
    ka, va, kb, vb = _join_inputs(R)
    got = G.join_output_rows(_oracle_inner(ka, va, 3, kb, vb, 2, R), R)
    assert len(got[0]) > len(ka) // 2
    G.assert_rows_equal(got, G.join_rows("inner", ka, va, kb, vb), G.JOIN_COLS)


@pytest.mark.parametrize("R", R_VALUES)
@pytest.mark.parametrize("kind", ["left", "right", "full"])
def test_outer_joins_match_outer_join_ref(kind, R):
    ka, va, kb, vb = _join_inputs(R)
    parts = []
    for d in outer_join_parts(kind, ka, va, 3, kb, vb, 2, R):
        rows = [(k,) + x for k, xs in d.items() for x in xs]
        cols = [np.array([r[i] for r in rows], dtype=np.uint64) for i in range(5)]
        parts.append(tuple(cols[:3]) + (cols[3].astype(np.uint8), cols[4].astype(np.uint8)))
    want = G.join_rows(kind, ka, va, kb, vb)
    assert {(1, 0), (0, 1)} & set(zip(want[4].tolist(), want[5].tolist()))
    G.assert_rows_equal(G.join_output_rows(parts, R), want, G.JOIN_COLS)


def test_join_nesting_order():
    """Two left and three right values of one key: for v in vs { for w in ws }."""
    ka, va = np.array([5, 9, 5], np.uint64), np.array([10, 11, 12], np.int64)
    kb, vb = np.array([5, 5, 7, 5], np.uint64), np.array([20, 21, 22, 23], np.int64)
    k, pos, v, w, vv, wv = G.join_rows("full", ka, va, kb, vb)
    assert list(zip(k.tolist(), pos.tolist(), v.tolist(), w.tolist(), vv.tolist(), wv.tolist())) == [
        (5, 0, 10, 20, 1, 1), (5, 1, 10, 21, 1, 1), (5, 2, 10, 23, 1, 1),
        (5, 3, 12, 20, 1, 1), (5, 4, 12, 21, 1, 1), (5, 5, 12, 23, 1, 1),
        (7, 0, 0, 22, 0, 1), (9, 0, 11, 0, 1, 0)]


@pytest.mark.parametrize("R", R_VALUES)
def test_cogroup_matches_pyref(R):
    rng = np.random.default_rng([R, 3])
    ka, va = _pairs(rng, 800, 150)
    kb, vb = _pairs(rng, 600, 200)
    rows = lambda k, v: list(zip(k.tolist(), v.view(np.uint64).tolist()))
    by_part = [[] for _ in range(R)]
    for k, (vs, ws) in P.cogroup(rows(ka, va), 3, rows(kb, vb), 2, R):
        by_part[O.get_partition(k, R)].append((k, vs, ws))
    parts = []
    for items in by_part:
        keys = np.array([k for k, _, _ in items], dtype=np.uint64)
        side = lambda i: (np.r_[0, np.cumsum([len(x[i]) for x in items])].astype(np.uint64),
                          np.array([v for x in items for v in x[i]], dtype=np.uint64))
        parts.append((keys, side(1), side(2)))
    G.assert_cogroup_equal(parts, ka, va, kb, vb, R)


@pytest.mark.parametrize("key_width", [8, 4])
def test_hash_matches_oracle_partitioner(key_width):
    rng = np.random.default_rng(key_width)
    if key_width == 8:
        keys = rng.integers(0, 1 << 64, 10_000, dtype=np.uint64)
        keys[:4] = [0, 1, 1 << 63, EMPTY_KEY]
    else:                                                   # i32 keys as _Col widens them: sign-extended to 64 bits
        keys = G.u64(rng.integers(-(1 << 31), 1 << 31, 10_000).astype(np.int32))
        keys[:4] = G.u64(np.array([0, -1, -(1 << 31), (1 << 31) - 1], dtype=np.int32))
    for R in (1, 7, 300, 65536):
        want = np.array([O.get_partition(k, R, key_width) for k in keys.tolist()])
        assert np.array_equal(G.partition_of(keys, R, key_width), want), R
    want_h = [O.metrohash64_1(int(k).to_bytes(8, "little")[:key_width]) for k in keys[:200].tolist()]
    assert G.metrohash64_1(keys[:200], key_width).tolist() == want_h
