"""Vectorised references of group_by_key, cogroup and the joins (test infrastructure), exact at tens of millions of rows.

The map tasks of a shuffle are contiguous ParallelCollection slices, fetched in map-id order, so every key's value
list is its values in input order, whatever the number of map tasks.  A grouped result is therefore one
(key, position in the key's list, value) triple per row, and two results are equal when their triples, ordered by key
then position, are equal.  The order of keys inside a partition is unspecified and is not compared.

Joins: for a key with left values vs and right values ws (each in that order), the rows are
    key on both sides      for v in vs { for w in ws } -> (k, v, w)    every kind
    key only on the left   (k, v, None) for each v                    left, full
    key only on the right  (k, None, w) for each w                    right, full
and a join result is one (key, position among the key's rows, v, w, v valid, w valid) row per output row, None as
0 with valid 0.

Placement is HashPartitioner's: MetroHash64_1 (seed 0) of the key's 8 or 4 little-endian bytes, modulo R.
tests/test_group_ref_cpu.py pins every function here to the C oracle and to oracle/pyref.py on small inputs.
"""
import numpy as np

MASK64 = (1 << 64) - 1
_K0, _K1, _K2, _K3 = 0xC83A91E1, 0x8648DBDB, 0x7BDEC03B, 0x2F5870A5
KEEP = {"inner": (False, False), "left": (True, False), "right": (False, True), "full": (True, True)}


def u64(a):
    """The 64-bit pattern of an integer or f64 array; 4-byte integers widened as _Col widens them (sign-extended)."""
    a = np.ascontiguousarray(a)
    if a.dtype.itemsize == 8:
        return a.view(np.uint64)
    return a.astype(np.int64 if a.dtype.kind == "i" else np.uint64).view(np.uint64)


def _rotr(v, k):
    return (v >> np.uint64(k)) | (v << np.uint64(64 - k))


def metrohash64_1(keys, key_width=8):
    """MetroHash64_1 with seed 0 of every key's key_width little-endian bytes (the low 4 for key_width 4)."""
    k = u64(keys)
    K0, K1, K3 = np.uint64(_K0), np.uint64(_K1), np.uint64(_K3)
    h0 = np.uint64((_K2 * _K0 + key_width) & MASK64)        # ((seed + k2) * k0) + len
    if key_width == 8:
        h = h0 + k * K3
        h ^= _rotr(h, 33) * K1
    else:
        assert key_width == 4, key_width
        h = h0 + (k & np.uint64(0xFFFFFFFF)) * K3
        h ^= _rotr(h, 15) * K1
    h ^= _rotr(h, 33)
    h *= K0
    h ^= _rotr(h, 33)
    return h


def partition_of(keys, R, key_width=8):
    return (metrohash64_1(keys, key_width) % np.uint64(R)).astype(np.int64)


def runs(sorted_keys):
    """(distinct keys, start of each run, length of each run) of a sorted key array."""
    n = len(sorted_keys)
    if n == 0:
        return sorted_keys[:0], np.zeros(0, np.int64), np.zeros(0, np.int64)
    starts = np.flatnonzero(np.r_[True, sorted_keys[1:] != sorted_keys[:-1]])
    return sorted_keys[starts], starts, np.diff(np.r_[starts, n])


def _positions(lengths):
    """Position of every element inside its run, for back-to-back runs of these lengths."""
    lengths = np.asarray(lengths, dtype=np.int64)
    return np.arange(int(lengths.sum()), dtype=np.int64) - np.repeat(np.cumsum(lengths) - lengths, lengths)


def group_triples(keys, vals):
    """group_by_key of the rows: (key, position, value) per row, ordered by key then position."""
    k, v = u64(keys), u64(vals)
    order = np.argsort(k, kind="stable")
    ks = k[order]
    return ks, _positions(runs(ks)[2]), v[order]


def _member(sorted_unique, x):
    """x[i] in sorted_unique, for every i."""
    if len(sorted_unique) == 0:
        return np.zeros(len(x), dtype=bool)
    i = np.minimum(np.searchsorted(sorted_unique, x), len(sorted_unique) - 1)
    return sorted_unique[i] == x


def _by_key_then_pos(cols):
    order = np.lexsort((cols[1], cols[0]))
    return tuple(c[order] for c in cols)


def join_rows(kind, ka, va, kb, vb):
    """The rows of an inner ("inner") or outer ("left" / "right" / "full") join as
    (key, position, v, w, v_valid, w_valid), ordered by key then position."""
    keep_l, keep_r = KEEP[kind]
    lk, lp, lv = group_triples(ka, va)
    rk, rp, rv = group_triples(kb, vb)
    ul, ls, lc = runs(lk)
    ur, rs, rc = runs(rk)
    _, il, ir = np.intersect1d(ul, ur, assume_unique=True, return_indices=True)
    m = lc[il] * rc[ir]                                   # rows per shared key
    pos = _positions(m)
    per_w = np.repeat(rc[ir], m)
    pieces = [(np.repeat(ul[il], m), pos, lv[np.repeat(ls[il], m) + pos // per_w], rv[np.repeat(rs[ir], m) + pos % per_w],
               np.ones(len(pos), np.uint8), np.ones(len(pos), np.uint8))]
    zero = lambda n: np.zeros(n, np.uint64)
    if keep_l:
        only = ~_member(ur, lk)
        n = int(only.sum())
        pieces.append((lk[only], lp[only], lv[only], zero(n), np.ones(n, np.uint8), np.zeros(n, np.uint8)))
    if keep_r:
        only = ~_member(ul, rk)
        n = int(only.sum())
        pieces.append((rk[only], rp[only], zero(n), rv[only], np.zeros(n, np.uint8), np.ones(n, np.uint8)))
    cols = [np.concatenate([p[i] for p in pieces]) for i in range(6)]
    cols[1] = cols[1].astype(np.int64)
    return _by_key_then_pos(cols)


# ---- turning device results into the same form -------------------------------------------------------------------
def _check_placement(keys, r, R, key_width, what):
    bad = np.flatnonzero(partition_of(keys, R, key_width) != r)
    assert not len(bad), f"{what}: {len(bad)} keys of partition {r} hash elsewhere, first {int(keys[bad[0]]):#x}"


def csr_triples(parts, R, key_width=8, allow_empty=False):
    """parts[r] = (keys, offsets, values) of reduce partition r, as a group shuffle returns them.  Checks the CSR and
    that every key hashes to its partition; returns (key, position, value) per value, ordered by key then position.
    allow_empty: a key may have an empty list (one side of a cogroup)."""
    assert len(parts) == R, (len(parts), R)
    ks, ps, vs = [], [], []
    for r, (k, o, v) in enumerate(parts):
        k, v = u64(k), u64(v)
        o = np.asarray(o).astype(np.int64)
        assert len(o) == len(k) + 1 and o[0] == 0 and o[-1] == len(v), f"partition {r}: bad CSR bounds"
        cnt = np.diff(o)
        assert (cnt >= 0).all(), f"partition {r}: offsets are not monotone"
        assert allow_empty or (cnt > 0).all(), f"partition {r}: a key with an empty list"
        _check_placement(k, r, R, key_width, "group")
        ks.append(np.repeat(k, cnt))
        ps.append(_positions(cnt))
        vs.append(v)
    cat = lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dt)
    return _by_key_then_pos((cat(ks, np.uint64), cat(ps, np.int64), cat(vs, np.uint64)))


def join_output_rows(parts, R, key_width=8):
    """parts[r] = (k, v, w, v_valid, w_valid) of join partition r.  Checks that each key's rows are one contiguous run
    and that every key hashes to its partition; returns the rows as join_rows does."""
    assert len(parts) == R, (len(parts), R)
    cols = [[] for _ in range(6)]
    for r, (k, v, w, vv, wv) in enumerate(parts):
        k = u64(k)
        uk, _, lengths = runs(k)
        assert len(np.unique(uk)) == len(uk), f"partition {r}: the rows of a key are not contiguous"
        _check_placement(uk, r, R, key_width, "join")
        for c, x in zip(cols, (k, _positions(lengths), u64(v), u64(w), np.asarray(vv, np.uint8), np.asarray(wv, np.uint8))):
            c.append(x)
    cols = [np.concatenate(c) for c in cols]
    cols[1] = cols[1].astype(np.int64)
    return _by_key_then_pos(cols)


def assert_rows_equal(got, want, names):
    """Equal column tuples (each ordered by key then position); reports the first row that differs."""
    assert len(got) == len(want) == len(names)
    n_got, n_want = len(got[0]), len(want[0])
    if n_got == n_want and all(np.array_equal(g, w) for g, w in zip(got, want)):
        return
    n = min(n_got, n_want)
    diff = np.zeros(n, dtype=bool)
    for g, w in zip(got, want):
        diff |= g[:n] != w[:n]
    i = int(np.flatnonzero(diff)[0]) if diff.any() else n
    row = lambda cols: {nm: (int(c[i]) if i < len(c) else None) for nm, c in zip(names, cols)}
    raise AssertionError(f"{n_got} rows, want {n_want}; {int(diff.sum())} of the first {n} differ; first at row {i}: "
                         f"got {row(got)}, want {row(want)}")


GROUP_COLS = ("key", "pos", "value")
JOIN_COLS = ("key", "pos", "v", "w", "v_valid", "w_valid")


def assert_group_equal(parts, keys, vals, R, key_width=8):
    """A group shuffle's partitions against group_by_key of (keys, vals): every key, its partition, its list."""
    assert_rows_equal(csr_triples(parts, R, key_width), group_triples(keys, vals), GROUP_COLS)


def assert_cogroup_equal(parts, ka, va, kb, vb, R, key_width=8):
    """parts[r] = (keys, (left offsets, left values), (right offsets, right values)): every key of either side once,
    in its partition, with both lists; no key with two empty lists."""
    assert len(parts) == R
    keys = []
    for r, (k, (lo, _), (ro, _)) in enumerate(parts):
        both_empty = (np.diff(np.asarray(lo).astype(np.int64)) == 0) & (np.diff(np.asarray(ro).astype(np.int64)) == 0)
        assert not both_empty.any(), f"partition {r}: a key with two empty lists"
        keys.append(u64(k))
    keys = np.sort(np.concatenate(keys)) if keys else np.zeros(0, np.uint64)
    want = np.union1d(u64(ka), u64(kb))
    assert len(keys) == len(want) and np.array_equal(keys, want), \
        f"{len(keys)} keys, want {len(want)} (the union of both sides, each once)"
    for side, (k, v) in ((1, (ka, va)), (2, (kb, vb))):
        got = csr_triples([(p[0], p[side][0], p[side][1]) for p in parts], R, key_width, allow_empty=True)
        assert_rows_equal(got, group_triples(k, v), GROUP_COLS)
