"""Reference outer joins for the tests (test infrastructure).

vega has no outer joins, so there is no reference output to compare against.  These restate Spark's leftOuterJoin /
rightOuterJoin / fullOuterJoin over vega's cogroup (oracle/pyref.py:cogroup, co_grouped_rdd.rs:206-249).  For a key with
left values vs and right values ws, each in cogroup order (map-id order, then encounter order):

    key on both sides      for v in vs { for w in ws } -> (k, (v, w))    every kind
    key only on the left   (k, (v, None)) for each v                    left, full
    key only on the right  (k, (None, w)) for each w                    right, full

`outer_join` works on arbitrary keys and values (small cases).  `outer_join_parts` handles arrays too large for pure
Python: the matched rows come from the C oracle's inner join, the unmatched rows of a kept side from numpy, in input
order.
"""
import numpy as np

from oracle import oracle as O
from oracle import pyref as P

KEEP = {"left": (True, False), "right": (False, True), "full": (True, True)}


def outer_join(kind, rows_a, slices_a, rows_b, slices_b, n_reduce, int_width=8):
    keep_l, keep_r = KEEP[kind]
    out = []
    for k, (vs, ws) in P.cogroup(rows_a, slices_a, rows_b, slices_b, n_reduce, int_width):
        if vs and ws:
            out += [(k, (v, w)) for v in vs for w in ws]
        elif vs and keep_l:
            out += [(k, (v, None)) for v in vs]
        elif ws and keep_r:
            out += [(k, (None, w)) for w in ws]
    return out


def left_outer_join(rows_a, slices_a, rows_b, slices_b, n_reduce, int_width=8):
    return outer_join("left", rows_a, slices_a, rows_b, slices_b, n_reduce, int_width)


def right_outer_join(rows_a, slices_a, rows_b, slices_b, n_reduce, int_width=8):
    return outer_join("right", rows_a, slices_a, rows_b, slices_b, n_reduce, int_width)


def full_outer_join(rows_a, slices_a, rows_b, slices_b, n_reduce, int_width=8):
    return outer_join("full", rows_a, slices_a, rows_b, slices_b, n_reduce, int_width)


def _u64(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64) if a.dtype.itemsize == 8 else a.astype(np.int64).view(np.uint64)


def key_partitions(keys, n_reduce, key_width=8):
    """HashPartitioner partition of every key (the C oracle places the distinct keys)."""
    keys = _u64(keys)
    uniq, inv = np.unique(keys, return_inverse=True)
    part = np.zeros(len(uniq), dtype=np.int64)
    for r, p in enumerate(O.shuffle("count", uniq, None, 1, n_reduce, key_width=key_width)):
        part[np.searchsorted(uniq, p["keys"])] = r
    return part[inv]


def unmatched_rows(kind, ka, va, kb, vb, n_reduce, key_width=8):
    """Per partition, the rows of keys on one side only that the kind keeps, in input order, as u64 arrays
    (k, v, w, v_valid, w_valid) with 0 in a None slot."""
    keep_l, keep_r = KEEP[kind]
    ka, va, kb, vb = _u64(ka), _u64(va), _u64(kb), _u64(vb)
    parts = []
    sides = []
    if keep_l:
        only = ~np.isin(ka, kb)
        sides.append((ka[only], va[only], key_partitions(ka[only], n_reduce, key_width) if only.any() else np.zeros(0, np.int64), True))
    if keep_r:
        only = ~np.isin(kb, ka)
        sides.append((kb[only], vb[only], key_partitions(kb[only], n_reduce, key_width) if only.any() else np.zeros(0, np.int64), False))
    for r in range(n_reduce):
        k, v, w, vv, wv = [], [], [], [], []
        for keys, vals, part, is_left in sides:
            sel = part == r
            n = int(sel.sum())
            zero, one = np.zeros(n, np.uint64), np.ones(n, np.uint8)
            k.append(keys[sel])
            v.append(vals[sel] if is_left else zero)
            w.append(zero if is_left else vals[sel])
            vv.append(one if is_left else one * 0)
            wv.append(one * 0 if is_left else one)
        cat = lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dt)
        parts.append((cat(k, np.uint64), cat(v, np.uint64), cat(w, np.uint64), cat(vv, np.uint8), cat(wv, np.uint8)))
    return parts


def outer_join_parts(kind, ka, va, slices_a, kb, vb, slices_b, n_reduce, key_width=8):
    """Per reduce partition, {key: [(v, w, v_valid, w_valid), ...]} in the nesting order above (u64 bits, 0 for None):
    matched rows from oracle.join, then the unmatched rows of a kept side."""
    inner = O.join(_u64(ka), _u64(va), slices_a, _u64(kb), _u64(vb), slices_b, n_reduce, key_width=key_width)
    extra = unmatched_rows(kind, ka, va, kb, vb, n_reduce, key_width)
    out = []
    for (k, v, w), (k2, v2, w2, vv2, wv2) in zip(inner, extra):
        d = {}
        for a, b, c in zip(k.tolist(), v.tolist(), w.tolist()):
            d.setdefault(a, []).append((b, c, 1, 1))
        for a, b, c, x, y in zip(k2.tolist(), v2.tolist(), w2.tolist(), vv2.tolist(), wv2.tolist()):
            assert a not in d or d[a][0][2:] == (x, y), "a key both matched and unmatched"
            d.setdefault(a, []).append((b, c, x, y))
        out.append(d)
    return out
