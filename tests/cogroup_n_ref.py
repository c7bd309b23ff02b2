"""References of the cogroup and inner join of any number of parents (test infrastructure).

cogroup_n / join_n restate CoGroupedRdd::compute (src/rdd/co_grouped_rdd.rs:206-249) for n parents on Python rows.
ref_parts_n is the array reference the GPU tests use: each side's C-oracle group shuffle, joined by key union.
assert_cogroup_n_equal compares device partitions with numpy (key, position, value) triples per side (tests/group_ref.py)
for inputs too large for either of the others.
"""
import itertools

import numpy as np

from oracle import pyref as P
from tests import group_ref as G
from tests.test_gpu_cogroup import _group


def cogroup_n(parents, n_reduce, int_width=8):
    """CoGroupedRdd::compute with parents [(rows, num_slices), ...]: each parent is shuffled with the Vec-append
    aggregator (:78-124); per partition, the deps in order and each dep's map outputs in map-id order extend the key's
    list of that dep, every key starting from vec![Vec::new(); n]."""
    agg = P.Aggregator.default()
    outs = [[P.map_task(s, n_reduce, agg, int_width) for s in P.slice_(rows, ns)] for rows, ns in parents]
    res = []
    for r in range(n_reduce):
        g = {}
        for dep_num, dep in enumerate(outs):
            for m in range(len(dep)):
                for k, vals in dep[m][r]:
                    g.setdefault(k, [[] for _ in parents])[dep_num].extend(vals)
        res.extend(g.items())
    return res


def join_n(parents, n_reduce, int_width=8):
    """Inner join of all parents: per key on every parent, for v0 in l0 { for v1 in l1 { ... } } -> (k, [v0, v1, ...])."""
    return [(k, list(row)) for k, lists in cogroup_n(parents, n_reduce, int_width) for row in itertools.product(*lists)]


def ref_parts_n(sides, R, key_width=8):
    """sides [(keys, vals, num_slices), ...] -> per partition {key: (list of side 0, list of side 1, ...)} (u64 bits),
    the union of every side's keys, [] where a side lacks the key."""
    groups = [_group(k, v, M, R, key_width) for k, v, M in sides]
    out = []
    for r in range(R):
        keys = set().union(*(g[r].keys() for g in groups))
        out.append({k: tuple(g[r].get(k, []) for g in groups) for k in keys})
    return out


def join_of_parts(parts):
    """The inner join of cogroup partitions: per partition {key: [row tuples in nested order]}, keys on every side."""
    return [{k: list(itertools.product(*lists)) for k, lists in d.items() if all(lists)} for d in parts]


def assert_cogroup_n_equal(parts, sides, R, key_width=8):
    """parts[r] = (keys, [(offsets, values) per side]); sides [(keys, values), ...]: every key of any side once, in its
    partition, no key with every list empty, and each side's lists equal group_by_key of that side."""
    assert len(parts) == R
    keys = []
    for r, (k, lists) in enumerate(parts):
        empty = np.ones(len(k), dtype=bool)
        for o, _ in lists:
            empty &= np.diff(np.asarray(o).astype(np.int64)) == 0
        assert not empty.any(), f"partition {r}: a key with every list empty"
        keys.append(G.u64(k))
    keys = np.sort(np.concatenate(keys)) if keys else np.zeros(0, np.uint64)
    want = np.unique(np.concatenate([G.u64(k) for k, _ in sides]))
    assert len(keys) == len(want) and np.array_equal(keys, want), f"{len(keys)} keys, want {len(want)} (the union, each once)"
    for j, (k, v) in enumerate(sides):
        got = G.csr_triples([(p[0], p[1][j][0], p[1][j][1]) for p in parts], R, key_width, allow_empty=True)
        G.assert_rows_equal(got, G.group_triples(k, v), G.GROUP_COLS)
