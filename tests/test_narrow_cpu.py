"""CPU-side checks of reduce results as join and cogroup parents: the narrow restatement (each reduce partition cogrouped
where it is, no second shuffle) equals oracle/pyref.py's cogroup of the parents' reduce outputs, and the mirror's
argument errors are raised before any device work."""
import operator

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref as P
from tests import cogroup_n_ref as CN


def _reduce_parts(rows, f, num_slices, R, int_width=8):
    """ShuffledRdd::compute of every partition of reduce_by_key(f): [[(k, c), ...] per partition]."""
    agg = P.Aggregator.reducing(f)
    outs = [P.map_task(s, R, agg, int_width) for s in P.slice_(rows, num_slices)]
    return [P.reduce_task(r, outs, agg) for r in range(R)]


def _narrow_cogroup(parents, R):
    """The cogroup of reduce results under their own partitioner, partition by partition (the OneToOneDependency of
    co_grouped_rdd.rs:103-112): partition r's keys from every parent's partition r, each with the list [c]."""
    out = []
    for r in range(R):
        g = {}
        for j, parts in enumerate(parents):
            for k, c in parts[r]:
                g.setdefault(k, [[] for _ in parents])[j].append(c)
        out.append(g)
    return out


def _by_partition(items, R, int_width=8):
    out = [dict() for _ in range(R)]
    for k, lists in items:
        out[P.get_partition(k, R, int_width)][k] = [list(x) for x in lists]
    return out


@pytest.mark.parametrize("R", [1, 2, 4])
def test_narrow_restatement_equals_the_reference_cogroup(R):
    # tests/test_pair_rdd.rs:8-37 (test_group_by_key: "x" -> 1..7 and "y" -> 1..8, here keys 10 and 20) reduced with +,
    # and test_count_by_value's data (tests/test_pair_rdd.rs:84-109) counted; the file has no reduce_by_key test of its own
    a_rows = [(10, v) for v in range(1, 8)] + [(20, v) for v in range(1, 9)]
    b_rows = [(x, 1) for x in [1, 2, 1, 3, 2, 3, 3, 2, 3]] + [(10, 1)]
    a, b = _reduce_parts(a_rows, operator.add, 4, R), _reduce_parts(b_rows, operator.add, 2, R)
    want = P.cogroup([kc for p in a for kc in p], 1, [kc for p in b for kc in p], 3, R)   # the result rows as parents
    got = _narrow_cogroup([a, b], R)
    assert got == _by_partition(want, R)
    assert sorted((k, [list(x) for x in ls]) for d in got for k, ls in d.items()) == \
        [(1, [[], [2]]), (2, [[], [3]]), (3, [[], [4]]), (10, [[28], [1]]), (20, [[36], []])]
    # the join and the N-way restatement agree with it
    assert sorted(P.join([kc for p in a for kc in p], 2, [kc for p in b for kc in p], 1, R)) == [(10, (28, 1))]
    assert _by_partition(CN.cogroup_n([([kc for p in a for kc in p], 3), ([kc for p in b for kc in p], 2)], R), R) == got


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_mirror_argument_errors_before_device_work():
    ctx = _NoDevice()
    k64, k32 = np.arange(5, dtype=np.uint64), np.arange(5, dtype=np.int32)
    a = vb.Context.parallelize(ctx, (k64, k64), 2)
    s = a.reduce_by_key("sum", 3)
    # valid parents: lazy, no device work yet
    assert vb.JoinedRdd(s, a.count_by_key(3), 3).num_slices == 3
    assert len(vb.CoGroupedRdd([s, a, a.count_by_key(3)], 3).rdds) == 3
    comb = vb.Context.parallelize(ctx, k64, 2, values=(k64, k64)).combine_by_key({"avg": ("mean", 0), "n": ("count", None)}, 3)
    assert isinstance(comb.aggregate("avg"), vb.AggregateRdd)
    a.join(comb.aggregate("n"), 4)
    s.cogroup(a, 3)
    s.left_outer_join(a, 3), s.right_outer_join(a, 3), s.full_outer_join(a, 3)
    # unknown aggregate name
    with pytest.raises(ValueError):
        comb.aggregate("sum")
    # group / cogroup / sort results are not join parents
    for bad in (a.group_by_key(3), a.sort_by_key(3), vb.ShuffledRdd(a, "cogroup", 3)):
        with pytest.raises(TypeError):
            bad.join(s, 3)
        with pytest.raises(TypeError):
            s.join(bad, 3)
        with pytest.raises(TypeError):
            vb.CoGroupedRdd([s, bad], 3)
    # String keys
    strs = vb.Context.parallelize(ctx, ["x", "y"], 1, values=k64[:2]).reduce_by_key("sum", 3)
    for m in ("join", "left_outer_join", "right_outer_join", "full_outer_join", "cogroup"):
        with pytest.raises(TypeError):
            getattr(strs, m)(s, 3)
    with pytest.raises(TypeError):
        s.join(strs, 3)
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([s, strs], 3)
    # key types that differ: 4-byte against 8-byte keys, i64 against u64 keys
    s32 = vb.Context.parallelize(ctx, (k32, k64), 2).reduce_by_key("max", 3)
    si64 = vb.Context.parallelize(ctx, (k64.astype(np.int64), k64), 2).count_by_key(3)
    for x, y in ((s, s32), (s32, a), (s, si64), (a, si64)):
        with pytest.raises(TypeError):
            x.join(y, 3)
        with pytest.raises(TypeError):
            vb.CoGroupedRdd([x, y], 3)
    with pytest.raises(ValueError):
        s.join(a, 0)
    with pytest.raises(TypeError):
        s.join(k64, 3)
