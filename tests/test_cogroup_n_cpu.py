"""CPU-side checks of the N-way cogroup and join: the restatement in tests/cogroup_n_ref.py against oracle/pyref.py
(n = 2 is the cogroup, n = 1 is group_by_key) and the reference's tests/test_rdd.rs data with a third parent, the array
reference the GPU tests use against that restatement, CoGroupedRdd's assembly of its results, and its argument errors,
which are raised before any device work."""
import random

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref as P
from tests import cogroup_n_ref as CN


def _by_partition(items, R, key_width=8):
    out = [dict() for _ in range(R)]
    for k, lists in items:
        out[P.get_partition(k, R, key_width)][k] = tuple(tuple(x) for x in lists)
    return out


def _rows(rng, n, keys):
    return [(rng.choice(keys), rng.randrange(1 << 64)) for _ in range(n)]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_two_parents_are_the_cogroup_and_one_is_group_by_key(seed):
    rng = random.Random(seed)
    keys = [0, 2 ** 64 - 1] + [rng.randrange(1 << 64) for _ in range(40)]
    a, b = _rows(rng, 300, keys[:30]), _rows(rng, 200, keys[12:])
    R = 4
    got = CN.cogroup_n([(a, 3), (b, 5)], R)
    assert _by_partition(got, R) == _by_partition([(k, (vs, ws)) for k, (vs, ws) in P.cogroup(a, 3, b, 5, R)], R)
    assert sorted(CN.join_n([(a, 3), (b, 5)], R)) == sorted((k, [v, w]) for k, (v, w) in P.join(a, 3, b, 5, R))
    one = CN.cogroup_n([(a, 3)], R)
    assert _by_partition(one, R) == _by_partition([(k, (vs,)) for k, vs in P.group_by_key(a, 3, R)], R)
    assert sorted(CN.join_n([(a, 3)], R)) == sorted((k, [v]) for k, v in a)


def test_test_rdd_cogroup_data_with_a_third_parent():
    # tests/test_rdd.rs:434-456: (1,"A"), (2,"B"), (3,"C"), (4,"D") cogrouped with itself; a third parent adds key 4
    # twice and key 5
    rows = [(1, "A"), (2, "B"), (3, "C"), (4, "D")]
    third = [(4, "X"), (5, "Y"), (4, "Z")]
    got = sorted(CN.cogroup_n([(rows, 2), (rows, 2), (third, 2)], 2, int_width=4))
    assert got == [(1, [["A"], ["A"], []]), (2, [["B"], ["B"], []]), (3, [["C"], ["C"], []]),
                   (4, [["D"], ["D"], ["X", "Z"]]), (5, [[], [], ["Y"]])]
    assert sorted(CN.join_n([(rows, 2), (rows, 2), (third, 2)], 2, int_width=4)) == [(4, ["D", "D", "X"]), (4, ["D", "D", "Z"])]
    assert sorted(CN.cogroup_n([(rows, 2), (rows, 2)], 2, int_width=4)) == \
        sorted((k, [vs, ws]) for k, (vs, ws) in P.cogroup(rows, 2, rows, 2, 2, int_width=4))


def test_join_nesting_order():
    a = [(1, 10), (1, 11)]
    b = [(1, 20), (1, 21), (2, 5)]
    c = [(1, 30), (3, 7)]
    got = CN.join_n([(a, 1), (b, 2), (c, 1)], 1)
    assert got == [(1, [10, 20, 30]), (1, [10, 21, 30]), (1, [11, 20, 30]), (1, [11, 21, 30])]


@pytest.mark.parametrize("key_width", [8, 4])
def test_array_reference_matches_the_restatement(key_width):
    rng = np.random.default_rng(key_width)
    if key_width == 8:
        ks = [rng.integers(lo, lo + 60, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) for lo, n in ((0, 300), (30, 200), (50, 250))]
        ks[0][:2] = [0, 2 ** 64 - 1]
        ks[2][:1] = [2 ** 64 - 1]
        to_py = int
    else:
        ks = [rng.integers(lo, lo + 60, n).astype(np.int32) for lo, n in ((-30, 300), (0, 200), (20, 250))]
        to_py = lambda k: int(k) & 0xFFFFFFFF
    vs = [rng.integers(0, 1 << 62, len(k)).astype(np.uint64) for k in ks]
    Ms, R = (3, 2, 4), 5
    got = CN.ref_parts_n(list(zip(ks, vs, Ms)), R, key_width)
    u64_of = lambda k: int(np.int64(k).view(np.uint64)) if key_width == 4 else int(k)
    want = [dict() for _ in range(R)]
    parents = [([(to_py(x), int(y)) for x, y in zip(k, v)], M) for k, v, M in zip(ks, vs, Ms)]
    back = {to_py(x): u64_of(x) for k in ks for x in k}
    for k, lists in CN.cogroup_n(parents, R, key_width):
        want[P.get_partition(k, R, key_width)][back[k]] = tuple(lists)
    assert got == want
    joined = CN.join_of_parts(got)
    assert sum(len(rows) for d in joined for rows in d.values()) == len(CN.join_n(parents, R, key_width))


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_python_mirror_argument_errors_before_device_work():
    k64 = np.arange(5, dtype=np.uint64)
    ctx = _NoDevice()
    a = vb.Context.parallelize(ctx, (k64, k64), 2)
    b = vb.Context.parallelize(ctx, (k64, np.arange(5, dtype=np.float64)), 3)
    with pytest.raises(ValueError):
        vb.CoGroupedRdd([], 3)
    with pytest.raises(ValueError):
        vb.CoGroupedRdd([a] * 17, 3)
    with pytest.raises(ValueError):
        vb.CoGroupedRdd([a, b], 0)
    with pytest.raises(ValueError):
        vb.CoGroupedRdd([a, vb.Context.parallelize(_NoDevice(), (k64, k64), 2)], 3)       # another context
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([a, vb.Context.parallelize(ctx, (np.arange(5, dtype=np.int32), k64), 2)], 3)   # 4-byte keys
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([a, vb.Context.parallelize(ctx, (np.arange(5, dtype=np.int64), k64), 2)], 3)   # i64 keys
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([a, vb.Context.parallelize(ctx, ["x", "y"], 2, values=k64[:2])], 3)            # String keys
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([a, vb.Context.parallelize(ctx, k64, 2, values=(k64, k64))], 3)                # two value columns
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([a, k64], 3)
    cg = vb.CoGroupedRdd([a, b, a], 3)                 # valid: lazy, no device work yet
    assert cg.num_slices == 3 and len(cg.rdds) == 3
    assert len(vb.CoGroupedRdd([a] * 16, 1).rdds) == 16


class _FakeCoGrouped(vb.CoGroupedRdd):
    """A CoGroupedRdd whose compute / join_compute return fixed partitions instead of calling the device."""

    def __init__(self, parts, joins, n):
        self.num_slices, self._parts, self._joins, self.rdds = len(parts), parts, joins, [None] * n

    def compute(self, split):
        return self._parts[split]

    def join_compute(self, split):
        return self._joins[split]


def test_collect_assembles_the_lists():
    u = lambda *x: np.array(x, dtype=np.uint64)
    parts = [
        (u(4, 7), [(u(0, 2, 2), u(10, 11)), (u(0, 1, 3), u(20, 21, 22)), (u(0, 0, 1), np.array([-5]))]),
        (u(), [(u(0), u()), (u(0), u()), (u(0), np.array([], dtype=np.int64))]),
        (u(9), [(u(0, 0), u()), (u(0, 0), u()), (u(0, 1), np.array([3]))]),
    ]
    joins = [(u(4), [u(10), u(20), np.array([-5])]), (u(), [u(), u(), np.array([], dtype=np.int64)]),
             (u(), [u(), u(), np.array([], dtype=np.int64)])]
    cg = _FakeCoGrouped(parts, joins, 3)
    got = cg.collect()
    assert [k for k, _ in got] == [4, 7, 9]
    assert [[x.tolist() for x in ls] for _, ls in got] == [[[10, 11], [20], []], [[], [21, 22], [-5]], [[], [], [3]]]
    assert got[1][1][2].dtype == np.int64
    k, vs = cg.join_collect()
    assert k.tolist() == [4] and [v.tolist() for v in vs] == [[10], [20], [-5]] and vs[2].dtype == np.int64
