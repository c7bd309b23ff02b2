"""CPU checks of the String-key cogroup and join: the Python references (tests/cogroup_n_ref.py,
tests/join_n_outer_ref.py) over `str` rows, against a hand-written result on the reference's "x" / "y" group_by data
(tests/test_pair_rdd.rs:8-37) and against the integer references under a one-to-one renaming of the keys; the
StrCoGroupedRdd mirror's argument errors before any device work; and its assembly of the device's keyed join output."""
import itertools
import random

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref as P
from tests import cogroup_n_ref as CN
from tests import join_n_outer_ref as JO

XY = [("x", i) for i in range(1, 8)] + [("y", i) for i in range(1, 9)]
OTHER = [("x", 10), ("z", 20), ("y", 30), ("x", 11)]


def _by_partition(rows, R):
    """[(k, ...)] -> per partition the list of keys in row order, placed by pyref.get_partition"""
    parts = [[] for _ in range(R)]
    for row in rows:
        parts[P.get_partition(row[0], R)].append(row[0])
    return parts


def test_cogroup_reference_on_the_group_by_data():
    R = 4
    got = CN.cogroup_n([(XY, 4), (OTHER, 2)], R)
    want = {"x": [[1, 2, 3, 4, 5, 6, 7], [10, 11]], "y": [[1, 2, 3, 4, 5, 6, 7, 8], [30]], "z": [[], [20]]}
    assert dict(got) == want and len(got) == 3
    # the reference emits each partition's keys together, in partition order
    order = [P.get_partition(k, R) for k, _ in got]
    assert order == sorted(order)


def test_join_references_on_the_group_by_data():
    R = 4
    xs, ys = list(range(1, 8)), list(range(1, 9))
    inner = [("x", [v, w]) for v in xs for w in (10, 11)] + [("y", [v, 30]) for v in ys]
    assert sorted(CN.join_n([(XY, 4), (OTHER, 2)], R)) == sorted(inner)
    assert sorted(JO.join_n_outer([(XY, 4), (OTHER, 2)], R, 0b11)) == sorted(inner)
    assert sorted(JO.join_n_outer([(XY, 4), (OTHER, 2)], R, 0b01)) == sorted(inner)          # left: z has no left side
    right = inner + [("z", [None, 20])]
    assert sorted(JO.join_n_outer([(XY, 4), (OTHER, 2)], R, 0b10), key=repr) == sorted(right, key=repr)
    assert sorted(JO.join_n_outer([(XY, 4), (OTHER, 2)], R, 0), key=repr) == sorted(right, key=repr)
    # rows of one key are contiguous, the last side varying fastest
    rows = [r for r in JO.join_n_outer([(XY, 4), (OTHER, 2)], R, 0b11) if r[0] == "x"]
    assert [v for _, v in rows] == [[v, w] for v in xs for w in (10, 11)]


def _words(rng, n, pool):
    return [pool[rng.randrange(len(pool))] for _ in range(n)]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_string_references_equal_the_integer_references_under_renaming(seed):
    rng = random.Random(seed)
    pool = ["", "a", "ab", "abc", "x" * 40, "\x00", "a\x00b", "é", "日本", "zz"] + [f"w{i}" for i in range(30)]
    ids = {w: 1000 + 7 * i for i, w in enumerate(pool)}             # one-to-one: word -> integer key
    back = {v: k for k, v in ids.items()}
    R = rng.choice([1, 3, 7])
    parents = []
    for _ in range(3):
        n = rng.randrange(0, 60)
        parents.append((list(zip(_words(rng, n, pool), [rng.randrange(100) for _ in range(n)])), rng.randrange(1, 5)))
    ints = [([(ids[k], v) for k, v in rows], ns) for rows, ns in parents]
    s_cg, i_cg = dict(CN.cogroup_n(parents, R)), {back[k]: v for k, v in CN.cogroup_n(ints, R)}
    assert s_cg == i_cg                                               # per key: the same lists on every side
    for rows, _ in parents:                                           # each key placed as Rust places a String
        for k, _ in rows:
            assert 0 <= P.get_partition(k, R) < R
    for required in range(8):
        s = JO.join_n_outer(parents, R, required)
        i = [(back[k], v) for k, v in JO.join_n_outer(ints, R, required)]
        per_key = lambda rows: {k: [v for kk, v in rows if kk == k] for k in {kk for kk, _ in rows}}
        assert per_key(s) == per_key(i), required


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_mirror_argument_errors_before_device_work():
    sc = _NoDevice()
    v = np.arange(3, dtype=np.uint64)
    a = vb.Context.parallelize(sc, ["x", "y", "x"], 2, values=v)
    b = vb.Context.parallelize(sc, ["x", "z", "w"], 3, values=np.arange(3, dtype=np.float64))
    with pytest.raises(ValueError):
        vb.StrCoGroupedRdd([], 3)
    with pytest.raises(ValueError):
        vb.StrCoGroupedRdd([a] * 17, 3)
    with pytest.raises(ValueError):
        vb.StrCoGroupedRdd([a, b], 0)
    with pytest.raises(TypeError):                                    # integer parent
        vb.StrCoGroupedRdd([a, vb.Context.parallelize(sc, (v, v), 2)], 3)
    with pytest.raises(TypeError):                                    # an integer reduce result
        vb.StrCoGroupedRdd([a, vb.Context.parallelize(sc, (v, v), 2).reduce_by_key("sum", 3)], 3)
    with pytest.raises(TypeError):                                    # a group_by_key result
        vb.StrCoGroupedRdd([a, b.group_by_key(3)], 3)
    with pytest.raises(TypeError):                                    # another context
        vb.StrCoGroupedRdd([a, vb.Context.parallelize(_NoDevice(), ["x"], 1, values=v[:1])], 3)
    with pytest.raises(TypeError):
        vb.StrCoGroupedRdd([a, ["x", "y"]], 3)
    cg = vb.StrCoGroupedRdd([a, b.reduce_by_key("max", 2), a.count_by_key(5), a], 3)   # valid: lazy, no device work
    assert cg.num_slices == 3 and len(cg.rdds) == 4
    assert len(vb.StrCoGroupedRdd([a] * 16, 1).rdds) == 16
    assert cg._required_mask([0, 2]) == 0b101 and cg._required_mask(0b1111) == 0b1111
    for bad in (16, -1, [4]):
        with pytest.raises(ValueError):
            cg._required_mask(bad)
    with pytest.raises(TypeError):
        cg._required_mask(["0"])
    # the existing refusals stay: the binary String joins and CoGroupedRdd over String parents
    for method in ("join", "left_outer_join", "right_outer_join", "full_outer_join", "cogroup"):
        with pytest.raises(TypeError):
            getattr(a, method)(b, 2)
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([a, b], 2)


class _FakeStrCoGrouped(vb.StrCoGroupedRdd):
    """A StrCoGroupedRdd whose raw partitions are fixed instead of read from the device."""

    def __init__(self, cogroups, joins, n):
        self.num_slices, self._cg, self._joins, self.rdds = len(cogroups), cogroups, joins, [None] * n

    def compute_raw(self, split):
        return self._cg[split]

    def join_raw(self, split, required):
        return self._joins[split]


def _col(strs):
    k = vb.StrKeys.from_strs(strs)
    return k.offsets.copy(), k.data.copy()


def test_mirror_assembles_keys_lists_and_rows():
    u = lambda *x: np.array(x, dtype=np.uint64)
    ko, kb = _col(["ab", "", "日本"])
    ko2, kb2 = _col([])
    cogroups = [(ko, kb, [(u(0, 2, 2, 3), u(1, 2, 3)), (u(0, 1, 2, 2), np.array([-4.5, 7.0]))]),
                (ko2, kb2, [(u(0), u()), (u(0), np.zeros(0))])]
    # the left join (parent 0 required) of that partition: "ab" x 2 rows, "日本" with None on parent 1
    jko, jkb = _col(["ab", "日本"])
    joins = [(jko, jkb, u(0, 2, 3), [u(1, 2, 3), np.array([-4.5, -4.5, 0.0])], [None, np.array([1, 1, 0], dtype=np.uint8)]),
             (ko2, kb2, u(0), [u(), np.zeros(0)], [None, np.zeros(0, dtype=np.uint8)])]
    cg = _FakeStrCoGrouped(cogroups, joins, 2)
    got = cg.collect()
    assert [k for k, _ in got] == ["ab", "", "日本"]
    assert [[x.tolist() for x in ls] for _, ls in got] == [[[1, 2], [-4.5]], [[], [7.0]], [[3], []]]
    k, vs = cg.outer_join_collect(0b01)
    assert k.tolist() == ["ab", "ab", "日本"]
    assert vs[0].tolist() == [1, 2, 3] and not isinstance(vs[0], np.ma.MaskedArray)
    assert isinstance(vs[1], np.ma.MaskedArray) and vs[1].tolist() == [-4.5, -4.5, None]
