"""CPU-side checks of the N-way outer join: the restatement in tests/join_n_outer_ref.py on hand-written cases and
against the two-side outer joins of tests/outer_join_ref.py (n = 2, all four masks), its array form against the
restatement, and the Python mirror's argument errors, which are raised before any device work."""
import random

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref as P
from tests import cogroup_n_ref as CN
from tests import join_n_outer_ref as JO
from tests import outer_join_ref as OJ


def test_three_parents_by_hand():
    a = [(1, 10), (2, 20), (1, 11), (5, 50)]
    b = [(1, 100), (3, 300), (1, 101)]
    c = [(1, 1000), (2, 2000), (3, 3000)]
    parents = [(a, 2), (b, 1), (c, 2)]
    key1 = [(1, [10, 100, 1000]), (1, [10, 101, 1000]), (1, [11, 100, 1000]), (1, [11, 101, 1000])]
    by_key = lambda rows: sorted(rows, key=lambda r: r[0])          # stable: keeps each key's nested order
    assert by_key(JO.join_n_outer(parents, 3, 0b111)) == key1
    assert by_key(JO.join_n_outer(parents, 3, 0b001)) == key1 + [(2, [20, None, 2000]), (5, [50, None, None])]
    assert by_key(JO.join_n_outer(parents, 3, 0b100)) == key1 + [(2, [20, None, 2000]), (3, [None, 300, 3000])]
    assert by_key(JO.join_n_outer(parents, 3, 0b110)) == key1 + [(3, [None, 300, 3000])]
    assert by_key(JO.join_n_outer(parents, 3, 0)) == key1 + [(2, [20, None, 2000]), (3, [None, 300, 3000]),
                                                             (5, [50, None, None])]


def test_none_slots_and_nesting_order():
    a = [(7, 1), (7, 2)]
    b = [(8, 5)]
    c = [(7, 30), (7, 31), (8, 6)]
    got = sorted(JO.join_n_outer([(a, 1), (b, 1), (c, 1)], 1, 0), key=lambda r: r[0])
    assert got == [(7, [1, None, 30]), (7, [1, None, 31]), (7, [2, None, 30]), (7, [2, None, 31]), (8, [None, 5, 6])]
    # one parent: every mask gives each row once, as group_by_key lists them
    one = JO.join_n_outer([(a + b, 2)], 1, 0)
    assert one == JO.join_n_outer([(a + b, 2)], 1, 1) and sorted(one) == sorted((k, [v]) for k, v in a + b)
    # the same parent twice: no key is ever missing, so every mask is the inner join
    for m in range(4):
        assert sorted(JO.join_n_outer([(c, 2), (c, 1)], 2, m)) == sorted(CN.join_n([(c, 2), (c, 1)], 2))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_two_parents_are_the_two_side_joins(seed):
    rng = random.Random(seed)
    keys = [0, 2 ** 64 - 1] + [rng.randrange(1 << 64) for _ in range(40)]
    a = [(rng.choice(keys[:30]), rng.randrange(1 << 64)) for _ in range(300)]
    b = [(rng.choice(keys[12:]), rng.randrange(1 << 64)) for _ in range(200)]
    R = 4
    got = lambda m: sorted(JO.join_n_outer([(a, 3), (b, 5)], R, m))
    assert got(0b11) == sorted((k, [v, w]) for k, (v, w) in P.join(a, 3, b, 5, R))
    for m, kind in ((0b01, "left"), (0b10, "right"), (0b00, "full")):
        assert got(m) == sorted((k, [v, w]) for k, (v, w) in OJ.outer_join(kind, a, 3, b, 5, R)), kind


@pytest.mark.parametrize("key_width", [8, 4])
def test_array_reference_matches_the_restatement(key_width):
    rng = np.random.default_rng(key_width)
    if key_width == 8:
        ks = [rng.integers(lo, lo + 40, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) for lo, n in ((0, 120), (20, 90), (30, 60))]
        ks[0][:2] = [0, 2 ** 64 - 1]
        to_py = int
    else:
        ks = [rng.integers(lo, lo + 40, n).astype(np.int32) for lo, n in ((-20, 120), (0, 90), (10, 60))]
        to_py = lambda k: int(k) & 0xFFFFFFFF
    vs = [rng.integers(1, 1 << 62, len(k)).astype(np.uint64) for k in ks]
    Ms, R = (3, 2, 4), 5
    parts = CN.ref_parts_n(list(zip(ks, vs, Ms)), R, key_width)
    parents = [([(to_py(x), int(y)) for x, y in zip(k, v)], M) for k, v, M in zip(ks, vs, Ms)]
    u64_of = {to_py(x): int(np.int64(x).view(np.uint64)) if key_width == 4 else int(x) for k in ks for x in k}
    for m in range(8):
        want = sorted((u64_of[k], tuple(0 if v is None else v for v in row) + tuple(int(v is not None) for v in row))
                      for k, row in JO.join_n_outer(parents, R, m, key_width))
        got = JO.outer_of_parts(parts, m)
        assert sorted((k, row) for d in got for k, rows in d.items() for row in rows) == want, m
        for r, d in enumerate(got):               # each key's rows in nested order, in the key's partition
            assert all(P.get_partition(k if key_width == 8 else k & 0xFFFFFFFF, R, key_width) == r for k in d)


@pytest.mark.parametrize("mask,kind", [(0b01, "left"), (0b10, "right"), (0b00, "full"), (0b11, None)])
def test_array_reference_at_two_sides_is_outer_join_parts(mask, kind):
    rng = np.random.default_rng(mask)
    ka = rng.integers(0, 300, 2000).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    kb = rng.integers(150, 500, 1500).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    va, vb_ = rng.integers(1, 1 << 62, len(ka)).astype(np.uint64), rng.integers(1, 1 << 62, len(kb)).astype(np.uint64)
    R = 4
    got = JO.outer_of_parts(CN.ref_parts_n([(ka, va, 3), (kb, vb_, 2)], R), mask)
    if kind is None:
        want = [{k: [row + (1, 1) for row in rows] for k, rows in d.items()}
                for d in CN.join_of_parts(CN.ref_parts_n([(ka, va, 3), (kb, vb_, 2)], R))]
    else:
        want = OJ.outer_join_parts(kind, ka, va, 3, kb, vb_, 2, R)
    assert got == want


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_python_mirror_argument_errors_before_device_work():
    k64 = np.arange(5, dtype=np.uint64)
    ctx = _NoDevice()
    a = vb.Context.parallelize(ctx, (k64, k64), 2)
    b = vb.Context.parallelize(ctx, (k64, np.arange(5, dtype=np.float64)), 3)
    cg = vb.CoGroupedRdd([a, b, a], 3)
    for call in (lambda m: cg.outer_join_compute(0, m), cg.outer_join_collect):
        for bad in (8, 1 << 16, -1, [3], [0, 3], (-1,), [0, 5]):
            with pytest.raises(ValueError):
                call(bad)
        for bad in (None, 1.0, "1", [0.0], [True], True, [None]):
            with pytest.raises(TypeError):
                call(bad)
    assert cg._required_mask(0) == 0 and cg._required_mask(7) == 7 and cg._required_mask(np.uint32(5)) == 5
    assert cg._required_mask([]) == 0 and cg._required_mask([2, 0]) == 5 and cg._required_mask({1}) == 2
    assert cg._required_mask(range(3)) == 7 and cg._required_mask([np.int64(1), 1]) == 2
    big = vb.CoGroupedRdd([a] * 16, 1)
    assert big._required_mask(0xFFFF) == 0xFFFF and big._required_mask(range(16)) == 0xFFFF
    with pytest.raises(ValueError):
        big.outer_join_compute(0, 1 << 16)
    with pytest.raises(ValueError):
        vb.CoGroupedRdd([a] * 17, 3)                  # side counts are the cogroup's
    with pytest.raises(ValueError):
        vb.CoGroupedRdd([], 3)


class _FakeCoGrouped(vb.CoGroupedRdd):
    """A CoGroupedRdd whose outer_join_compute returns fixed partitions instead of calling the device."""

    def __init__(self, parts, n):
        self.num_slices, self._parts, self.rdds = len(parts), parts, [None] * n

    def outer_join_compute(self, split, required):
        return self._parts[split]


def test_outer_join_collect_keeps_the_masks():
    u = lambda *x: np.array(x, dtype=np.uint64)
    ma = lambda data, mask: np.ma.MaskedArray(np.array(data, dtype=np.uint64), mask=mask)
    parts = [(u(4, 4), [u(10, 11), ma([20, 0], [False, True])]), (u(), [u(), ma([], [])]), (u(9), [u(3), ma([0], [True])])]
    k, vs = _FakeCoGrouped(parts, 2).outer_join_collect(0b01)
    assert k.tolist() == [4, 4, 9] and vs[0].tolist() == [10, 11, 3] and not isinstance(vs[0], np.ma.MaskedArray)
    assert isinstance(vs[1], np.ma.MaskedArray) and vs[1].tolist() == [20, None, None]
