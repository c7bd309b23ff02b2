"""CPU-side checks of the cogroup: the array reference the GPU tests use (the C oracle's group shuffle of each side)
against oracle/pyref.py:cogroup, and JoinedRdd.cogroup_collect's assembly of (k, (vs, ws)) from cogroup_compute's
CSR output, with a stand-in for the device call."""
import random

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref as P
from tests.test_gpu_cogroup import part_dict, ref_parts


def _pyref_parts(rows_a, Ma, rows_b, Mb, R, key_width=8):
    out = [dict() for _ in range(R)]
    for k, (vs, ws) in P.cogroup(rows_a, Ma, rows_b, Mb, R, key_width):
        out[P.get_partition(k, R, key_width)][k] = (vs, ws)
    return out


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_array_reference_matches_pyref_cogroup(seed):
    rng = random.Random(seed)
    keys = [0, 2 ** 64 - 1] + [rng.randrange(1 << 64) for _ in range(40)]
    rows_a = [(rng.choice(keys[:30]), rng.randrange(1 << 64)) for _ in range(300)]
    rows_b = [(rng.choice(keys[12:]), rng.randrange(1 << 64)) for _ in range(200)]
    R, Ma, Mb = 4, 3, 5
    arr = lambda rows, i: np.array([r[i] for r in rows], dtype=np.uint64)
    got = ref_parts(arr(rows_a, 0), arr(rows_a, 1), Ma, arr(rows_b, 0), arr(rows_b, 1), Mb, R)
    assert got == _pyref_parts(rows_a, Ma, rows_b, Mb, R)
    # a key that a side lacks has an empty list there, never two empty lists
    lists = [x for d in got for x in d.values()]
    assert all(vs or ws for vs, ws in lists) and any(not vs for vs, _ in lists) and any(not ws for _, ws in lists)


def test_array_reference_empty_and_4_byte_keys():
    e = np.empty(0, dtype=np.uint64)
    assert ref_parts(e, e, 1, e, e, 1, 3) == [{}, {}, {}]
    k = np.array([1, 2, 3, 4], dtype=np.int32)
    v = np.arange(4, dtype=np.uint64)
    rows = list(zip(k.tolist(), v.tolist()))
    assert ref_parts(k, v, 2, k, v, 2, 2, key_width=4) == _pyref_parts(rows, 2, rows, 2, 2, key_width=4)


def test_part_dict_checks_the_structure():
    keys = np.array([5, 9, 11], dtype=np.uint64)
    R = 1
    lo, lv = np.array([0, 2, 2, 3], dtype=np.uint64), np.array([1, 2, 3], dtype=np.uint64)
    ro, rv = np.array([0, 1, 3, 3], dtype=np.uint64), np.array([7, 8, 9], dtype=np.uint64)
    assert part_dict(keys, lo, lv, ro, rv, 0, R) == {5: ([1, 2], [7]), 9: ([], [8, 9]), 11: ([3], [])}
    with pytest.raises(AssertionError):          # key 9 with two empty lists
        part_dict(keys, lo, lv, np.array([0, 1, 1, 3], dtype=np.uint64), rv, 0, R)
    with pytest.raises(AssertionError):          # a key twice
        part_dict(np.array([5, 5, 11], dtype=np.uint64), lo, lv, ro, rv, 0, R)
    with pytest.raises(AssertionError):          # offsets that do not end at the value count
        part_dict(keys, lo, lv, ro, rv[:2], 0, R)


class _FakeCogroup(vb.JoinedRdd):
    """A JoinedRdd whose cogroup_compute returns fixed CSR partitions instead of calling the device."""

    def __init__(self, parts):
        self.num_slices, self._parts = len(parts), parts

    def cogroup_compute(self, split):
        return self._parts[split]


def test_cogroup_collect_assembles_the_lists():
    u = lambda *x: np.array(x, dtype=np.uint64)
    parts = [
        (u(4, 7), (u(0, 2, 2), u(10, 11)), (u(0, 1, 3), u(20, 21, 22))),
        (u(), (u(0), u()), (u(0), u())),
        (np.array([-3], dtype=np.int64), (u(0, 0), np.array([], dtype=np.float64)), (u(0, 1), np.array([1.5]))),
    ]
    got = _FakeCogroup(parts).cogroup_collect()
    assert [k for k, _ in got] == [4, 7, -3]
    assert [(vs.tolist(), ws.tolist()) for _, (vs, ws) in got] == [([10, 11], [20]), ([], [21, 22]), ([], [1.5])]
    assert all(isinstance(vs, np.ndarray) and isinstance(ws, np.ndarray) for _, (vs, ws) in got)
    assert got[2][1][1].dtype == np.float64
