"""repartition(n) = coalesce(n, shuffle = true) without a GPU: the restatement in tests/repartition_ref.py against an
independent restatement of vega's route (partition_by_key over (position, item) pairs), the shape of the reference's
test_coalesced, and the Python mirror's argument checks."""
import struct

import numpy as np
import pytest

from oracle import pyref
from tests import repartition_ref as RP
from oracle import oracle as O
from vega_b200.rdd import PairRdd, Rdd, StrPairRdd, StrRdd, _BytesCol, _Col, _StrCol


def partition_by_key_route(map_items, starts, n_reduce):
    """pair_rdd.rs:157-171 over (position, item): group by position (Vec append, a dict standing in for the HashMap) in
    the partition of the oracle's C restatement of HashPartitioner (MetroHash64 of the 8 LE bytes, modulo n), then flatten
    the groups and drop the keys."""
    groups = [dict() for _ in range(n_reduce)]
    for m, items in enumerate(map_items):
        for i, x in enumerate(items):
            pos = (starts[m] + 1 + i) % (1 << 64)
            p = O.metrohash64_1(struct.pack("<Q", pos), 0) % n_reduce
            groups[p].setdefault(pos, []).append(x)
    return [[x for vs in g.values() for x in vs] for g in groups]


@pytest.mark.parametrize("n_reduce", [1, 3, 256, 257, 1000])
@pytest.mark.parametrize("start_kind", ["zero", "r_minus_1", "wrap"])
def test_restatement_matches_partition_by_key(n_reduce, start_kind):
    rng = np.random.default_rng(n_reduce)
    map_items = [list(rng.integers(0, 1 << 20, size=int(k))) for k in (0, 700, 1, 1300, 0, 400)]
    start = {"zero": 0, "r_minus_1": n_reduce - 1, "wrap": (1 << 64) - 3}[start_kind]
    starts = [start, start, start + 5 & RP.MASK, start, 17, start]
    got = RP.repartition(map_items, starts, n_reduce)
    want = partition_by_key_route(map_items, starts, n_reduce)
    assert len(got) == n_reduce
    assert [sorted(p) for p in got] == [sorted(p) for p in want]
    assert sum(len(p) for p in got) == sum(len(x) for x in map_items)


def test_positions_share_groups_across_maps():
    """Equal positions of different map partitions share a group in vega; they still land in the same partition."""
    map_items = [["a", "b", "c"], ["x", "y", "z"]]
    got = RP.repartition(map_items, [0, 0], 7)
    for i in range(3):
        p = pyref.get_partition(RP.position(0, i), 7)
        assert got[p].index(map_items[0][i]) < got[p].index(map_items[1][i])


def test_coalesced_shape():
    """tests/test_rdd.rs:364-385 test_coalesced, shuffle case: 100 items in 20 slices -> 100 partitions, 100 items."""
    slices = pyref.slice_([1] * 100, 20)
    parts = RP.repartition(slices, [0] * len(slices), 100)
    assert len(parts) == 100
    assert sum(len(p) for p in parts) == 100


def test_wrap_around():
    assert RP.position((1 << 64) - 3, 0) == (1 << 64) - 2
    assert RP.position((1 << 64) - 3, 2) == 0
    assert RP.position((1 << 64) - 1, 5) == 5


def _rdd(n=10, slices=3):
    return Rdd(None, _Col(np.arange(n, dtype=np.uint64)), slices)


def test_argument_checks():
    r = _rdd()
    with pytest.raises(NotImplementedError):
        r.coalesce(4)                                   # shuffle=False: the narrow CoalescedRdd
    with pytest.raises(NotImplementedError):
        r.coalesce(4, shuffle=False)
    for bad in (0, -1, 2.5, True):
        with pytest.raises(ValueError):
            r.repartition(bad)
    with pytest.raises(ValueError):
        r.repartition(4, starts=[0, 0])                 # 3 map partitions
    with pytest.raises(ValueError):
        r.repartition(4, starts=[0, -1, 0])
    with pytest.raises(ValueError):
        r.repartition(4, starts=[0, 1 << 64, 0])
    rr = r.repartition(4, starts=np.array([0, (1 << 64) - 1, 7], dtype=np.uint64))
    assert rr.starts == [0, (1 << 64) - 1, 7] and rr.number_of_splits() == 4
    assert r.repartition(4).starts == [0, 0, 0]


def test_item_shapes():
    k = _Col(np.arange(6, dtype=np.uint64))
    v = _Col(np.arange(6, dtype=np.int64), role="value")
    assert len(PairRdd(None, k, v, 2).repartition(3).cols) == 2
    rows = _Col(np.arange(12, dtype=np.uint64).reshape(6, 2), allow_rows=True)
    rr = PairRdd(None, rows, None, 2).repartition(3)
    assert len(rr.cols) == 2 and rr.cols[1].owner.tolist() == [1, 3, 5, 7, 9, 11]
    pb = PairRdd(None, k, _BytesCol(["a", "bb", "", "c", "d", "e"]), 2).repartition(3)
    assert len(pb.cols) == 1 and pb.bcol is not None and not pb.bytes_first
    with pytest.raises(NotImplementedError):
        PairRdd(None, k, None, 2, cols=(v, v)).repartition(3)
    sk = _StrCol(["a", "b", "c", "d", "e", "f"])
    sp = StrPairRdd(None, sk, v, 2).repartition(3)
    assert len(sp.cols) == 1 and sp.bytes_first
    with pytest.raises(NotImplementedError):
        StrPairRdd(None, sk, _BytesCol(["x"] * 6), 2).repartition(3)
    with pytest.raises(NotImplementedError):
        StrPairRdd(None, sk, None, 2, cols=(v, v)).repartition(3)
    s = StrRdd(None, sk, 2).repartition(3)
    assert s.cols == () and s.bcol is not None
