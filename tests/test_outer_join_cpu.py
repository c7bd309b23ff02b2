"""CPU-side checks of the outer joins: the reference definitions in tests/outer_join_ref.py on hand-written cases, their
agreement with inner join + unmatched rows and with the array reference the GPU tests use, and the Python mirror's
argument errors, which are raised before any device work."""
import random

import numpy as np
import pytest

import vega_b200 as vb
from oracle import pyref as P
from tests import outer_join_ref as OJ

# the reference's examples/join.rs / tests/test_pair_rdd.rs:39-82 data
COL1 = [(1, ("A", "B")), (2, ("C", "D")), (3, ("E", "F")), (4, ("G", "H"))]
COL2 = [(1, "A1"), (1, "A2"), (2, "B1"), (2, "B2"), (3, "C1"), (3, "C2")]
MATCHED = [(1, (("A", "B"), "A1")), (1, (("A", "B"), "A2")), (2, (("C", "D"), "B1")), (2, (("C", "D"), "B2")),
           (3, (("E", "F"), "C1")), (3, (("E", "F"), "C2"))]


def test_join_rs_data():
    assert sorted(OJ.left_outer_join(COL1, 4, COL2, 4, 4, int_width=4)) == sorted(MATCHED + [(4, (("G", "H"), None))])
    assert sorted(P.join(COL1, 4, COL2, 4, 4, int_width=4)) == sorted(MATCHED)       # the inner join drops key 4
    assert sorted(OJ.right_outer_join(COL1, 4, COL2, 4, 4, int_width=4)) == sorted(MATCHED)
    assert sorted(OJ.full_outer_join(COL1, 4, COL2, 4, 4, int_width=4)) == sorted(MATCHED + [(4, (("G", "H"), None))])
    want = [(k, (w, v)) for k, (v, w) in MATCHED] + [(4, (None, ("G", "H")))]
    assert sorted(OJ.right_outer_join(COL2, 4, COL1, 4, 4, int_width=4)) == sorted(want)


def test_hand_written_cases():
    a = [(1, 10), (2, 20), (1, 11), (5, 50)]
    b = [(1, 100), (3, 300), (1, 101), (3, 301)]
    rows = lambda kind: sorted(OJ.outer_join(kind, a, 2, b, 3, 1))
    nested = [(1, (10, 100)), (1, (10, 101)), (1, (11, 100)), (1, (11, 101))]
    assert rows("left") == sorted(nested + [(2, (20, None)), (5, (50, None))])
    assert rows("right") == sorted(nested + [(3, (None, 300)), (3, (None, 301))], key=str)
    assert rows("full") == sorted(nested + [(2, (20, None)), (5, (50, None)), (3, (None, 300)), (3, (None, 301))], key=str)
    # nesting order of one key: for v in vs { for w in ws }, each list in input order
    assert [r for r in OJ.outer_join("full", a, 1, b, 1, 1) if r[0] == 1] == nested
    # no shared key, one side empty, both empty
    assert sorted(OJ.outer_join("left", [(1, 1)], 1, [(2, 2)], 1, 2)) == [(1, (1, None))]
    assert sorted(OJ.outer_join("right", [(1, 1)], 1, [(2, 2)], 1, 2)) == [(2, (None, 2))]
    assert OJ.outer_join("right", a, 2, [], 1, 3) == [] and OJ.outer_join("left", [], 1, b, 2, 3) == []
    assert sorted(OJ.outer_join("full", [], 1, b, 2, 3), key=str) == sorted([(k, (None, w)) for k, w in b], key=str)
    assert OJ.outer_join("full", [], 1, [], 1, 2) == []


def _random_rows(rng, n, n_keys, wide):
    keys = [rng.randrange(n_keys) * (0x9E3779B97F4A7C15 if wide else 1) % (1 << 64) for _ in range(n)]
    return [(k, rng.randrange(1 << 40)) for k in keys]


@pytest.mark.parametrize("kind", ["left", "right", "full"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_outer_is_inner_plus_unmatched(kind, seed):
    rng = random.Random(seed)
    a, b = _random_rows(rng, 300, 60, True), _random_rows(rng, 200, 80, True)
    keep_l, keep_r = OJ.KEEP[kind]
    ka, kb = {k for k, _ in a}, {k for k, _ in b}
    extra = [(k, (v, None)) for k, v in a if keep_l and k not in kb] + [(k, (None, w)) for k, w in b if keep_r and k not in ka]
    got = OJ.outer_join(kind, a, 3, b, 4, 5)
    assert sorted(got, key=str) == sorted(P.join(a, 3, b, 4, 5) + extra, key=str)
    # rows per key: max(|vs|,1) * max(|ws|,1) when the key is on a kept side or on both, else none
    nv = {k: sum(1 for x, _ in a if x == k) for k in ka | kb}
    nw = {k: sum(1 for x, _ in b if x == k) for k in ka | kb}
    kept = lambda k: (k in ka and k in kb) or (keep_l and k in ka) or (keep_r and k in kb)
    assert len(got) == sum(max(nv[k], 1) * max(nw[k], 1) for k in ka | kb if kept(k))


@pytest.mark.parametrize("kind", ["left", "right", "full"])
@pytest.mark.parametrize("key_width", [8, 4])
def test_array_reference_matches_cogroup_definition(kind, key_width):
    """outer_join_parts (C oracle inner join + numpy) equals the cogroup definition, partition by partition and in
    nesting order; keys include 0 and 2^64-1 (8-byte) or negative values (4-byte)."""
    rng = np.random.default_rng(key_width)
    n_keys = 50
    if key_width == 8:
        ka = rng.integers(0, n_keys, 400).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        kb = rng.integers(20, n_keys + 30, 300).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        ka[:2] = [0, 2 ** 64 - 1]
        kb[:2] = [2 ** 64 - 1, 5]
        to_py = lambda k: int(k)
    else:
        ka = rng.integers(-30, 20, 400).astype(np.int64)
        kb = rng.integers(0, 40, 300).astype(np.int64)
        to_py = lambda k: int(k) & 0xFFFFFFFF      # the 4 key bytes the partitioner hashes
    va = rng.integers(0, 1 << 40, len(ka)).astype(np.uint64)
    vb_ = rng.integers(0, 1 << 40, len(kb)).astype(np.uint64)
    R, Ma, Mb = 4, 3, 2
    got = OJ.outer_join_parts(kind, ka, va, Ma, kb, vb_, Mb, R, key_width=key_width)
    rows_a = [(to_py(k), int(v)) for k, v in zip(ka, va)]
    rows_b = [(to_py(k), int(v)) for k, v in zip(kb, vb_)]
    want = [dict() for _ in range(R)]
    u64_of = {to_py(k): int(np.int64(k).view(np.uint64)) if key_width == 4 else int(k) for k in np.concatenate([ka, kb])}
    for k, (v, w) in OJ.outer_join(kind, rows_a, Ma, rows_b, Mb, R, int_width=key_width):
        want[P.get_partition(k, R, key_width)].setdefault(u64_of[k], []).append(
            (v or 0, w or 0, int(v is not None), int(w is not None)))
    assert got == want


def test_key_partitions_match_the_partitioner():
    keys = np.array([0, 1, 2 ** 64 - 1, 12345, 2 ** 63, 7, 7, 0], dtype=np.uint64)
    part = OJ.key_partitions(keys, 5)
    assert part.tolist() == [P.get_partition(int(k), 5) for k in keys]


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_python_mirror_argument_errors_before_device_work():
    k64 = np.arange(5, dtype=np.uint64)
    k32 = np.arange(5, dtype=np.int32)
    a = vb.Context.parallelize(_NoDevice(), (k64, k64), 2)
    b32 = vb.Context.parallelize(_NoDevice(), (k32, k64), 2)
    for method in ("left_outer_join", "right_outer_join", "full_outer_join"):
        with pytest.raises(TypeError):
            getattr(a, method)(b32, 3)                     # 8-byte against 4-byte keys: different partitioners
        with pytest.raises(ValueError):
            getattr(a, method)(a, 0)
        j = getattr(a, method)(a, 3)                       # valid: lazy, no device work yet
        assert j.kind == method.split("_")[0] and j.num_slices == 3
    with pytest.raises(ValueError):
        vb.JoinedRdd(a, a, 3, "inner")                     # the inner join is join(); no other kind exists
    with pytest.raises(ValueError):
        vb.JoinedRdd(a, a, 3, "outer")
