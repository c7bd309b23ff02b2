"""sort_by_key over String keys without a GPU: the reference of tests/str_sort_ref.py (byte order, stability, cuts), and
the argument errors of vb.StrSortedRdd, raised before any device work."""
import numpy as np
import pytest

import vega_b200 as vb
from tests import str_sort_ref as SR


def test_byte_order_prefix_first_and_unsigned():
    want = [b"", b"\x00", b"a", b"a\x00", b"a\x00\x00", b"ab", b"\x7f", b"\x80", b"\xff", b"\xff\x00"]
    rng = np.random.default_rng(0)
    for _ in range(20):
        keys = [want[i] for i in rng.permutation(len(want))]
        assert SR.sort_rows(keys)[0] == want


def test_utf8_byte_order_is_str_order():
    rng = np.random.default_rng(1)
    alphabet = list("ab\x00é日🙂\x7f\x80")
    keys = ["".join(rng.choice(alphabet, int(rng.integers(0, 6)))) for _ in range(500)]
    assert [k.decode() for k in SR.sort_rows(keys)[0]] == sorted(keys)


def test_equal_keys_keep_input_order():
    keys = ["b", "a", "b", "a", "c", "a"]
    vals = np.arange(6, dtype=np.uint64)
    sk, sv, ranks = SR.sort_rows(keys, vals)
    assert sk == [b"a", b"a", b"a", b"b", b"b", b"c"]
    assert sv.tolist() == [1, 3, 5, 0, 2, 4]
    assert ranks.tolist() == [0, 0, 0, 1, 1, 2]


def test_cuts_never_split_a_key():
    keys = ["a"] * 5 + ["b"] * 3 + ["c"]
    parts = SR.partitions(keys, None, 3)                       # floor(p·9/3) = 3, 6: moved to 5 and 8
    assert [p[0] for p in parts] == [[b"a"] * 5, [b"b"] * 3, [b"c"]]
    assert [len(p[0]) for p in SR.partitions(["x"] * 4, None, 3)] == [4, 0, 0]
    assert [len(p[0]) for p in SR.partitions(["y", "x"], None, 5)] == [0, 0, 1, 0, 1]   # R > n: empty partitions
    assert [len(p[0]) for p in SR.partitions([], None, 2)] == [0, 0]


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_sorted_rdd_argument_errors_before_device_work():
    sc = _NoDevice()
    keys = ["x", "y", "x"]
    vals = np.array([1, 2, 3], dtype=np.uint64)
    pair = vb.Context.parallelize(sc, keys, 2, values=vals)
    one_col = vb.Context.parallelize(sc, keys, 2, values=(vals,))
    two_cols = vb.Context.parallelize(sc, keys, 2, values=(vals, vals))
    only_keys = vb.Context.parallelize(sc, keys, 2)
    with pytest.raises(TypeError):
        vb.StrSortedRdd(two_cols, 2)
    with pytest.raises(TypeError):
        vb.StrSortedRdd(vb.Context.parallelize(sc, np.arange(3, dtype=np.uint64), 2, values=vals), 2)
    with pytest.raises(TypeError):
        vb.StrSortedRdd(vb.Context.parallelize(sc, np.arange(3, dtype=np.uint64), 2), 2)
    for p in (pair, only_keys):
        with pytest.raises(ValueError):
            vb.StrSortedRdd(p, 0)
    # valid: lazy, no device work yet
    assert vb.StrSortedRdd(pair, 3).num_slices == 3
    assert vb.StrSortedRdd(one_col, 1).vals is one_col.cols[0]
    assert vb.StrSortedRdd(only_keys, 4).vals is None
    # the String-key RDDs keep refusing their own sort methods
    with pytest.raises(TypeError):
        pair.sort_by_key(2)
    with pytest.raises(TypeError):
        only_keys.sort(2)
