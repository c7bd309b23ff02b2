"""Sorted value lists without a GPU: the reference order against Python's own comparisons, the sort_values argument
checks, and the ABI declaration of vb_shuffle_set_value_order."""
import math
import re
import struct
from pathlib import Path

import numpy as np
import pytest

from tests import sorted_groups_ref as S
from vega_b200 import _lib as L
from vega_b200 import rdd

HEADER = Path(__file__).resolve().parents[1] / "include" / "vega_b200.h"


def total_cmp_key(x):
    """f64::total_cmp as a Python sort key: the IEEE 754 totalOrder of the bits."""
    b = struct.unpack("<q", struct.pack("<d", x))[0]
    return b ^ ((1 << 63) - 1) if b < 0 else b


@pytest.mark.parametrize("dtype", [np.uint64, np.int64, np.float64])
def test_reference_sorts_every_list_in_the_dtype_order(dtype):
    rng = np.random.default_rng(7)
    lens = [0, 1, 2, 3, 31, 32, 33, 200]
    offs = np.concatenate([[0], np.cumsum(lens)])
    vals = S.full_range(rng, int(offs[-1]), dtype)
    got = S.sort_lists(offs, vals)
    assert got.dtype == vals.dtype
    for i in range(len(lens)):
        run = vals[offs[i]:offs[i + 1]].tolist()
        want = sorted(run, key=total_cmp_key) if dtype == np.float64 else sorted(run)
        g = got[offs[i]:offs[i + 1]]
        assert np.array_equal(g.view(np.uint64), np.array(want, dtype=dtype).view(np.uint64))


def test_f64_order_is_total_cmp():
    sp = S.f64_specials()
    got = S.sort_lists([0, len(sp)], sp)
    bits = [int(b) for b in got.view(np.uint64)]
    assert bits[0] == 0xFFFFFFFFFFFFFFFF and bits[-1] == 0x7FFFFFFFFFFFFFFF     # -NaN max payload first, +NaN last
    assert bits.index(0x8000000000000000) + 1 == bits.index(0)                  # -0.0 just before +0.0
    finite = [x for x in got.tolist() if not math.isnan(x)]
    assert finite == sorted(finite, key=total_cmp_key)
    assert [x for x in finite if x != 0] == sorted(x for x in finite if x != 0)


def test_triples_ignore_key_order():
    a = S.triples(np.array([5, 3]), [0, 2, 3], np.array([1, 2, 3], dtype=np.uint64))
    b = S.triples(np.array([3, 5]), [0, 1, 3], np.array([3, 1, 2], dtype=np.uint64))
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


class _Parent:
    def __init__(self, vals):
        self.vals = vals


def test_value_order_argument():
    assert rdd._value_order(False, []) == L.VB_VALORDER_INPUT
    assert rdd._value_order(True, [_Parent(None)]) == L.VB_VALORDER_ASC
    assert rdd._value_order(np.bool_(True), []) == L.VB_VALORDER_ASC
    for bad in (1, 0, "yes", None, 1.0):
        with pytest.raises(TypeError, match="sort_values must be a bool"):
            rdd._value_order(bad, [])
    bcol = rdd._BytesCol(["a", "bc"])
    with pytest.raises(TypeError, match="byte-string values have no value order"):
        rdd._value_order(True, [_Parent(None), _Parent(bcol)])
    assert rdd._value_order(False, [_Parent(bcol)]) == L.VB_VALORDER_INPUT


def test_sort_values_keyword_on_every_grouping_entry():
    import inspect
    for fn in (rdd.PairRdd.group_by_key, rdd.PairRdd.cogroup, rdd.PairRdd.join, rdd.PairRdd.left_outer_join,
               rdd.PairRdd.right_outer_join, rdd.PairRdd.full_outer_join, rdd.CoGroupedRdd.__init__,
               rdd.StrPairRdd.group_by_key, rdd.StrCoGroupedRdd.__init__):
        p = inspect.signature(fn).parameters["sort_values"]
        assert p.default is False, fn
    for cls in (rdd.Shuffle, rdd.StrShuffle):
        assert inspect.signature(cls.__init__).parameters["value_order"].default == L.VB_VALORDER_INPUT
    from vega_b200 import dist
    for fn in (dist.run_shuffle, dist.run_str_shuffle):
        assert inspect.signature(fn).parameters["value_order"].default == L.VB_VALORDER_INPUT


def test_lib_declares_the_abi():
    h = HEADER.read_text()
    assert re.search(r"enum vb_value_order \{ VB_VALORDER_INPUT = 0, VB_VALORDER_ASC = 1 \};", h)
    assert "VB_API int32_t vb_shuffle_set_value_order(vb_shuf *s, int32_t order" in h
    assert (L.VB_VALORDER_INPUT, L.VB_VALORDER_ASC) == (0, 1)
    assert L.SYMBOLS["vb_shuffle_set_value_order"] == (L._i32, [L._vp, L._i32])
