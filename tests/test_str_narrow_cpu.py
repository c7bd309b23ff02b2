"""CPU checks of String reduce and combine results as cogroup / join parents (StrCoGroupedRdd over views of
vb_shuffle_create_narrow_str): the mirror's argument errors come before any device work, StrAggregateRdd parents are
accepted lazily, the refusals that stay are still raised, and the C ABI declares the new entry point."""
import os

import numpy as np
import pytest

import vega_b200 as vb


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def _pair(sc, keys=("x", "y", "x"), cols=True):
    n = len(keys)
    if cols:
        return vb.Context.parallelize(sc, list(keys), 2, values=(np.arange(n, dtype=np.uint64), np.linspace(0, 1, n)))
    return vb.Context.parallelize(sc, list(keys), 2, values=np.arange(n, dtype=np.uint64))


def test_aggregate_parents_are_accepted_lazily():
    sc = _NoDevice()
    comb = _pair(sc).combine_by_key({"s": ("sum", 0), "avg": ("mean", 1), "n": ("count", None)}, 3)
    agg = comb.aggregate("avg")
    assert isinstance(agg, vb.StrAggregateRdd) and agg.num_slices == 3 and agg.combined is comb
    plain = _pair(sc, cols=False)
    cg = vb.StrCoGroupedRdd([plain, comb.aggregate("s"), agg, comb.aggregate("n"), plain.reduce_by_key("max", 3),
                             plain.count_by_key(4)], 3)
    assert cg.num_slices == 3 and len(cg.rdds) == 6
    assert vb.StrCoGroupedRdd([agg], 5).num_slices == 5                 # another num_splits: reshuffled when run
    assert vb.StrCoGroupedRdd([agg, agg], 3).rdds == [agg, agg]


def test_result_columns_and_dtypes():
    sc = _NoDevice()
    comb = _pair(sc).combine_by_key({"s": ("sum", 0), "lo": ("min", 1), "avg": ("mean", 0), "n": ("count", None)}, 3)
    L = vb._lib
    got = [comb.aggregate(name)._result_col(None) for name in ("s", "lo", "avg", "n")]
    assert got == [(0, 4, L.VB_U64), (1, 4, L.VB_F64), (2, 4, L.VB_F64), (3, 4, L.VB_U64)]


def test_unknown_aggregate_name():
    sc = _NoDevice()
    comb = _pair(sc).combine_by_key({"s": ("sum", 0)}, 3)
    for bad in ("sum", "S", "", None):
        with pytest.raises(ValueError):
            comb.aggregate(bad)


def test_invalid_parents_before_device_work():
    sc = _NoDevice()
    p = _pair(sc)
    comb = p.combine_by_key({"s": ("sum", 0)}, 3)
    ints = vb.Context.parallelize(sc, (np.arange(3, dtype=np.uint64), np.arange(3, dtype=np.uint64)), 2)
    int_comb = vb.Context.parallelize(sc, np.arange(3, dtype=np.uint64), 2, values=(np.arange(3, dtype=np.uint64),)) \
        .combine_by_key({"s": ("sum", 0)}, 3)
    for bad in (comb, int_comb.aggregate("s"), ints.reduce_by_key("sum", 3), _pair(sc, cols=False).group_by_key(3), ints):
        with pytest.raises(TypeError):
            vb.StrCoGroupedRdd([comb.aggregate("s"), bad], 3)
    with pytest.raises(TypeError):                                       # another context
        vb.StrCoGroupedRdd([comb.aggregate("s"), _pair(_NoDevice()).combine_by_key({"s": ("sum", 0)}, 3).aggregate("s")], 3)
    with pytest.raises(ValueError):
        vb.StrCoGroupedRdd([comb.aggregate("s")], 0)
    # the integer cogroup and join keep refusing String parents, a String aggregate included
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([comb.aggregate("s")], 3)
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([int_comb.aggregate("s"), comb.aggregate("s")], 3)
    with pytest.raises(TypeError):
        vb.JoinedRdd(int_comb.aggregate("s"), comb.aggregate("s"), 3)


def test_pinned_refusals_stay():
    sc = _NoDevice()
    a, b = _pair(sc, cols=False), _pair(sc, ("y", "z"), cols=False)
    for rdd in (a, a.reduce_by_key("sum", 3), a.count_by_key(3)):
        for method in ("join", "left_outer_join", "right_outer_join", "full_outer_join", "cogroup"):
            with pytest.raises(TypeError):
                getattr(rdd, method)(b, 2)
    with pytest.raises(TypeError):
        a.sort_by_key(2)
    with pytest.raises(TypeError):
        vb.StrCoGroupedRdd([_pair(sc).combine_by_key({"s": ("sum", 0)}, 2), a], 2)
    with pytest.raises(TypeError):
        vb.CoGroupedRdd([a, b], 2)


def test_abi_declares_the_entry_point():
    assert "vb_shuffle_create_narrow_str" in vb.SYMBOLS
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "vega_b200.h")).read()
    assert "VB_API int32_t vb_shuffle_create_narrow_str(vb_shuf *parent, uint32_t out_col, vb_shuf **out);" in header
