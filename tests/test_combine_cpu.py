"""CPU-side checks of combine_by_key: the vb_agg_col layout, and argument errors raised before any device work."""
import ctypes

import numpy as np
import pytest

import vega_b200 as vb
from vega_b200 import _lib as L


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def _rdd(n_cols=3, n=10, lengths=None):
    keys = np.arange(n, dtype=np.uint64)
    cols = tuple(np.arange(lengths[i] if lengths else n, dtype=np.uint64) for i in range(n_cols))
    return vb.Context.parallelize(_NoDevice(), keys, 2, values=cols)


def test_agg_col_layout():
    assert ctypes.sizeof(L.vb_agg_col) == 8
    assert [f for f, _ in L.vb_agg_col._fields_] == ["agg", "src"]
    assert L.VB_AGG_MEAN == 7 and L.VB_MAX_VAL_COLS == 4 and L.VB_MAX_AGGS == 8


def test_combine_by_key_accepts_a_valid_spec_without_device_work():
    r = _rdd().combine_by_key({"n": ("count", None), "avg": ("mean", 0), "hi": ("max", 1), "s": ("sum", 2)}, 4)
    assert r.names == ["n", "avg", "hi", "s"]
    assert r.spec == [(L.VB_AGG_COUNT, 0), (L.VB_AGG_MEAN, 0), (L.VB_AGG_MAX, 1), (L.VB_AGG_SUM, 2)]
    assert r.out_dtypes == [np.uint64, np.float64, np.uint64, np.uint64]
    # 7 aggregates with a MEAN: its COUNT makes 8 accumulators
    r = _rdd(1).combine_by_key({f"a{i}": ("mean" if i == 0 else "sum", 0) for i in range(7)}, 2)
    assert len(r.spec) == 7


@pytest.mark.parametrize("aggs", [
    {"x": ("median", 0)},                                   # not a named op
    {"x": ("sum", 3)},                                      # column out of range
    {"x": ("sum", -1)},
    {"x": ("max", None)},                                   # only count ignores its column
    {"x": ("sum",)},                                        # not (op, column)
    {f"a{i}": ("sum", 0) for i in range(9)},                # more than 8 aggregates
    {**{f"a{i}": ("sum", 0) for i in range(7)}, "m": ("mean", 1)},    # 8 + the COUNT a MEAN needs
    {},
])
def test_combine_by_key_rejects_bad_specs(aggs):
    with pytest.raises(ValueError):
        _rdd().combine_by_key(aggs, 4)


def test_combine_by_key_rejects_bad_columns():
    with pytest.raises(ValueError):
        _rdd(5)                                             # more than 4 value columns
    with pytest.raises(ValueError):
        _rdd(3, lengths=[10, 9, 10])                        # mismatched column lengths
    with pytest.raises(ValueError):
        _rdd().combine_by_key({"s": ("sum", 0)}, 0)         # no reduce partitions
    with pytest.raises(TypeError):
        _rdd().reduce_by_key("sum", 2)                      # single-column operators need a single value column


def test_a_list_of_values_stays_one_value_column():
    keys = np.arange(3, dtype=np.uint64)
    r = vb.Context.parallelize(_NoDevice(), keys, 2, values=[5, 6, 7])
    assert r.vals is not None and r.vals.n == 3 and len(r.cols) == 1
    r = vb.Context.parallelize(_NoDevice(), keys, 2, values=([5, 6, 7], [1, 2, 3]))
    assert r.vals is None and len(r.cols) == 2
