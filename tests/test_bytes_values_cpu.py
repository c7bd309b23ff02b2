"""Byte-string values without a GPU: Context.parallelize's forms, and the TypeErrors raised before any device work (a
Context that never reached the device is enough, since nothing here runs a shuffle)."""
import numpy as np
import pytest

import vega_b200 as vb
from vega_b200 import _lib as L
from vega_b200 import dist
from vega_b200.rdd import StrCoGroupedRdd, StrKeys, StrPairRdd, StrSortedRdd, _BytesCol


@pytest.fixture
def sc():
    return vb.Context.__new__(vb.Context)      # no device: parallelize and the refusals do not touch it


def test_parallelize_forms(sc):
    keys = np.arange(3, dtype=np.uint64)
    for vals, as_str in ((["a", "", "é\x00"], True), (np.array(["a", "", "b"]), True), ([b"\xff", b"", b"\x00"], False),
                         (StrKeys(np.array([2, 3, 3, 5], dtype=np.uint64), b"..abc"), True)):
        p = sc.parallelize(keys, 2, values=vals)
        assert type(p) is vb.PairRdd and isinstance(p.vals, _BytesCol)
        assert p.vals.code == L.VB_BYTES and p.vals.as_str is as_str and p.vals.n == 3 and p.vals.loc == L.VB_HOST
    p = sc.parallelize(["x", "y"], 2, values=[b"1", b"2"])
    assert isinstance(p, StrPairRdd) and isinstance(p.vals, _BytesCol) and p.vals.n_bytes == 2
    # numeric values keep their column
    assert not isinstance(sc.parallelize(keys, 2, values=np.arange(3, dtype=np.int64)).vals, _BytesCol)


def test_bytes_encoding():
    c = _BytesCol(["ab", "", "\x00é"])
    raw = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_uint8 * c.n_bytes).from_address(c.data_ptr)).tobytes()
    assert raw == "ab\x00é".encode()
    with pytest.raises(TypeError):
        _BytesCol(["a", b"b"])


def test_refusals_before_device_work(sc):
    keys = np.arange(4, dtype=np.uint64)
    p = sc.parallelize(keys, 2, values=["a", "b", "c", "d"])
    with pytest.raises(TypeError):
        p.reduce_by_key("sum", 2)
    with pytest.raises(TypeError):
        p.count_by_key(2)
    with pytest.raises(TypeError):
        p.combine_by_key({"n": ("count", None)}, 2)
    s = sc.parallelize(["a", "b"], 1, values=["x", "y"])
    with pytest.raises(TypeError):
        s.reduce_by_key("max", 2)
    with pytest.raises(TypeError):
        s.count_by_key(2)
    with pytest.raises(TypeError):
        s.combine_by_key({"n": ("count", None)}, 2)
    with pytest.raises(TypeError):
        dist.run_shuffle(None, [], 1, 1, L.VB_U64, L.VB_BYTES, L.VB_AGG_GROUP, 0, 2)
    with pytest.raises(TypeError):
        dist.run_str_shuffle(None, [], 1, 1, L.VB_BYTES, L.VB_AGG_GROUP, 0, 2)
    # the binary String-key join family stays refused
    with pytest.raises(TypeError):
        s.join(s, 2)
    # the op classes themselves construct without device work
    StrCoGroupedRdd([s, s], 2)
    StrSortedRdd(s, 2)


def test_bytes_keys_still_refused(sc):
    with pytest.raises(TypeError):
        sc.parallelize([b"a", b"b"], 1, values=["x", "y"])
    with pytest.raises(TypeError):
        sc.parallelize(np.array([b"a", b"b"]), 1, values=["x", "y"])
