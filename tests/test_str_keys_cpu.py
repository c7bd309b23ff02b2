"""String keys without a GPU: the library's host hash of a byte-string key is MetroHash64_1(bytes ‖ 0xFF) (Rust's
`impl Hash for str` fed to the MetroHasher), its partition is pyref's, the mirror's (offsets, bytes) encoding
round-trips, and argument errors are raised before any device work."""
import ctypes

import numpy as np
import pytest

import vega_b200 as vb
from oracle import oracle as O
from oracle import pyref


def _hash(b):
    return vb.lib().vb_hash_str(ctypes.c_char_p(b), len(b))


def test_hash_matches_metrohash_with_str_suffix_every_length():
    rng = np.random.default_rng(1)
    for n in range(0, 301):
        for b in (bytes(rng.integers(0, 256, n, dtype=np.uint8)), b"\x00" * n, b"a" * n):
            assert _hash(b) == O.metrohash64_1(b + b"\xff", 0), n


def test_hash_of_utf8_and_nul_keys():
    for s in ["", "x", "y", "\x00", "a\x00b", "é", "日本語", "🙂" * 9, "k" * 10_000]:
        b = s.encode()
        assert _hash(b) == O.metrohash64_1(pyref.key_bytes(s), 0)


@pytest.mark.parametrize("R", [1, 3, 300, 65536])
def test_partition_matches_pyref(R):
    rng = np.random.default_rng(R)
    keys = ["", "x", "y", "\x00", "é"] + ["".join(rng.choice(list("abc\x00é"), int(rng.integers(0, 40)))) for _ in range(300)]
    for k in keys:
        b = k.encode()
        assert vb.lib().vb_get_partition_str(ctypes.c_char_p(b), len(b), R) == pyref.get_partition(k, R)


def test_mirror_encoding_round_trips():
    keys = ["", "a", "\x00", "ab\x00", "é", "日本語", "x" * 1000, "trailing nul\x00"]
    k = vb.StrKeys.from_strs(keys)
    assert k.offsets.dtype == np.uint64 and k.offsets[0] == 0 and len(k) == len(keys)
    assert k.offsets.tolist() == np.cumsum([0] + [len(s.encode()) for s in keys]).tolist()
    assert k.data.tobytes() == b"".join(s.encode() for s in keys)
    assert k.to_strs().tolist() == keys                       # NULs survive (a numpy 'U' array would strip trailing ones)
    # a slice of a larger column: offsets need not start at 0
    sub = vb.StrKeys(k.offsets[2:5], k.data)
    assert sub.to_strs().tolist() == keys[2:4]
    assert vb.StrKeys.from_strs([]).to_strs().tolist() == []


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_python_mirror_argument_errors_before_device_work():
    sc = _NoDevice()
    keys = ["x", "y", "x"]
    vals = np.array([1, 2, 3], dtype=np.uint64)
    with pytest.raises(TypeError):
        vb.Context.parallelize(sc, [b"x", b"y"], 2, values=vals)       # Vec<u8> hashes with a length prefix
    with pytest.raises(TypeError):
        vb.Context.parallelize(sc, np.array([b"x", b"y"]), 2)
    with pytest.raises(TypeError):
        vb.Context.parallelize(sc, ["x", 1], 2)
    a = vb.Context.parallelize(sc, keys, 2, values=vals)
    assert isinstance(a, vb.StrPairRdd) and a.n == 3
    assert isinstance(vb.Context.parallelize(sc, (keys, vals), 2), vb.StrPairRdd)
    assert isinstance(vb.Context.parallelize(sc, np.array(keys), 2, values=vals), vb.StrPairRdd)
    r = vb.Context.parallelize(sc, keys, 2)
    assert isinstance(r, vb.StrRdd)
    for method, args in [("join", (a, 2)), ("left_outer_join", (a, 2)), ("right_outer_join", (a, 2)), ("full_outer_join", (a, 2)),
                         ("cogroup", (a, 2)), ("sort_by_key", (2,)), ("combine_by_key", ({"n": ("count", None)}, 2))]:
        with pytest.raises(TypeError):
            getattr(a, method)(*args)
    for method, args in [("sort", (2,)), ("intersection", (r,)), ("subtract", (r,)), ("group_by", (len,))]:
        with pytest.raises(TypeError):
            getattr(r, method)(*args)
    with pytest.raises(ValueError):
        a.reduce_by_key("mean", 2)
    with pytest.raises(ValueError):
        a.group_by_key(0)
    # valid: lazy, no device work yet
    assert a.reduce_by_key("sum", 3).num_slices == 3
    assert a.group_by_key(2).agg_name == "group"
    assert a.count_by_key().num_slices == 2
    assert r.count_by_value().agg_name == "count"
    a.partition_by_key(4)
    r.distinct(3)
    # integer keys keep their path
    assert type(vb.Context.parallelize(sc, np.arange(4, dtype=np.uint64), 2)) is vb.Rdd
