"""Byte-slice keys without a GPU: the placement restated in tests/bytes_keys_ref.py is MetroHash64_1(le64(len) ‖ bytes)
by the C oracle, the library's vb_hash_bytes / vb_get_partition_bytes equal it, the two key kinds place keys
differently, and the Python mirror's argument errors come before any device work."""
import ctypes
import struct

import numpy as np
import pytest

import vega_b200 as vb
from oracle import oracle as O
from tests import bytes_keys_ref as B


def _keys():
    rng = np.random.default_rng(7)
    keys = [b""] + [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in range(1, 301)]
    keys += [b"\x00" * n for n in range(0, 80)] + [b"\xff" * n for n in range(0, 80)]
    keys += [bytes(rng.integers(0, 256, int(rng.integers(0, 301)), dtype=np.uint8)) for _ in range(500)]
    return keys


def test_restatement_matches_oracle_metrohash():
    keys = _keys()
    o, d = B.encode(keys)
    want = [O.metrohash64_1(struct.pack("<Q", len(k)) + k, 0) for k in keys]
    assert B.metro64_1_bytes(o, d).tolist() == want
    same = [keys[57]] * 6                    # one length class: read as one matrix
    o, d = B.encode(same)
    assert B.metro64_1_bytes(o, d).tolist() == want[57:58] * 6


def test_library_hash_and_partition_match_restatement():
    lib = vb.lib()
    keys = _keys()
    o, d = B.encode(keys)
    h = B.metro64_1_bytes(o, d)
    for k, hk in zip(keys, h.tolist()):
        assert lib.vb_hash_bytes(ctypes.c_char_p(k), len(k)) == hk, len(k)
    for R in (1, 3, 257, 65536):
        want = (h % np.uint64(R)).tolist()
        got = [lib.vb_get_partition_bytes(ctypes.c_char_p(k), len(k), R) for k in keys]
        assert got == want, R
    assert lib.vb_get_partition_bytes(ctypes.c_char_p(b"x"), 1, 0) == 0


def test_the_two_kinds_place_keys_differently():
    """A kind silently ignored would still pass every multiset check: the placements must differ for most keys."""
    lib = vb.lib()
    keys = _keys()
    hs = [lib.vb_hash_str(ctypes.c_char_p(k), len(k)) for k in keys]
    hb = [lib.vb_hash_bytes(ctypes.c_char_p(k), len(k)) for k in keys]
    assert all(a != b for a, b in zip(hs, hb))
    R = 257
    differ = sum(lib.vb_get_partition_str(ctypes.c_char_p(k), len(k), R) != lib.vb_get_partition_bytes(ctypes.c_char_p(k), len(k), R)
                 for k in keys)
    assert differ > 0.9 * len(keys)


def test_bytes_keys_column():
    keys = [b"", b"x", b"\x00", b"\xff\xfe", b"ab\x00", bytes(range(256)), b"\x80not utf-8"]
    k = vb.BytesKeys.from_bytes(keys)
    assert isinstance(k, vb.StrKeys) and len(k) == len(keys)
    assert k.offsets.tolist() == np.cumsum([0] + [len(x) for x in keys]).tolist()
    assert k.data.tobytes() == b"".join(keys)
    assert k.to_bytes().tolist() == keys
    assert vb.BytesKeys(k.offsets[1:4], k.data).to_bytes().tolist() == keys[1:3]
    assert vb.BytesKeys.from_bytes([bytearray(b"q")]).to_bytes().tolist() == [b"q"]
    assert vb.BytesKeys.from_bytes([]).to_bytes().tolist() == []


class _NoDevice:
    """Stands in for a Context: any use of it (a device call) fails the test."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the arguments were checked")


def test_python_argument_errors_before_device_work():
    sc = _NoDevice()
    vals = np.array([1, 2, 3], dtype=np.uint64)
    # a plain list or array of bytes is still refused, and the message points to BytesKeys
    for data in ([b"x", b"y", b"x"], np.array([b"x", b"y", b"x"])):
        with pytest.raises(TypeError, match="BytesKeys"):
            vb.Context.parallelize(sc, data, 2, values=vals)
    bk = vb.BytesKeys.from_bytes([b"x", b"y", b"x"])
    a = vb.Context.parallelize(sc, bk, 2, values=vals)
    assert isinstance(a, vb.StrPairRdd) and a.n == 3 and a.keys.key_kind == vb._lib.VB_STRKEY_BYTES
    r = vb.Context.parallelize(sc, bk, 2)
    assert isinstance(r, vb.StrRdd) and r.keys.key_kind == vb._lib.VB_STRKEY_BYTES
    s = vb.Context.parallelize(sc, ["x", "y", "x"], 2, values=vals)
    assert s.keys.key_kind == vb._lib.VB_STRKEY_STR
    bv = vb.Context.parallelize(sc, bk, 2, values=["p", "q", "r"])        # byte-string values beside bytes keys
    assert isinstance(bv, vb.StrPairRdd) and bv.keys.key_kind == vb._lib.VB_STRKEY_BYTES
    # lazy ops build without device work
    assert a.reduce_by_key("sum", 3).num_slices == 3
    a.group_by_key(2)
    a.count_by_key()
    r.count_by_value()
    r.distinct(3)
    # cogroup / joins: bytes-keyed and String-keyed parents are refused before any device work, in any position
    for rdds in ([a, s], [s, a], [a, a, s], [a.reduce_by_key("sum", 2), s], [s.count_by_key(2), a.group_by_key(2).parent]):
        with pytest.raises(TypeError, match="BytesKeys"):
            vb.StrCoGroupedRdd(rdds, 2)
    assert vb.StrCoGroupedRdd([a, a.reduce_by_key("sum", 2)], 2).key_kind == vb._lib.VB_STRKEY_BYTES
    assert vb.StrCoGroupedRdd([s, s], 2).key_kind == vb._lib.VB_STRKEY_STR


def test_header_documents_the_kind():
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vega_b200.h")).read()
    assert "VB_STRKEY_STR = 0, VB_STRKEY_BYTES = 1" in src
    for name in ("vb_shuffle_set_str_key", "vb_hash_bytes", "vb_get_partition_bytes"):
        assert name in vb.SYMBOLS
