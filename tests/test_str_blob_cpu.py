"""The Vec<(String, u64)> codec of tests/str_blob_ref.py that the String-key blob tests compare against (no GPU)."""
import struct

import numpy as np
import pytest

from oracle import bincode_ref as B
from tests import str_blob_ref as S


def test_literal():
    assert S.encode_str_pairs([("ab", 3)]) == b"\x01" + b"\x00" * 7 + b"\x02" + b"\x00" * 7 + b"ab" + b"\x03" + b"\x00" * 7
    assert S.encode_str_pairs([]) == b"\x00" * 8


def test_string_field_matches_the_reference_fixture():
    """(0, "example data") is the only bincode the reference pins: its String field (u64 length, then the bytes) is
    the key field of a String record."""
    fixture = B.encode_i32_string_vec([(0, "example data")])
    ours = S.encode_str_pairs([("example data", 7)])
    assert fixture[:8] == ours[:8]                       # the Vec length
    assert fixture[8 + 4:] == ours[8:-8]                 # after the i32: u64 len | bytes
    assert ours[-8:] == struct.pack("<Q", 7)


def test_round_trip():
    rng = np.random.default_rng(5)
    keys = ["", "é", "日本語", "\x00"] + ["k" * n for n in range(1, 18)] + ["z" * 70_000]
    pairs = [(k, int(rng.integers(0, 2 ** 64, dtype=np.uint64))) for k in keys] + [("max", 2 ** 64 - 1)]
    blob = S.encode_str_pairs(pairs)
    assert len(blob) == 8 + 16 * len(pairs) + sum(len(k.encode()) for k, _ in pairs)
    assert S.decode_str_pairs(blob) == [(k.encode(), v) for k, v in pairs]
    assert S.decode_str_pairs(b"\x00" * 8) == []
    assert S.encode_str_pairs([(b"\xff\xfe", 1)]) == S.encode_str_pairs([(bytearray(b"\xff\xfe"), 1)])


def corrupt_blobs():
    """One blob of each malformed shape, each from the valid [("ab", 3), ("", 4)]."""
    good = S.encode_str_pairs([("ab", 3), ("", 4)])
    return {
        "short": good[:7],
        "too_many_records": struct.pack("<Q", 3) + good[8:],
        "huge_count": struct.pack("<Q", 2 ** 63) + good[8:],
        "length_runs_past_end": good[:8 + 18] + b"\x00" * 4,
        "key_runs_past_end": good[:8] + struct.pack("<Q", 2 ** 40) + good[16:],
        "value_runs_past_end": good[:-3],
        "trailing_bytes": good + b"\x00",
    }


@pytest.mark.parametrize("shape", list(corrupt_blobs()))
def test_decoder_rejects(shape):
    with pytest.raises(ValueError):
        S.decode_str_pairs(corrupt_blobs()[shape])
