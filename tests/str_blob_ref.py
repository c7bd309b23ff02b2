"""Vec<(String, u64)>, the bincode 1.2.1 bucket of a String-key reduce partition — TEST INFRASTRUCTURE ONLY.

The layout follows the same published bincode defaults as oracle/bincode_ref.py (little-endian, fixed-width integers,
`String` = u64 length then the bytes, tuples = fields in order); its String field is the one of that module's
encode_i32_string_vec, the type of the reference's only bincode fixture.  Byte-level parity with vega is otherwise
unpinned: the reference holds no String bucket bytes.
"""
import struct


def encode_str_pairs(pairs):
    """Vec<(String,u64)> — a String-key reduce partition; keys are str (UTF-8) or bytes, values u64 bit patterns.
    Each record is u64 len | key bytes | u64 value, unaligned; the String field is laid out as in encode_i32_string_vec."""
    out = [struct.pack("<Q", len(pairs))]
    for k, c in pairs:
        b = k.encode() if isinstance(k, str) else bytes(k)
        out.append(struct.pack("<Q", len(b)) + b + struct.pack("<Q", c & (2 ** 64 - 1)))
    return b"".join(out)


def decode_str_pairs(blob):
    """The inverse: [(key bytes, u64)].  Raises ValueError on every malformed shape: fewer than 8 bytes, more records
    than the bytes can hold, a record whose length, key or value runs past the end, trailing bytes."""
    if len(blob) < 8:
        raise ValueError("corrupted blob")
    (n,) = struct.unpack_from("<Q", blob, 0)
    if n > (len(blob) - 8) // 16:
        raise ValueError("corrupted blob")
    pos, out = 8, []
    for _ in range(n):
        if len(blob) - pos < 16:
            raise ValueError("corrupted blob")
        (ln,) = struct.unpack_from("<Q", blob, pos)
        if ln > len(blob) - pos - 16:
            raise ValueError("corrupted blob")
        key = bytes(blob[pos + 8:pos + 8 + ln])
        (c,) = struct.unpack_from("<Q", blob, pos + 8 + ln)
        out.append((key, c))
        pos += 16 + ln
    if pos != len(blob):
        raise ValueError("corrupted blob")
    return out

