"""Reference of sorted value lists (vb_shuffle_set_value_order, sort_values=True) (test infrastructure).

Each key's list is sorted ascending by the value's order key, the library's tx_fwd: the bits themselves for u64, the
bits with the sign bit flipped for i64, and for f64 all bits flipped on a negative value and the sign bit set on any
other, which is f64::total_cmp (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN, NaNs by payload).  Two values tie
only when their bits are equal, so a sorted list is unique and compares bit for bit.
"""
import numpy as np

SIGN = np.uint64(1 << 63)


def order_key(vals):
    """tx_fwd of every value (u64, i64 or f64 array) as u64."""
    v = np.ascontiguousarray(vals)
    b = v.view(np.uint64)
    if v.dtype == np.int64:
        return b ^ SIGN
    if v.dtype == np.float64:
        return np.where(b & SIGN, ~b, b | SIGN)
    assert v.dtype == np.uint64, v.dtype
    return b.copy()


def sort_lists(offsets, vals):
    """vals with every run vals[offsets[i] .. offsets[i+1]) sorted by order_key; same dtype."""
    offsets = np.asarray(offsets, dtype=np.int64)
    v = np.ascontiguousarray(vals)
    run = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    return v[np.lexsort((order_key(v), run))]


def triples(keys, offsets, vals):
    """(key, position in the key's list, value bits) per value, ordered by key then position: two grouped results are
    equal when these are, whatever the order of the keys."""
    offsets = np.asarray(offsets, dtype=np.int64)
    lens = np.diff(offsets)
    k = np.repeat(np.asarray(keys), lens)
    pos = np.arange(len(k)) - np.repeat(offsets[:-1], lens)
    bits = np.ascontiguousarray(vals).view(np.uint64)
    o = np.lexsort((pos, k))
    return k[o], pos[o], bits[o]


def f64_specials():
    """Bit patterns of every f64 class whose order the sort must get right, as float64."""
    pats = [0x0000000000000000, 0x8000000000000000,                            # +0.0, -0.0
            0x7FF0000000000000, 0xFFF0000000000000,                            # +inf, -inf
            0x7FF8000000000000, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF,        # +NaNs: quiet, signalling, max payload
            0xFFF8000000000000, 0xFFF0000000000001, 0xFFFFFFFFFFFFFFFF,        # -NaNs
            0x0000000000000001, 0x000FFFFFFFFFFFFF, 0x8000000000000001,        # subnormals of both signs
            0x800FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF,        # smallest normal, largest finite
            0xFFEFFFFFFFFFFFFF, 0x3FF0000000000000, 0xBFF0000000000000]        # -max, 1.0, -1.0
    return np.array(pats, dtype=np.uint64).view(np.float64)


def full_range(rng, n, dtype):
    """n values of dtype over its full bit range, with the f64 specials (and i64 / u64 extremes) mixed in."""
    bits = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    if dtype == np.float64:
        sp = f64_specials().view(np.uint64)
    else:
        sp = np.array([0, 1, (1 << 63) - 1, 1 << 63, (1 << 64) - 1], dtype=np.uint64)
    if n:
        at = rng.integers(0, n, max(1, n // 8))
        bits[at] = sp[rng.integers(0, len(sp), len(at))]
    return bits.view(dtype)
