"""Placement of byte-slice keys (Rust `Vec<u8>`, `&[u8]`, `Box<[u8]>`, `[u8; N]`), restated in numpy.

`<[u8] as Hash>::hash` writes the slice length as a usize and then the bytes, so the reference's buffering MetroHasher
hashes the stream le64(len) ‖ bytes with MetroHash64_1 (seed 0), and HashPartitioner puts the key in partition
hash % R.  The rounds are those of tests/str_group_ref.py's vectorised restatement (its constants, rotation and
length classes); only the stream differs.  tests/test_bytes_keys_cpu.py pins this to the C oracle's MetroHash64_1."""
import numpy as np

from tests import str_group_ref as S


def _metro_stream(T, n):
    """MetroHash64_1 (seed 0) of every row of the (m, n + 8) byte matrix T, whose first n bytes are the stream."""
    m = T.shape[0]
    K0, K1, K2, K3 = (np.uint64(k) for k in (S._K0, S._K1, S._K2, S._K3))
    rotr = S._rotr

    def w(pos, nb):
        x = np.zeros((m, 8), np.uint8)
        x[:, :nb] = T[:, pos:pos + nb]
        return x.view("<u8")[:, 0]
    with np.errstate(over="ignore"):
        h = np.full(m, (S._K2 * S._K0 + n) & S.MASK64, np.uint64)
        pos = 0
        if n >= 32:
            v0, v1, v2, v3 = h.copy(), h.copy(), h.copy(), h.copy()
            while pos + 32 <= n:
                v0 += w(pos, 8) * K0
                v0 = rotr(v0, 29) + v2
                v1 += w(pos + 8, 8) * K1
                v1 = rotr(v1, 29) + v3
                v2 += w(pos + 16, 8) * K2
                v2 = rotr(v2, 29) + v0
                v3 += w(pos + 24, 8) * K3
                v3 = rotr(v3, 29) + v1
                pos += 32
            v2 ^= rotr(((v0 + v3) * K0) + v1, 33) * K1
            v3 ^= rotr(((v1 + v2) * K1) + v0, 33) * K0
            v0 ^= rotr(((v0 + v2) * K0) + v3, 33) * K1
            v1 ^= rotr(((v1 + v3) * K1) + v2, 33) * K0
            h += v0 ^ v1
        if n - pos >= 16:
            a = h + w(pos, 8) * K0
            a = rotr(a, 33) * K1
            b = h + w(pos + 8, 8) * K1
            b = rotr(b, 33) * K2
            a ^= rotr(a * K0, 35) + b
            b ^= rotr(b * K3, 35) + a
            h += b
            pos += 16
        for nb, rot in ((8, 33), (4, 15), (2, 13), (1, 25)):
            if n - pos >= nb:
                h += w(pos, nb) * K3
                h ^= rotr(h, rot) * K1
                pos += nb
        h ^= rotr(h, 33)
        h *= K0
        h ^= rotr(h, 33)
    return h


def metro64_1_bytes(offsets, data):
    """MetroHash64_1 (seed 0) of le64(len) ‖ key for every key data[offsets[i] .. offsets[i + 1])."""
    h = np.zeros(len(offsets) - 1, np.uint64)
    for rows, L, B in S._classes(offsets, np.asarray(data)):
        T = np.zeros((len(rows), L + 16), np.uint8)
        T[:, :8] = np.frombuffer(np.uint64(L).tobytes(), np.uint8)
        T[:, 8:8 + L] = B
        h[rows] = _metro_stream(T, L + 8)
    return h


def encode(keys):
    """(offsets, data) of a list of bytes keys."""
    offs = np.zeros(len(keys) + 1, np.uint64)
    np.cumsum([len(k) for k in keys], out=offs[1:])
    return offs, np.frombuffer(b"".join(keys), np.uint8)


def partition_of(keys, R):
    """HashPartitioner's partition of every bytes key under Vec<u8> hashing."""
    o, d = encode(keys)
    return (metro64_1_bytes(o, d) % np.uint64(R)).astype(np.int64)


def hash_one(key):
    o, d = encode([key])
    return int(metro64_1_bytes(o, d)[0])
