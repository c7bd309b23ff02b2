"""Vectorised references of String-key group_by_key, cogroup and the joins (test infrastructure), exact at tens of
millions of rows.

Keys are built from integer ranks by a bijection, so the integer references of tests/group_ref.py (group_triples,
join_rows, _by_key_then_pos) give the expected lists and join rows with the ranks as keys:
    key(rank) = the rank's 8 little-endian bytes cut to L bytes, then pad bytes PAD[8 .. L),
    L = max(lens[rank % len(lens)], bytes the rank needs).
Distinct ranks give distinct keys (equal lengths: the first min(L, 8) bytes hold the whole rank), and a key decodes
from its first min(L, 8) bytes.  With LENS the lengths cross every step of MetroHash64_1 over the hashed stream
key ‖ 0xFF: 0 (rank 0 is the empty key), 1-3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 64, 65 and 100 bytes.  Keys hold NUL
bytes (the rank's high zero bytes, PAD) and 0xFF bytes (rank 2^(8j) - 1 is j bytes of 0xFF: rank 255 is b"\\xff";
PAD).  Keys of different lengths share prefixes (rank r and rank r + 256^j k of a longer length).  encode (numpy) and
encode_torch (host or device tensors) write the same bytes.

decode checks every byte of every key against the encoding of the rank it decodes to, so equal ranks mean equal
bytes.  Placement is HashPartitioner's over `impl Hash for str`: MetroHash64_1 (seed 0) of key ‖ 0xFF, modulo R
(metro64_1_str).  tests/test_str_group_ref_cpu.py pins every function here to the C oracle and to oracle/pyref.py.
"""
import numpy as np

from tests import group_ref as G

LENS = (0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 32, 33, 64, 65, 100, 4)
ALL_FF = 255                      # rank of the key b"\xff" (255 % len(LENS) == 0, LENS[0] == 0)
MASK64 = (1 << 64) - 1
_K0, _K1, _K2, _K3 = 0xC83A91E1, 0x8648DBDB, 0x7BDEC03B, 0x2F5870A5


def pad(L):
    """The pad bytes PAD[0 .. L) (bytes 0-7 of a key are the rank's): 0x00 every 7th, 0xFF every 5th byte."""
    j = np.arange(L, dtype=np.int64)
    p = (j * 0x9D + 0x1F) & 0xFF
    p[j % 5 == 0] = 0xFF
    p[j % 7 == 0] = 0x00
    return p.astype(np.uint8)


def key_lens(ranks, lens=LENS):
    """Key length of every rank (u64 array)."""
    r = np.asarray(ranks, dtype=np.uint64)
    nb = np.zeros(len(r), np.int64)
    for s in range(8):
        nb += (r >> np.uint64(8 * s)) > 0
    return np.maximum(np.asarray(lens, np.int64)[(r % np.uint64(len(lens))).astype(np.int64)], nb)


def _byte(r, t, P):
    """Byte t of the keys of ranks r (all at least t + 1 bytes long)."""
    if t < 8:
        return ((r >> np.uint64(8 * t)) & np.uint64(0xFF)).astype(np.uint8)
    return np.full(len(r), P[t], np.uint8)


def encode(ranks, lens=LENS):
    """(offsets u64 [n + 1] from 0, bytes u8) of the keys of ranks, in order."""
    r = np.asarray(ranks, dtype=np.uint64)
    L = key_lens(r, lens)
    offs = np.zeros(len(r) + 1, np.uint64)
    np.cumsum(L, out=offs[1:])
    data = np.empty(int(offs[-1]), np.uint8)
    P = pad(int(L.max(initial=0)))
    for u in np.unique(L).tolist():
        rows = np.flatnonzero(L == u)
        o = offs[:-1][rows].astype(np.int64)
        for t in range(u):
            data[o + t] = _byte(r[rows], t, P)
    return offs, data


def encode_torch(ranks, lens=LENS):
    """encode of an int64 tensor of ranks (each below 2^63) with torch, on the ranks' device: int64 offsets, uint8
    bytes."""
    import torch
    r = ranks
    dev = r.device
    nb = torch.zeros_like(r)
    for s in range(8):
        nb += (r >> (8 * s)) > 0
    L = torch.maximum(torch.tensor(lens, dtype=torch.int64, device=dev)[r % len(lens)], nb)
    offs = torch.zeros(len(r) + 1, dtype=torch.int64, device=dev)
    torch.cumsum(L, 0, out=offs[1:])
    data = torch.empty(int(offs[-1]), dtype=torch.uint8, device=dev)
    P = torch.from_numpy(pad(int(L.max()) if len(r) else 0)).to(dev)
    uniq = torch.unique(L).tolist()
    for u in uniq:
        if len(uniq) == 1:                                   # one length: the keys are the rows of an (n, u) matrix
            m = data.view(len(r), u)
            for t in range(min(u, 8)):
                m[:, t] = ((r >> (8 * t)) & 0xFF).to(torch.uint8)
            if u > 8:
                m[:, 8:] = P[8:u]
            break
        rows = torch.nonzero(L == u).flatten()
        o = offs[:-1][rows]
        rr = r[rows]
        for t in range(u):
            data[o + t] = ((rr >> (8 * t)) & 0xFF).to(torch.uint8) if t < 8 else P[t]
    return offs, data


# ---- MetroHash64_1 of key ‖ 0xFF ------------------------------------------------------------------------------------
def _rotr(v, k):
    return (v >> np.uint64(k)) | (v << np.uint64(64 - k))


def _metro_rows(B):
    """MetroHash64_1 (seed 0) of every row of the (m, L) byte matrix B followed by one 0xFF byte."""
    m, L = B.shape
    n = L + 1
    S = np.zeros((m, n + 8), np.uint8)
    S[:, :L] = B
    S[:, L] = 0xFF
    K0, K1, K2, K3 = (np.uint64(k) for k in (_K0, _K1, _K2, _K3))

    def w(pos, nb):
        x = np.zeros((m, 8), np.uint8)
        x[:, :nb] = S[:, pos:pos + nb]
        return x.view("<u8")[:, 0]
    h = np.full(m, (_K2 * _K0 + n) & MASK64, np.uint64)
    pos = 0
    if n >= 32:
        v0, v1, v2, v3 = h.copy(), h.copy(), h.copy(), h.copy()
        while pos + 32 <= n:
            v0 += w(pos, 8) * K0
            v0 = _rotr(v0, 29) + v2
            v1 += w(pos + 8, 8) * K1
            v1 = _rotr(v1, 29) + v3
            v2 += w(pos + 16, 8) * K2
            v2 = _rotr(v2, 29) + v0
            v3 += w(pos + 24, 8) * K3
            v3 = _rotr(v3, 29) + v1
            pos += 32
        v2 ^= _rotr(((v0 + v3) * K0) + v1, 33) * K1
        v3 ^= _rotr(((v1 + v2) * K1) + v0, 33) * K0
        v0 ^= _rotr(((v0 + v2) * K0) + v3, 33) * K1
        v1 ^= _rotr(((v1 + v3) * K1) + v2, 33) * K0
        h += v0 ^ v1
    if n - pos >= 16:
        a = h + w(pos, 8) * K0
        a = _rotr(a, 33) * K1
        b = h + w(pos + 8, 8) * K1
        b = _rotr(b, 33) * K2
        a ^= _rotr(a * K0, 35) + b
        b ^= _rotr(b * K3, 35) + a
        h += b
        pos += 16
    for nb, rot in ((8, 33), (4, 15), (2, 13), (1, 25)):
        if n - pos >= nb:
            h += w(pos, nb) * K3
            h ^= _rotr(h, rot) * K1
            pos += nb
    h ^= _rotr(h, 33)
    h *= K0
    h ^= _rotr(h, 33)
    return h


def _classes(offsets, data):
    """(rows, L, (m, L) byte matrix) for every key length L of the keys data[offsets[i] .. offsets[i + 1])."""
    o = np.asarray(offsets).astype(np.int64)
    lens = np.diff(o)
    n = len(lens)
    assert (lens >= 0).all(), "key offsets are not monotone"
    if n and (lens == lens[0]).all():                         # one length: the keys are the rows of a matrix
        u = int(lens[0])
        yield np.arange(n), u, np.asarray(data[o[0]:o[0] + n * u]).reshape(n, u)
        return
    for u in np.unique(lens).tolist():
        rows = np.flatnonzero(lens == u)
        starts = o[:-1][rows]
        B = np.empty((len(rows), u), np.uint8)
        for t in range(u):
            B[:, t] = data[starts + t]
        yield rows, u, B


def metro64_1_str(offsets, data):
    """MetroHash64_1 (seed 0) of every key ‖ 0xFF: `str::hash` fed to HashPartitioner's MetroHasher."""
    h = np.zeros(len(offsets) - 1, np.uint64)
    for rows, _, B in _classes(offsets, data):
        h[rows] = _metro_rows(B)
    return h


def decode(offsets, data, lens=LENS, with_hash=False):
    """The rank of every key, asserting that each key is the encoding of its rank byte for byte; with_hash: also
    metro64_1_str of every key."""
    n = len(offsets) - 1
    ranks = np.zeros(n, np.uint64)
    h = np.zeros(n, np.uint64) if with_hash else None
    for rows, u, B in _classes(offsets, data):
        r = np.zeros(len(rows), np.uint64)
        for t in range(min(u, 8)):
            r |= B[:, t].astype(np.uint64) << np.uint64(8 * t)
        bad = np.flatnonzero(key_lens(r, lens) != u)
        assert not len(bad), f"{len(bad)} keys of {u} bytes are not the encoding of a rank, first {B[bad[0]].tobytes()!r}"
        for t in range(min(u, 8)):
            bad = np.flatnonzero(B[:, t] != _byte(r, t, None))
            assert not len(bad), f"byte {t} of {len(bad)} keys of {u} bytes differs, first key {B[bad[0]].tobytes()!r}"
        P = pad(u)[8:]
        step = max(1, (1 << 26) // max(u, 1))
        for a in range(0, len(rows) if u > 8 else 0, step):
            bad = np.flatnonzero(~(B[a:a + step, 8:] == P).all(axis=1))
            assert not len(bad), f"a pad byte of {len(bad)} keys of {u} bytes differs, first key {B[a + bad[0]].tobytes()!r}"
        ranks[rows] = r
        if with_hash:
            h[rows] = _metro_rows(B)
    return (ranks, h) if with_hash else ranks


def partition_of(ranks, R, lens=LENS):
    """The partition of the key of every rank."""
    o, d = encode(ranks, lens)
    return (metro64_1_str(o, d) % np.uint64(R)).astype(np.int64)


def distinct_ranks(D, first=0):
    """D distinct ranks first, first + 1, ...; from D >= 3 on, with first = 0, the empty key (rank 0) and b"\\xff"
    (ALL_FF) are among them."""
    r = np.arange(first, first + D, dtype=np.uint64)
    if first == 0 and 3 <= D <= ALL_FF:
        r[-1] = ALL_FF
    return r


def rows_over(rng, pool, n, hot=0.0):
    """n rows over exactly the ranks of pool: every rank once, plus n - len(pool) random draws, shuffled; hot > 0:
    about that share of the rows is pool[2]."""
    D = len(pool)
    extra = rng.integers(0, D, n - D)
    if hot:
        extra[rng.random(n - D) < hot * n / (n - D)] = 2
    return pool[rng.permutation(np.concatenate([np.arange(D), extra]))]


def rank_rows(rng, n, D, hot=0.0, first=0):
    """rows_over distinct_ranks(D, first)."""
    return rows_over(rng, distinct_ranks(D, first), n, hot)


# ---- device results in the form of tests/group_ref.py ----------------------------------------------------------------
def _check_offsets(o, total, what, allow_empty=True):
    o = np.asarray(o).astype(np.int64)
    assert len(o) >= 1 and o[0] == 0 and o[-1] == total, f"{what}: offsets run {o[:1]} .. {o[-1:]}, want 0 .. {total}"
    cnt = np.diff(o)
    assert (cnt >= 0).all(), f"{what}: offsets are not monotone"
    assert allow_empty or (cnt > 0).all(), f"{what}: a key with an empty list"
    return cnt


def str_keys_of(parts, R, lens=LENS, placed=None):
    """parts[r][0:2] = (key offsets, key bytes) of partition r.  Checks the key offsets, decodes every key, checks that
    it is in partition metro64_1_str(key) % R and that no key appears twice; returns (ranks of every partition's keys
    in order, the partition of each).  placed: (sorted ranks, their partitions) of keys already checked, which then
    stand for the hash of these keys."""
    assert len(parts) == R, (len(parts), R)
    offs, datas, part, base = [np.zeros(1, np.int64)], [], [], 0
    for r, p in enumerate(parts):
        ko, kb = p[0], p[1]
        cnt = _check_offsets(ko, len(kb), f"partition {r} key bytes")
        offs.append(np.asarray(ko[1:]).astype(np.int64) + base)
        datas.append(np.asarray(kb))
        part.append(np.full(len(cnt), r, np.int64))
        base += len(kb)
    offs = np.concatenate(offs)
    data = np.concatenate(datas) if len(datas) > 1 else datas[0] if datas else np.zeros(0, np.uint8)
    part = np.concatenate(part) if part else np.zeros(0, np.int64)
    if R == 1:                                                # every hash is in partition 0
        ranks = decode(offs, data, lens)
    elif placed is not None:
        ranks = decode(offs, data, lens)
        pr, pp = placed
        i = np.minimum(np.searchsorted(pr, ranks), max(len(pr) - 1, 0))
        assert len(pr) or not len(ranks)
        bad = np.flatnonzero((pr[i] != ranks) | (pp[i] != part)) if len(ranks) else []
        assert not len(bad), f"{len(bad)} keys not in the partition of the checked key, first rank {int(ranks[bad[0]])}"
    else:
        ranks, h = decode(offs, data, lens, with_hash=True)
        bad = np.flatnonzero((h % np.uint64(R)).astype(np.int64) != part)
        assert not len(bad), f"{len(bad)} keys hash to another partition, first rank {int(ranks[bad[0]])} in {int(part[bad[0]])}"
    assert len(np.unique(ranks)) == len(ranks), "a key appears twice"
    return ranks, part


def _values(v, vlens):
    """A partition's values as u64: numbers as they are, byte strings ((offsets, bytes)) decoded to their ranks."""
    if isinstance(v, tuple):
        o, d = v
        _check_offsets(o, len(d), "value bytes")
        return decode(np.asarray(o).astype(np.int64) - int(o[0]), d, vlens)
    return G.u64(v)


def str_csr_triples(parts, R, lens=LENS, vlens=LENS, allow_empty=False, keys=None):
    """parts[r] = (key offsets, key bytes, value offsets, values) of partition r, values as numbers or as byte strings
    (value byte offsets, value bytes).  Checks both CSRs and each key's placement; returns (rank, position, value) per
    value, ordered by rank then position.  keys: str_keys_of(parts) when already known."""
    ranks, _ = keys if keys is not None else str_keys_of(parts, R, lens)
    cnts, vals = [], []
    for r, p in enumerate(parts):
        nk = len(p[0]) - 1
        v = _values(p[3], vlens)
        cnt = _check_offsets(p[2], len(v), f"partition {r} values", allow_empty)
        assert len(cnt) == nk, f"partition {r}: {len(cnt)} value lists for {nk} keys"
        cnts.append(cnt)
        vals.append(v)
    cnt = np.concatenate(cnts) if cnts else np.zeros(0, np.int64)
    v = np.concatenate(vals) if vals else np.zeros(0, np.uint64)
    return G._by_key_then_pos((np.repeat(ranks, cnt), G._positions(cnt), v))


def assert_str_group_equal(parts, ranks, vals, R, lens=LENS, vlens=LENS):
    """A String GROUP shuffle's partitions against group_by_key of (keys of ranks, vals): every key once, in its
    partition, its list element for element (vals: numbers, or the ranks of byte-string values)."""
    G.assert_rows_equal(str_csr_triples(parts, R, lens, vlens), G.group_triples(ranks, vals), G.GROUP_COLS)


def assert_str_cogroup_equal(parts, sides, R, lens=LENS):
    """parts[r] = (key offsets, key bytes, [(offsets, values) per side]); sides = [(ranks, vals) per side]: every key
    of any side once, in its partition, with every side's list; no key with only empty lists.  Returns (sorted ranks,
    their partitions) for str_join_rows."""
    keys = str_keys_of(parts, R, lens)
    want = np.unique(np.concatenate([G.u64(k) for k, _ in sides]))
    assert np.array_equal(np.sort(keys[0]), want), f"{len(keys[0])} keys, want {len(want)} (the union of the sides)"
    any_vals = np.zeros(len(keys[0]), bool)
    for j, (k, v) in enumerate(sides):
        side_parts = [(p[0], p[1], p[2][j][0], p[2][j][1]) for p in parts]
        any_vals |= np.concatenate([np.diff(np.asarray(p[2]).astype(np.int64)) > 0 for p in side_parts])
        G.assert_rows_equal(str_csr_triples(side_parts, R, lens, allow_empty=True, keys=keys), G.group_triples(k, v),
                            G.GROUP_COLS)
    assert any_vals.all(), "a key with only empty lists"
    o = np.argsort(keys[0])
    return keys[0][o], keys[1][o]


def str_join_rows(parts, R, lens=LENS, placed=None):
    """parts[r] = (key offsets, key bytes, row offsets, (v, w), (v valid, w valid)) of a two-side join partition.
    Checks the CSRs (every listed key has rows) and each key's placement (placed: as for str_keys_of); returns the
    rows as group_ref.join_rows does, with ranks as keys."""
    ranks, _ = str_keys_of(parts, R, lens, placed)
    cnts, cols = [], [[] for _ in range(4)]
    for r, (ko, _, ro, vs, oks) in enumerate(parts):
        cnt = _check_offsets(ro, len(vs[0]), f"partition {r} rows", allow_empty=False)
        assert len(cnt) == len(ko) - 1
        cnts.append(cnt)
        for c, x in zip(cols, (G.u64(vs[0]), G.u64(vs[1]), np.asarray(oks[0], np.uint8), np.asarray(oks[1], np.uint8))):
            c.append(x)
    cnt = np.concatenate(cnts)
    out = [np.repeat(ranks, cnt), G._positions(cnt)] + [np.concatenate(c) for c in cols]
    return G._by_key_then_pos(out)
