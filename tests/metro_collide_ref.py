"""Byte-string keys that share their full 64-bit MetroHash64_1 (test infrastructure), and a model of the String-key
dictionary's encode loop.

A String key hashes as key ‖ 0xFF, a Vec<u8> key as le64(len) ‖ key (vega_b200/csrc/strkeys.cuh), with MetroHash64_1
at seed 0, which HashPartitioner needs, so the hash cannot be seeded.  Its 32-byte block loop can be solved word by
word: with (a0, a1, a2, a3) the lanes before a block, the block

    w0 = (rotl(t0 - a2, 29) - a0) * inv(k0)     w1 = (rotl(t1 - a3, 29) - a1) * inv(k1)
    w2 = (rotl(t2 - t0, 29) - a2) * inv(k2)     w3 = (rotl(t3 - t1, 29) - a3) * inv(k3)      (mod 2^64)

takes them to any state T = (t0, t1, t2, t3) (the multipliers are odd, so they invert).  Keys of one length whose
last block is solved for one T, and that share the bytes after it, share the whole hash whatever their earlier blocks
hold.  Layouts (the solved block always lies inside the key):
    Vec<u8>, 56 bytes   stream le64(56) ‖ key: 64 bytes, 24 free key bytes, no tail;
    Vec<u8>, 64 / 96    stream of 72 / 104 bytes: 24 / 56 free key bytes, an 8-byte tail key[L-8 .. L);
    String, 71 bytes    stream key ‖ 0xFF: 72 bytes, 32 free key bytes, tail key[64 .. 71) ‖ 0xFF.
Every hash here comes from the numpy restatements (str_group_ref.metro64_1_str, bytes_keys_ref.metro64_1_bytes);
this module only steps and solves the block loop.

Families (deterministic from a seed; none of the keys is valid UTF-8 except by chance, so tests compare bytes):
  same_hash         n distinct keys with one hash; their free bytes are random;
  same_hash_lengths Vec<u8> keys of 64 and 96 bytes with one hash: the 96-byte tail word is the 64-byte one plus
                    (72 - 104) * inv(k3), so the sums after the tail agree (String has no such pair: LENGTH_PAIRS);
  wrap              one hash whose top 24 bits are all ones (WRAP_T, found by search_wrap): home is the last bucket of
                    every index of 2^4 .. 2^26 slots, and the chain wraps to bucket 0;
  pairs             n_pairs 2-key collisions with n_pairs different hashes;
  absent            more keys with a family's hash, none of them in the family.

encode_model restates str_encode (engine.cu) by bucket: the parent's abort-and-grow loop, and the fixed one."""
import numpy as np

from tests import bytes_keys_ref as B
from tests import str_group_ref as S

STR, BYTES = "str", "bytes"
MASK = S.MASK64
K = (S._K0, S._K1, S._K2, S._K3)
KINV = tuple(pow(k, -1, 1 << 64) for k in K)
STR_MAX_PROBE = 64               # buckets (strkeys.cuh)
STR_MAX_LOG_CAP = 33             # index slots (engine.cu)
BUCKET = 4
SLOT_BYTES = 12                  # index bytes per slot: u64 fingerprint + u32 entry id
DEFAULT_LEN = {STR: 71, BYTES: 56}
STR_TAIL = b"collide"            # key[64 .. 71) of the String families
# WRAP_T[kind]: a state whose hash (DEFAULT_LEN, STR_TAIL) has its top 24 bits all ones: search_wrap(kind, 24, seed=1)
WRAP_T = {
    STR: (0xD2AF1DBF3FC1F7D6, 0x3B192B0B3C0878AB, 0x8148387BDA4DE294, 0x9B169F5E7EE75E7E),
    BYTES: (0x6D7C8485F23AD072, 0x2BC52D76511FEB38, 0x64541F188530A052, 0xCF1F65C8327376DD),
}
WRAP_BITS = 24

_U = np.uint64


def _rotr(v, k):
    return (v >> _U(k)) | (v << _U(64 - k))


def _rotl(v, k):
    return (v << _U(k)) | (v >> _U(64 - k))


def block(lanes, w):
    """One round of the 32-byte block loop: lanes (4 u64 arrays) after the words w (4 u64 arrays)."""
    v0, v1, v2, v3 = (np.array(x, np.uint64) for x in lanes)
    with np.errstate(over="ignore"):
        v0 = _rotr(v0 + w[0] * _U(K[0]), 29) + v2
        v1 = _rotr(v1 + w[1] * _U(K[1]), 29) + v3
        v2 = _rotr(v2 + w[2] * _U(K[2]), 29) + v0
        v3 = _rotr(v3 + w[3] * _U(K[3]), 29) + v1
    return v0, v1, v2, v3


def solve(lanes, T):
    """The words of the block that takes lanes (a0..a3) to T (t0..t3): block(lanes, solve(lanes, T)) == T."""
    a0, a1, a2, a3 = (np.array(x, np.uint64) for x in lanes)
    t0, t1, t2, t3 = (np.array(x, np.uint64) for x in T)
    with np.errstate(over="ignore"):
        return ((_rotl(t0 - a2, 29) - a0) * _U(KINV[0]), (_rotl(t1 - a3, 29) - a1) * _U(KINV[1]),
                (_rotl(t2 - t0, 29) - a2) * _U(KINV[2]), (_rotl(t3 - t1, 29) - a3) * _U(KINV[3]))


def stream_len(kind, L):
    return L + (1 if kind == STR else 8)


def layout(kind, L):
    """(free key bytes before the solved block, tail key bytes after it) of keys of L bytes."""
    n = stream_len(kind, L)
    blocks = n // 32
    assert blocks >= 2, "the solved block needs a block before it"
    lead = 8 if kind == BYTES else 0                       # stream bytes before the key
    free = (blocks - 1) * 32 - lead
    tail = L - free - 32
    assert free >= 0 and tail >= 0 and (kind == BYTES or tail + 1 == n - blocks * 32), (kind, L)
    return free, tail


def lanes_after(kind, L, prefix):
    """Lanes after the blocks before the solved one, for every row of the (m, free) byte matrix prefix."""
    m = prefix.shape[0]
    n = stream_len(kind, L)
    st = np.zeros((m, prefix.shape[1] + (8 if kind == BYTES else 0)), np.uint8)
    if kind == BYTES:
        st[:, :8] = np.frombuffer(np.uint64(L).tobytes(), np.uint8)
        st[:, 8:] = prefix
    else:
        st[:] = prefix
    words = np.ascontiguousarray(st).view("<u8")
    with np.errstate(over="ignore"):
        h = np.full(m, (K[2] * K[0] + n) & MASK, np.uint64)
    v = (h, h, h, h)
    for b in range(words.shape[1] // 4):
        v = block(v, tuple(words[:, 4 * b + j] for j in range(4)))
    return v


def build(kind, L, prefix, T, tail):
    """(m, L) key matrix: prefix ‖ the block solved for T (one state, or one per row) ‖ tail."""
    w = solve(lanes_after(kind, L, prefix), T)
    mid = np.stack([np.broadcast_to(x, (prefix.shape[0],)) for x in w], axis=1).astype("<u8").view(np.uint8)
    t = np.broadcast_to(np.frombuffer(tail, np.uint8), (prefix.shape[0], len(tail)))
    return np.concatenate([prefix, mid, t], axis=1)


def hashes(kind, keys):
    """MetroHash64_1 of every bytes key under the kind's Hash, from the numpy restatements."""
    o, d = B.encode(list(keys))
    return (S.metro64_1_str if kind == STR else B.metro64_1_bytes)(o, d)


def _rows(M):
    return [bytes(r) for r in M]


def _random_T(rng, m=None):
    return tuple(rng.integers(0, 1 << 64, m, dtype=np.uint64) for _ in range(4))


def _tail(kind, L, rng):
    free, tail = layout(kind, L)
    if kind == STR and L == DEFAULT_LEN[STR]:
        return STR_TAIL
    return bytes(rng.integers(0, 256, tail, dtype=np.uint8))


def _distinct_prefixes(rng, n, free, exclude):
    """n distinct random prefixes of `free` bytes, none the prefix of a key in exclude."""
    ex = {k[:free] for k in exclude}
    out, seen = [], set()
    while len(out) < n:
        for r in _rows(rng.integers(0, 256, (2 * (n - len(out)) + 4, free), dtype=np.uint8)):
            if r not in ex and r not in seen:
                seen.add(r)
                out.append(r)
                if len(out) == n:
                    break
    return np.frombuffer(b"".join(out), np.uint8).reshape(n, free)


class Family:
    """Keys crafted to share one hash: kind, key length, state T and tail bytes, and the keys."""

    def __init__(self, kind, L, T, tail, keys):
        self.kind, self.L, self.T, self.tail, self.keys = kind, L, tuple(int(t) for t in T), tail, keys
        self.hash = int(hashes(kind, keys[:1])[0])

    def __len__(self):
        return len(self.keys)


def same_hash(kind, n, T=None, seed=0, L=None, tail=None, exclude=()):
    """n distinct keys of L bytes (DEFAULT_LEN) with one hash: random free bytes, the block solved for T (random from
    the seed if None), and one tail (random from the seed, STR_TAIL for the String default)."""
    rng = np.random.default_rng(seed)
    L = L or DEFAULT_LEN[kind]
    T = T if T is not None else tuple(int(t) for t in _random_T(rng))
    tail = tail if tail is not None else _tail(kind, L, rng)
    free, _ = layout(kind, L)
    keys = _rows(build(kind, L, _distinct_prefixes(rng, n, free, exclude), T, tail))
    return Family(kind, L, T, tail, keys)


def absent(fam, m, seed=1):
    """m keys with fam's hash (same length, state and tail), none of them in fam."""
    return same_hash(fam.kind, m, fam.T, seed=seed + 7919, L=fam.L, tail=fam.tail, exclude=fam.keys).keys


def tail_shift(n_from, n_to):
    """What the tail word of a key whose stream is n_from bytes long gains so that one of n_to bytes, from the same
    state after its blocks, reaches the same sum after the tail: h = k2 k0 + n + mix(T) + w k3."""
    return ((n_from - n_to) * KINV[3]) & MASK


# String keys of lengths L and L' (both 8-byte tails: L ≡ 7 mod 32) would share a hash if the shifted tail word kept
# its top byte 0xFF for some low bytes: tail_shift's top byte must be 0x00 or 0xFF.  None of these pairs has that.
LENGTH_PAIRS = tuple((71, 71 + 32 * j) for j in range(1, 9))


def str_length_pair():
    """The first of LENGTH_PAIRS whose tail correction leaves the 0xFF byte alone, or None."""
    for L1, L2 in LENGTH_PAIRS:
        if (tail_shift(L1 + 1, L2 + 1) >> 56) in (0x00, 0xFF):
            return L1, L2
    return None


def same_hash_lengths(n, seed=0):
    """Vec<u8> keys, n of 64 bytes and n of 96 bytes, all with one hash."""
    rng = np.random.default_rng(seed)
    T = tuple(int(t) for t in _random_T(rng))
    w = int(rng.integers(0, 1 << 64, dtype=np.uint64))
    w2 = (w + tail_shift(stream_len(BYTES, 64), stream_len(BYTES, 96))) & MASK
    a = same_hash(BYTES, n, T, seed=seed + 1, L=64, tail=w.to_bytes(8, "little"))
    b = same_hash(BYTES, n, T, seed=seed + 2, L=96, tail=w2.to_bytes(8, "little"))
    return Family(BYTES, None, T, None, a.keys + b.keys)


def wrap(kind, n, seed=0):
    """n keys of one hash whose top WRAP_BITS bits are all ones."""
    return same_hash(kind, n, WRAP_T[kind], seed=seed)


def pairs(kind, n_pairs, seed=0):
    """2 n_pairs keys: pair i (keys 2i, 2i + 1) shares a hash, and the n_pairs hashes differ."""
    rng = np.random.default_rng(seed)
    L = DEFAULT_LEN[kind]
    free, _ = layout(kind, L)
    T = _random_T(rng, n_pairs)
    T2 = tuple(np.repeat(t, 2) for t in T)
    return _rows(build(kind, L, _distinct_prefixes(rng, 2 * n_pairs, free, ()), T2, _tail(kind, L, rng)))


def search_wrap(kind, bits, seed=1, chunk=1 << 18, max_tries=1 << 28):
    """A state T (first found, deterministic from the seed) whose keys of DEFAULT_LEN (with the family tail) hash to a
    value with its top `bits` bits all ones.  The candidates are hashed as keys by the numpy restatements, chunk by
    chunk: one fixed prefix, the block solved for each candidate T."""
    rng = np.random.default_rng(seed)
    L = DEFAULT_LEN[kind]
    free, _ = layout(kind, L)
    prefix = rng.integers(0, 256, (1, free), dtype=np.uint8)
    tail = _tail(kind, L, np.random.default_rng(seed + 1))
    want = _U((1 << bits) - 1)
    for _ in range(0, max_tries, chunk):
        T = _random_T(rng, chunk)
        M = build(kind, L, np.broadcast_to(prefix, (chunk, free)), T, tail)
        o = np.arange(0, (chunk + 1) * L, L, dtype=np.uint64)
        h = (S.metro64_1_str if kind == STR else B.metro64_1_bytes)(o, M.reshape(-1))
        hit = np.flatnonzero((h >> _U(64 - bits)) == want)
        if len(hit):
            return tuple(int(t[hit[0]]) for t in T)
    return None


def home(h, log_cap):
    """strkeys.cuh:str_bucket: the index bucket a hash starts its probe at."""
    return (int(h) >> (66 - log_cap)) if log_cap > 2 else 0


# ---- str_encode, by bucket ---------------------------------------------------------------------------------------
def ceil_log2(x):
    return max(0, (int(x) - 1).bit_length())


def choose_log_cap(guess, hint):
    """engine.cu:choose_log_cap for a String index (never estimated)."""
    target = (hint * 5) // 2 if hint else min(2 * max(guess, 1), 1 << 21)
    if hint and target > (1 << 22):
        target = 2 * hint
    return min(STR_MAX_LOG_CAP, max(4, ceil_log2(target)))


class Index:
    """The dictionary by bucket: every entry's hash (entry order) and the bucket it sits in."""

    def __init__(self, log_cap):
        self.log_cap, self.fill, self.at, self.entries = log_cap, {}, {}, []

    def nb(self):
        return 1 << (self.log_cap - 2)

    def put(self, key, b):
        self.fill[b] = self.fill.get(b, 0) + 1
        self.at[key] = b

    def rebuilt(self, log_cap):
        """str_index_build: every entry re-inserted, in entry order, with no probe limit."""
        x = Index(log_cap)
        x.entries = list(self.entries)
        for key, h in x.entries:
            b = home(h, log_cap)
            while x.fill.get(b, 0) == BUCKET:
                b = (b + 1) % x.nb()
            x.put(key, b)
        return x


def encode_run(ix, keys, hs, max_entries, max_probe):
    """One str_encode_kernel launch over distinct keys (ids) with hashes hs, one row each, in order: None, or the
    reason it aborts ("load": n_entries reached max_entries at an empty slot, "chain": max_probe full buckets)."""
    nb = ix.nb()
    for key, h in zip(keys, hs):
        b = home(h, ix.log_cap)
        for _ in range(max_probe):
            if ix.at.get(key) == b:
                break
            if ix.fill.get(b, 0) < BUCKET:
                if len(ix.entries) >= max_entries:
                    return "load"
                ix.put(key, b)
                ix.entries.append((key, int(h)))
                break
            b = (b + 1) % nb
        else:
            return "chain"
    return None


def encode_model(hs, n_rows, hint=0, guess=None, fixed=True, ix=None, ids=None, mem_bytes=80 << 30):
    """str_encode over one call of n_rows rows whose distinct keys have the hashes hs, in row order.  ids: the keys'
    identities (default 0, 1, ...; equal ids are one key).  fixed: the growth rule of this build; else the parent's
    (grow 4x on every abort).  ix: the dictionary before the call (None: a new one sized from guess and hint).
    Returns (ix or None, {"ladder": index log_caps the call ran on, "restarts", "lifted", "error"}); error is
    "VB_ERR_OOM" when the next index (12 bytes a slot, beside the old one) does not fit mem_bytes, "VB_ERR_TOO_LARGE"
    past 2^STR_MAX_LOG_CAP slots."""
    hs = [int(h) for h in hs]
    keys = list(range(len(hs))) if ids is None else list(ids)
    if ix is None:
        ix = Index(choose_log_cap(guess if guess is not None else n_rows, hint))
    worst = len(ix.entries) + n_rows
    lifted = fixed and (1 << ix.log_cap) >= 2 * worst
    out = {"ladder": [], "restarts": 0, "lifted": False, "error": None}
    while True:
        cap, nb = 1 << ix.log_cap, ix.nb()
        max_entries = min((cap // 10) * 6, (1 << 32) - 1)
        out["ladder"].append(ix.log_cap)
        out["lifted"] = lifted
        why = encode_run(ix, keys, hs, max_entries, nb if lifted or nb < STR_MAX_PROBE else STR_MAX_PROBE)
        if why is None:
            return ix, out
        out["restarts"] += 1
        chain = len(ix.entries) < max_entries
        grow = True
        if fixed and chain:
            lifted = True
            grow = cap < 2 * worst
        if grow:
            lc = max(ix.log_cap + 2, ceil_log2(3 * len(ix.entries)))
            if lc > STR_MAX_LOG_CAP:
                out["error"] = "VB_ERR_TOO_LARGE"
                return None, out
            if SLOT_BYTES * ((1 << lc) + cap) > mem_bytes:
                out["error"] = "VB_ERR_OOM"
                return None, out
            ix = ix.rebuilt(lc)
