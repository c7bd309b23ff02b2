"""The integer hash table's slot hash, its inverse, and keys built to land where a test wants them (test infrastructure).

Every integer-key table (reduce, combine, the group and join dictionaries, narrow views) places key k in home bucket
slot_hash(k) >> (64 - (log_cap - 2)) of a table of 2^log_cap slots in 4-key buckets, probes linearly (wrapping from
the last bucket to bucket 0) and gives up after HA_MAX_PROBE buckets unless the table is at its final size
(vega_b200/csrc/kernels.cuh).  slot_hash (common.cuh) is two xor-shifts by 32, each its own inverse, and two odd
multipliers, so it is a bijection of the u64s: slot_hash_inv turns any wanted slot hash into the key that has it.

Families (keys 0 and 2^64-1 excluded: 0 has slot hash 0, home bucket 0, the first bucket a wrapped chain reaches, and
2^64-1 is the table's empty marker; the tests add both to every input themselves):
  same_home     slot hashes share their top 33 bits: one home bucket at every log_cap from 4 to 35;
  wrap          slot-hash top 33 bits all ones: the last bucket is home at every size, chains wrap to bucket 0;
  region_edge   home is the last bucket of a region of the partition-first path at one log_cap;
  cache_clash   slot hashes share their low 20 bits: both hot-key-cache choices (h & 1023, (h >> 10) & 1023, and the
                512-slot cache of combine_by_key) are the same for every key of the family;
  i32_same_home 4-byte keys sharing a home bucket at one log_cap, found by search (2^32 keys cannot reach every size).
Absent neighbours are more same_home keys with the input's keys excluded."""
import os
import re

import numpy as np

MASK = (1 << 64) - 1
EMPTY_KEY = MASK
M1, M2 = 0xD6E8FEB86659FD93, 0x9E3779B97F4A7C15
M1_INV, M2_INV = pow(M1, -1, 1 << 64), pow(M2, -1, 1 << 64)
HA_MAX_PROBE = 256            # buckets (kernels.cuh)
BUCKET = 4
TOP = 33                      # same_home / wrap: bits shared, enough for a home bucket at log_cap <= TOP + 2
ENGINE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vega_b200", "csrc", "engine.cu")

_U32 = np.uint64(32)


def slot_hash(keys):
    """common.cuh:slot_hash over a u64 array."""
    x = np.array(keys, dtype=np.uint64, copy=True)
    with np.errstate(over="ignore"):
        x ^= x >> _U32
        x *= np.uint64(M1)
        x ^= x >> _U32
        x *= np.uint64(M2)
    return x


def slot_hash_inv(h):
    """The keys whose slot hashes are h."""
    x = np.array(h, dtype=np.uint64, copy=True)
    with np.errstate(over="ignore"):
        x *= np.uint64(M2_INV)
        x ^= x >> _U32
        x *= np.uint64(M1_INV)
        x ^= x >> _U32
    return x


def home_bucket(keys, log_cap):
    return slot_hash(keys) >> np.uint64(64 - (log_cap - 2))


def _from_hashes(rng, n, fixed, fixed_mask, exclude=()):
    """n distinct keys, none in exclude, 0 or 2^64-1, whose slot hashes h have h & fixed_mask == fixed; the other
    bits are random."""
    ex = {0, EMPTY_KEY} | {int(k) for k in np.asarray(exclude, dtype=np.uint64).tolist()}
    out, seen = [], set()
    while len(out) < n:
        free = rng.integers(0, 1 << 64, 2 * (n - len(out)) + 8, dtype=np.uint64)
        h = (free & np.uint64(MASK ^ fixed_mask)) | np.uint64(fixed)
        for k in slot_hash_inv(h).tolist():
            if k not in ex and k not in seen:
                seen.add(k)
                out.append(k)
                if len(out) == n:
                    break
    return np.array(out, dtype=np.uint64)


def same_home(rng, n, top, exclude=()):
    """n keys whose slot hashes have the top 33 bits `top` (0 <= top < 2^33)."""
    return _from_hashes(rng, n, top << (64 - TOP), MASK ^ ((1 << (64 - TOP)) - 1), exclude)


def wrap(rng, n, exclude=()):
    """n keys homed in the last bucket at every log_cap from 4 to 35."""
    return same_home(rng, n, (1 << TOP) - 1, exclude)


def region_bits(log_cap):
    """Top slot-hash bits that split the input into table regions on the partition-first path at log_cap, read
    from launch_hash_agg_partitioned (engine.cu) so that the test follows the engine."""
    src = open(ENGINE).read()
    m = re.search(r"launch_hash_agg_partitioned\([^)]*\)\s*\{.*?pbits = std::min<u32>\((\d+), log_cap - (\d+)\)", src, re.S)
    assert m, "launch_hash_agg_partitioned no longer computes pbits as std::min<u32>(A, log_cap - B)"
    return min(int(m.group(1)), log_cap - int(m.group(2)))


def region_edge(rng, n_per_region, log_cap, exclude=()):
    """n_per_region keys homed in the last bucket of each region of the partition-first path at log_cap."""
    pbits, hb = region_bits(log_cap), log_cap - 2
    per = 1 << (hb - pbits)                                   # buckets per region
    out = []
    for r in range(1 << pbits):
        bucket = (r + 1) * per - 1
        out.append(_from_hashes(rng, n_per_region, bucket << (64 - hb), MASK ^ ((1 << (64 - hb)) - 1),
                                np.concatenate([np.asarray(exclude, np.uint64)] + out)))
    return np.concatenate(out)


def cache_clash(rng, n, low20, exclude=()):
    """n keys whose slot hashes end in the 20 bits low20: the same two hot-key-cache slots."""
    return _from_hashes(rng, n, low20, (1 << 20) - 1, exclude)


def i32_same_home(rng, n, log_cap, candidates=1 << 24):
    """n distinct i32 keys (not -1, which widens to the empty marker) that share one home bucket at log_cap, found
    among `candidates` random i32 values widened as the table widens them (sign extension)."""
    c = np.unique(rng.integers(-(1 << 31), 1 << 31, candidates, dtype=np.int64).astype(np.int32))
    c = c[c != -1]
    homes = home_bucket(c.astype(np.int64).view(np.uint64), log_cap)
    vals, counts = np.unique(homes, return_counts=True)
    best = vals[np.argmax(counts)]
    found = c[homes == best]
    assert len(found) >= n, (len(found), n)
    return found[:n]


def chain_model(keys, log_cap, limit=HA_MAX_PROBE):
    """The insert loop of the table: every distinct key (2^64-1 goes to the special slot) takes the first empty slot
    along its chain, inserted in the given order.  Returns (aborts, longest chain in buckets loaded): aborts when an
    insert finds no empty slot within `limit` buckets.  For keys that share one home bucket, and keys homed far
    from theirs, the result does not depend on the insertion order: the k-th key of a one-home family always lands
    k // 4 buckets past the home."""
    nb = 1 << (log_cap - 2)
    fill = np.zeros(nb, dtype=np.int64)
    longest = 0
    uk = list(dict.fromkeys(int(k) for k in np.asarray(keys, dtype=np.uint64).tolist()))
    uk = np.array([k for k in uk if k != EMPTY_KEY], dtype=np.uint64)
    for b in home_bucket(uk, log_cap).tolist():
        walked = 1
        while fill[b] == BUCKET:
            if walked == limit or walked == nb:
                return True, max(longest, walked)
            b = (b + 1) & (nb - 1)
            walked += 1
        fill[b] += 1
        longest = max(longest, walked)
    return False, longest
