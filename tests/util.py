"""Shared helpers for the parity tests (test infrastructure; may use oracle/)."""
import math

import numpy as np

from oracle import oracle as O
from tests import f64_sum_ref as F

MASK64 = (1 << 64) - 1
EMPTY_KEY = MASK64                       # the device table's empty marker: a real key with this value takes the special slot
CANON_NAN = 0x7FF8000000000000           # every NaN result is compared as this bit pattern (the payload is unspecified)
U64_SPECIAL = [0, 1, (1 << 63) - 1, 1 << 63, MASK64]
I64_SPECIAL = [-(1 << 63), (1 << 63) - 1, -1, 0]
NAN_BITS = [0x7FF8000000000000, 0x7FF8000000000001, 0x7FFC0000DEADBEEF, 0x7FFFFFFFFFFFFFFF,
            0xFFF8000000000000, 0xFFF80000000BEEF0, 0xFFFFFFFFFFFFFFFF]
F64_SPECIAL = [0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 2.5e-310, -1.1e-315, 2.2250738585072009e-308,
               -2.2250738585072014e-308, 1.7976931348623157e308, -1.7976931348623157e308]
VALUE_MODES = ("default", "full", "special", "exact", "subnormal", "cancel")


def oracle_reduce(op, keys, vals, M, R, vdtype="u64", key_width=8, threads=1):
    parts = O.shuffle(op, keys, vals, M, R, vdtype=vdtype, key_width=key_width, threads=threads)
    return [dict(zip(p["keys"].tolist(), p["combined"].tolist())) for p in parts]


def oracle_group(keys, vals, M, R, vdtype="u64", key_width=8):
    parts = O.shuffle("group", keys, vals, M, R, vdtype=vdtype, key_width=key_width)
    out = []
    for p in parts:
        o = p["offsets"]
        out.append({int(k): p["vals"][int(o[i]):int(o[i + 1])].tolist() for i, k in enumerate(p["keys"])})
    return out


def gpu_reduce_parts(rdd):
    """Per-partition {key: combined} of a vega_b200 ShuffledRdd (reduce ops)."""
    out = []
    for r in range(rdd.num_slices):
        k, c = rdd.compute(r)
        d = dict(zip(k.tolist(), c.tolist()))
        assert len(d) == len(k), "duplicate key inside one reduce partition"
        out.append(d)
    return out


def gpu_group_parts(rdd):
    out = []
    for r in range(rdd.num_slices):
        k, o, v = rdd.compute(r)
        assert o[0] == 0 and o[-1] == len(v)
        d = {int(kk): v[int(o[i]):int(o[i + 1])].tolist() for i, kk in enumerate(k)}
        assert len(d) == len(k), "duplicate key inside one reduce partition"
        out.append(d)
    return out


def bits_dict(keys, comb):
    """{key as u64: combined as u64 bits}, with every f64 NaN as CANON_NAN: exact comparison of any reduce result."""
    k = np.ascontiguousarray(keys)
    c = np.ascontiguousarray(comb)
    b = c.view(np.uint64).copy()
    if c.dtype == np.float64:
        b[np.isnan(c)] = np.uint64(CANON_NAN)
    d = dict(zip(k.view(np.uint64).tolist(), b.tolist()))
    assert len(d) == len(k), "duplicate key inside one reduce partition"
    return d


def oracle_reduce_bits(op, keys, vals, M, R, vdtype="u64", key_width=8, threads=1):
    parts = O.shuffle(op, keys, vals, M, R, vdtype=vdtype, key_width=key_width, threads=threads)
    return [bits_dict(p["keys"], p["combined"]) for p in parts]


def f64_total_key(x):
    """f64 → u64 with the order of Rust's f64::total_cmp (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN)."""
    b = np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)
    return np.where(b >> np.uint64(63), ~b, b | np.uint64(1 << 63))


def rand_pairs(rng, n, n_keys, vdtype="u64", wide_keys=True, values="default", hot=0.0):
    """n (key, value) rows over about n_keys keys; hot > 0 gives the first key that share of the rows (and the
    second key half of it).

    values="default" draws u64 below 2^40, i64 within +-2^40 and f64 N(0, 1) (sums never wrap).  The other modes
    cover the full value range, and their keys always include 0 and 2^64-1 (the table's empty marker):
      "full"       u64 / i64: uniform over all 64 bits plus the extreme values; per-key sums wrap.
      "special"    f64 for MIN/MAX: normals of both signs over a wide exponent range, +-0.0, +-inf, subnormals and
                   quiet NaNs of both signs with different payloads; some keys hold only NaNs, some only +-0.0.
      "exact"      f64: k * 2^-30 with integer |k| <= 2^20; every partial sum is exact, whatever the order.
      "subnormal"  f64: k * 2^-1074, |k| <= 2^20: every value and every sum is a subnormal, all exact.
      "cancel"     f64: rows come in pairs of one key, +-1e12 and -+1e12, each plus N(0, 1) noise.
    """
    assert values in VALUE_MODES, values
    ranks = rng.integers(0, max(n_keys, 1), n).astype(np.uint64)
    if hot:
        u = rng.random(n)
        ranks[u < 1.5 * hot] = np.uint64(1)
        ranks[u < hot] = np.uint64(0)
    keys = ranks * np.uint64(0x9E3779B97F4A7C15) + np.uint64(12345) if wide_keys else ranks
    if values == "default":
        if vdtype == "u64":
            vals = rng.integers(0, 1 << 40, n).astype(np.uint64)
        elif vdtype == "i64":
            vals = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
        else:
            vals = rng.standard_normal(n)
        return keys, vals
    if n >= 2:
        at = rng.choice(n, size=max(2, n // 4096), replace=False)
        keys[at[0::2]] = np.uint64(0)
        keys[at[1::2]] = np.uint64(EMPTY_KEY)
    sprinkle = rng.random(n) < 1 / 16
    if values == "full":
        assert vdtype in ("u64", "i64"), vdtype
        if vdtype == "u64":
            vals = rng.integers(0, 1 << 64, n, dtype=np.uint64)
            vals[sprinkle] = rng.choice(np.array(U64_SPECIAL, dtype=np.uint64), int(sprinkle.sum()))
        else:
            vals = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
            vals[sprinkle] = rng.choice(np.array(I64_SPECIAL, dtype=np.int64), int(sprinkle.sum()))
        return keys, vals
    assert vdtype == "f64", (values, vdtype)
    if values == "special":
        mag = rng.uniform(1.0, 2.0, n) * np.exp2(rng.integers(-1000, 1000, n).astype(np.float64))
        vals = np.where(rng.random(n) < 0.5, -mag, mag)
        bits = vals.view(np.uint64)
        pool = np.concatenate([np.array(F64_SPECIAL).view(np.uint64), np.array(NAN_BITS, dtype=np.uint64)])
        bits[sprinkle] = rng.choice(pool, int(sprinkle.sum()))
        all_nan = (ranks % np.uint64(101)) == np.uint64(7)
        bits[all_nan] = rng.choice(np.array(NAN_BITS, dtype=np.uint64), int(all_nan.sum()))
        only_zero = (ranks % np.uint64(103)) == np.uint64(5)
        bits[only_zero] = rng.choice(np.array([0.0, -0.0]).view(np.uint64), int(only_zero.sum()))
        return keys, vals
    if values in ("exact", "subnormal"):
        ints = rng.integers(-(1 << 20), (1 << 20), n, endpoint=True).astype(np.float64)
        return keys, np.ldexp(ints, -30 if values == "exact" else -1074)
    # "cancel"
    big = np.where(rng.random(n) < 0.5, 1e12, -1e12)
    vals = rng.standard_normal(n)
    half = n // 2
    keys[1:2 * half:2] = keys[0:2 * half:2]
    vals[0:2 * half:2] += big[:half]
    vals[1:2 * half:2] -= big[:half]
    return keys, vals


def assert_parts_equal(got, want):
    """Per-partition dicts equal, with a short report of what differs instead of a diff of every key."""
    assert len(got) == len(want), (len(got), len(want))
    bad = []
    for r, (g, w) in enumerate(zip(got, want)):
        if g != w:
            wrong = [k for k in g.keys() & w.keys() if g[k] != w[k]]
            bad.append((r, len(w.keys() - g.keys()), len(g.keys() - w.keys()), len(wrong),
                        [(hex(k), g[k], w[k]) for k in wrong[:3]]))
    assert not bad, (f"{len(bad)} of {len(want)} partitions differ; (partition, keys missing, keys extra, values wrong, "
                     f"first wrong (key, got, want)): {bad[:4]}")


def assert_f64_sums(got_parts, keys, vals, R, key_width=8, exact=False, lenient=None):
    """Check an f64 SUM result against tests/f64_sum_ref.py, the results some summation order can give, for every key.

    got_parts: one {key: sum} dict per reduce partition.  For each key of the input:
      * it is in partition hash(key) % R, and only there;
      * its sum is one the reference admits: NaN for a NaN or both infinities, the infinity present otherwise, the
        exact sum bit for bit (the sign of a zero included) when every partial sum is representable, and within
        gamma(m-1) * sum|x| of the exact sum otherwise.  Every summation order meets these (atomics in any order,
        hot-key partial sums, per-map partial sums merged at seal, other ranks' partial sums);
      * exact=True: the reference must pin every key to one value (the case's values have representable partial sums);
      * lenient: the keys allowed more than one outcome class (those whose partial sums can overflow); None: any key.
    """
    keys = np.ascontiguousarray(keys).view(np.uint64)
    assert len(got_parts) == R
    got = {}
    for r, d in enumerate(got_parts):
        for k, v in d.items():
            k = int(k) & MASK64
            assert k not in got, f"key {k:#x} in two partitions"
            assert O.get_partition(k, R, key_width) == r, f"key {k:#x} in partition {r}"
            got[k] = float(v)
    F.assert_outcomes(got, F.key_outcomes(keys, vals), exact=exact, lenient=lenient)
