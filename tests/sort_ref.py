"""Exact checks of sort_by_key results (test infrastructure), shared by the sort tests.

A sort shuffle's output is fully determined: the rows of the map tasks, concatenated in map-id order, stably sorted
by key in the key dtype's order (u64 unsigned, i64 signed, f64 f64::total_cmp), and cut into R partitions where
partition p starts at floor(p * n / R) moved forward past every key bit-equal to the key before it (a range
partitioner never splits a key).  Two ways to check it:
  * assert_sort_equal: against the C oracle (O.sort_by_key), bit for bit, partition by partition;
  * check_sorted_exact: without a reference sort, for inputs whose value column is the row index (0 .. n-1 in
    map-id order).  Keys never decrease, the values are a permutation of 0 .. n-1, every output key is the input
    key of its value's row, values increase within a run of equal keys, and the partition sizes follow the cut
    rule: together these admit exactly one output.  Runs on numpy arrays or torch tensors (CPU or CUDA), chunked,
    in O(n) memory.
Keys travel as their 64-bit patterns (int64 arrays / tensors); order_key maps them to int64 whose signed order is
the dtype's order, so one searchsorted / comparison serves every dtype.
tests/test_sort_ref_cpu.py pins every function here to the oracle.
"""
import numpy as np

from oracle import oracle as O
from tests.util import F64_SPECIAL, NAN_BITS, rand_pairs

INT64_MIN = -(1 << 63)
INT64_MAX = (1 << 63) - 1
MASK64 = (1 << 64) - 1
PHI = 0x9E3779B97F4A7C15                    # odd: i -> i * PHI is a bijection of Z / 2^64
PHI_INV = pow(PHI, -1, 1 << 64)
EDGE = {"u64": [0, 1, INT64_MAX, INT64_MIN, -1],          # as int64 patterns: 0, 1, 2^63-1, 2^63, 2^64-1
        "i64": [INT64_MIN, INT64_MAX, -1, 0, 1],
        "f64": np.concatenate([np.array(F64_SPECIAL).view(np.int64), np.array(NAN_BITS, np.uint64).view(np.int64)]).tolist()}


def _is_torch(x):
    return hasattr(x, "is_cuda")


def signed(x):
    """A 64-bit pattern (Python int) as the int64 of the same bits."""
    x &= MASK64
    return x - (1 << 64) if x >> 63 else x


def bits(a):
    """The 64-bit patterns of a numpy key array as int64; 4-byte integers widened as _Col widens them."""
    a = np.ascontiguousarray(a)
    if a.dtype.itemsize == 8:
        return a.view(np.int64)
    return a.astype(np.int64 if a.dtype.kind == "i" else np.uint64).view(np.int64)


def order_key(b, kdtype):
    """int64 key patterns (numpy or torch) -> int64 whose signed order is the order of the key dtype.
    u64: the sign bit flipped; i64: unchanged; f64: negative patterns get their low 63 bits flipped, which is
    f64::total_cmp (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN).  A bijection: equal order keys are
    bit-equal keys."""
    if kdtype == "u64":
        return b ^ INT64_MIN
    if kdtype == "i64":
        return b + 0                                    # a copy, like the others
    assert kdtype == "f64", kdtype
    return b ^ ((b >> 63) & INT64_MAX)


def _searchsorted_right(a, v):
    if _is_torch(a):
        import torch
        return torch.searchsorted(a, v, right=True)
    return np.searchsorted(a, v, side="right")


def cut_rule(sorted_okeys, R):
    """part_starts (R + 1 int64) of n sorted order keys: start p = floor(p * n / R), moved to the end of the run of
    the key just before it.  Numpy array in, numpy out; torch tensor in, torch tensor out."""
    n = len(sorted_okeys)
    c = np.array([p * n // R for p in range(R + 1)], dtype=np.int64)
    inner = np.flatnonzero((c > 0) & (c < n))
    if len(inner):
        idx = c[inner] - 1
        if _is_torch(sorted_okeys):
            import torch
            idx = torch.from_numpy(idx).to(sorted_okeys.device)
        c[inner] = np.asarray(_searchsorted_right(sorted_okeys, sorted_okeys[idx]).tolist(), dtype=np.int64)
    if _is_torch(sorted_okeys):
        import torch
        return torch.from_numpy(c)
    return c


def run_keys(rng, n, kdtype, D, hot=0.1):
    """n key patterns (int64) over a pool of D keys of the dtype: its edge values (every f64 special: +-0.0, +-inf,
    subnormals, NaNs of both signs with several payloads) and random keys over the full range.  Every pool key
    occurs when n >= D; about `hot` of the rows share one key, so runs of equal keys are long."""
    edge = EDGE[kdtype]
    assert D >= len(edge), (D, len(edge))
    if kdtype == "f64":
        rest = rand_pairs(rng, D, 1, "f64", values="special")[1].view(np.int64)
    else:
        rest = rng.integers(INT64_MIN, INT64_MAX, D, dtype=np.int64, endpoint=True)
    pool = np.concatenate([np.array(edge, np.int64), rest])[:D]
    m = min(n, D)
    extra = rng.integers(0, D, n - m)
    extra[rng.random(n - m) < hot] = min(len(edge), D - 1)          # the first random key
    return pool[rng.permutation(np.concatenate([np.arange(m), extra]))]


# ---- against the oracle ---------------------------------------------------------------------------------------------
def _first_diff(got, want):
    n = min(len(got), len(want))
    d = np.flatnonzero(got[:n] != want[:n])
    return int(d[0]) if len(d) else n


def assert_sort_equal(parts, keys, vals, R, kdtype):
    """parts[r] = (keys, values or None) of reduce partition r.  keys / vals: the input in map-id order (vals None:
    a key-only sort).  Every partition equals the oracle's, bit for bit: its size, its keys, its values; and the
    oracle's cuts follow cut_rule."""
    assert len(parts) == R, (len(parts), R)
    ok, ov, ps = O.sort_by_key(bits(keys), None if vals is None else bits(vals), R, kdtype)
    ps = ps.astype(np.int64)
    assert np.array_equal(ps, cut_rule(order_key(bits(ok), kdtype), R)), "the oracle's cuts break the cut rule"
    sizes = [len(p[0]) for p in parts]
    want_sizes = np.diff(ps).tolist()
    assert sizes == want_sizes, f"partition sizes {_short(sizes)}, want {_short(want_sizes)}"
    gk = bits(np.concatenate([np.asarray(p[0]) for p in parts])) if R else np.zeros(0, np.int64)
    wk = bits(ok)
    if not np.array_equal(gk, wk):
        i = _first_diff(gk, wk)
        raise AssertionError(f"keys differ at row {i} (partition {int(np.searchsorted(ps, i, side='right')) - 1}): "
                             f"got {int(gk[i]) & MASK64:#x}, want {int(wk[i]) & MASK64:#x}")
    if vals is None:
        assert all(p[1] is None for p in parts)
        return
    gv = bits(np.concatenate([np.asarray(p[1]) for p in parts]))
    wv = bits(ov)
    if not np.array_equal(gv, wv):
        i = _first_diff(gv, wv)
        raise AssertionError(f"values differ at row {i} (key {int(wk[i]) & MASK64:#x}): got {int(gv[i])}, want {int(wv[i])}")


def _short(xs):
    return xs if len(xs) <= 16 else f"{xs[:8]} ... {xs[-4:]} ({len(xs)} partitions)"


# ---- without a reference sort ---------------------------------------------------------------------------------------
def _all(x):
    return bool(x.all())


def _first(mask, base):
    if _is_torch(mask):
        import torch
        return base + int(torch.nonzero(mask)[0, 0])
    return base + int(np.flatnonzero(mask)[0])


def check_sorted_exact(in_keys, out_keys, out_vals, sizes, kdtype, chunk=1 << 26):
    """in_keys: int64 key patterns of the input in map-id order, whose value column was the row index; out_keys,
    out_vals: int64 patterns of every partition's output, concatenated; sizes: rows per partition.  numpy arrays or
    torch tensors on one device.  Raises AssertionError on the first property that fails."""
    n = len(in_keys)
    assert len(out_keys) == n and len(out_vals) == n, (len(out_keys), len(out_vals), n)
    assert sum(sizes) == n, (sum(sizes), n)
    th = _is_torch(out_keys)
    if th:
        import torch
        seen = torch.zeros(n, dtype=torch.bool, device=out_keys.device)
    else:
        seen = np.zeros(n, dtype=bool)
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        lo = max(a - 1, 0)                               # one row of overlap: pairs across chunk boundaries
        k, v = out_keys[lo:b], out_vals[lo:b]
        okc = order_key(k, kdtype)
        bad = okc[1:] < okc[:-1]
        assert not bad.any(), f"keys decrease at row {_first(bad, lo + 1)}"
        bad = (k[1:] == k[:-1]) & (v[1:] <= v[:-1])
        assert not bad.any(), f"equal keys out of input order (unstable) at row {_first(bad, lo + 1)}"
        vv = out_vals[a:b]
        bad = (vv < 0) | (vv >= n)
        assert not bad.any(), f"value out of 0..n-1 at row {_first(bad, a)}"
        seen[vv] = True
        bad = in_keys[vv] != out_keys[a:b]
        assert not bad.any(), f"row {_first(bad, a)}: its key is not the input key of its value's row"
        del k, v, okc, bad, vv
    assert _all(seen), f"{int((~seen).sum())} input rows missing (values not a permutation of 0..n-1)"
    del seen
    want = cut_rule(order_key(out_keys, kdtype), len(sizes))
    want = [int(x) for x in (want.tolist() if th else want)]
    assert list(sizes) == np.diff(want).tolist(), f"partition sizes {_short(list(sizes))}, cut rule {_short(np.diff(want).tolist())}"


# ---- keys ((i mod D) * PHI + c) mod 2^64: rank-checked sorts of any size ---------------------------------------------
def ranked_keys(i, D, c):
    """Key patterns (int64, wrapping arithmetic) of rows i (an int64 numpy array or torch tensor)."""
    return (i % D) * signed(PHI) + signed(c)


def rank_of(keys, c):
    """Inverse of ranked_keys: (key - c) * PHI^-1 mod 2^64, as int64 (the rank for keys it made)."""
    return (keys - signed(c)) * signed(PHI_INV)


def rank_counts(n, D):
    """Rows of each rank among i in [0, n)."""
    return np.full(D, n // D, dtype=np.int64) + (np.arange(D) < n % D)


def ranked_run_ends(n, D, c):
    """End (exclusive) of every run of equal keys in the sorted (unsigned) output of ranked_keys(0..n-1)."""
    cnt = rank_counts(n, D)
    k = ranked_keys(np.arange(D, dtype=np.int64), D, c)
    cnt = cnt[np.argsort(order_key(k, "u64"), kind="stable")]
    return np.cumsum(cnt)[cnt > 0]                      # ranks with no row (n < D) have no run


def cuts_from_run_ends(run_ends, n, R):
    """cut_rule from the run ends of the sorted output: start p = floor(p n / R) moved to the end of its run."""
    c = np.array([p * n // R for p in range(R + 1)], dtype=np.int64)
    inner = (c > 0) & (c < n)
    c[inner] = run_ends[np.searchsorted(run_ends, c[inner], side="left")]
    return c
