"""The checks of tests/sort_ref.py against the C oracle's sort, on numpy and on CPU torch: each accepts a correct
result and rejects a result with two equal-key rows swapped, a duplicated row, a cut moved inside a run of equal keys
and a partition boundary off by one."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import sort_ref as S
from tests.util import f64_total_key

KDTYPES = ["u64", "i64", "f64"]


def _case(kdtype, n=4000, D=60, seed=0):
    rng = np.random.default_rng([KDTYPES.index(kdtype), seed])
    keys = S.run_keys(rng, n, kdtype, D)
    vals = np.arange(n, dtype=np.int64)
    ok, ov, ps = O.sort_by_key(keys, vals, 8, kdtype)
    return keys, vals, S.bits(ok), S.bits(ov), ps.astype(np.int64)


def _parts(ok, ov, ps):
    return [(ok[ps[r]:ps[r + 1]], ov[ps[r]:ps[r + 1]]) for r in range(len(ps) - 1)]


def _exact(backend, keys, ok, ov, sizes, kdtype):
    if backend == "torch":
        import torch
        keys, ok, ov = (torch.from_numpy(np.ascontiguousarray(x)) for x in (keys, ok, ov))
    S.check_sorted_exact(keys, ok, ov, sizes, kdtype, chunk=700)      # several chunks: pairs across their boundaries


def _runs(ok):
    """(start, length) of every run of equal keys, longest first."""
    starts = np.flatnonzero(np.r_[True, ok[1:] != ok[:-1]])
    lens = np.diff(np.r_[starts, len(ok)])
    order = np.argsort(-lens, kind="stable")
    return starts[order], lens[order]


@pytest.mark.parametrize("kdtype", KDTYPES)
def test_order_key_is_the_dtype_order(kdtype):
    rng = np.random.default_rng(5)
    b = S.run_keys(rng, 5000, kdtype, 400, hot=0)
    got = np.argsort(S.order_key(b, kdtype), kind="stable")
    if kdtype == "u64":
        want = np.argsort(b.view(np.uint64), kind="stable")
    elif kdtype == "i64":
        want = np.argsort(b, kind="stable")
    else:
        want = np.argsort(f64_total_key(b.view(np.float64)), kind="stable")
    assert np.array_equal(got, want)
    assert len(np.unique(S.order_key(b, kdtype))) == len(np.unique(b))          # a bijection: equal means bit-equal
    if kdtype == "f64":
        assert set(S.EDGE["f64"]) <= set(b.tolist())                              # every special reaches the input


@pytest.mark.parametrize("backend", ["numpy", "torch"])
@pytest.mark.parametrize("kdtype", KDTYPES)
def test_checks_accept_the_oracle(kdtype, backend):
    keys, vals, ok, ov, ps = _case(kdtype)
    S.assert_sort_equal(_parts(ok, ov, ps), keys, vals, 8, kdtype)
    _exact(backend, keys, ok, ov, np.diff(ps).tolist(), kdtype)


@pytest.mark.parametrize("backend", ["numpy", "torch"])
@pytest.mark.parametrize("kdtype", KDTYPES)
@pytest.mark.parametrize("fault", ["swap_equal_keys", "duplicate_row", "cut_inside_run", "cut_off_by_one"])
def test_checks_reject(kdtype, backend, fault):
    keys, vals, ok, ov, ps = _case(kdtype, seed=1)
    ok, ov, ps = ok.copy(), ov.copy(), ps.copy()
    starts, lens = _runs(ok)
    s = int(starts[0])                                   # the longest run
    if fault == "swap_equal_keys":
        ov[s], ov[s + 1] = ov[s + 1], ov[s]
    elif fault == "duplicate_row":
        j = int(starts[1]) + 1                           # inside the second-longest run: keys stay sorted
        ok[j], ov[j] = ok[j - 1], ov[j - 1]
    elif fault == "cut_inside_run":
        p = int(np.flatnonzero((ps > 0) & (ps < len(ok)))[0])
        run_before = ok[ps[p] - 1] == ok[ps[p] - 2]
        assert run_before
        ps[p] -= 1                                       # now splits the run that ends at the cut
    else:
        p = int(np.flatnonzero((ps > 0) & (ps < len(ok)))[-1])
        ps[p] += 1
    with pytest.raises(AssertionError):
        S.assert_sort_equal(_parts(ok, ov, ps), keys, vals, 8, kdtype)
    with pytest.raises(AssertionError):
        _exact(backend, keys, ok, ov, np.diff(ps).tolist(), kdtype)


@pytest.mark.parametrize("backend", ["numpy", "torch"])
@pytest.mark.parametrize("n, R, D", [(1000, 1, 50), (7, 13, 3), (5, 8, 5), (0, 4, 1), (1, 3, 1), (9, 9, 9),
                                     (3000, 65536, 40), (5000, 16, 2)])
def test_cut_rule_matches_oracle(backend, n, R, D):
    """R = 1, R > n, R = n, and runs spanning several cuts (D = 2: about 90 % of the rows on one key)."""
    rng = np.random.default_rng([n, R, D])
    keys = rng.integers(0, D, n).astype(np.uint64) * np.uint64(S.PHI)
    if D == 2:
        keys[rng.random(n) < 0.9] = np.uint64(7)
    ok, _, ps = O.sort_by_key(keys, None, R, "u64")
    okeys = S.order_key(S.bits(ok), "u64")
    if backend == "torch":
        import torch
        got = S.cut_rule(torch.from_numpy(okeys), R).numpy()
    else:
        got = S.cut_rule(okeys, R)
    assert np.array_equal(got, ps.astype(np.int64))
    if D == 2 and n:
        assert (np.diff(got) == 0).sum() >= 8                 # several empty partitions


@pytest.mark.parametrize("backend", ["numpy", "torch"])
def test_ranked_keys_round_trip(backend):
    """rank_of inverts ranked_keys under wrapping int64 arithmetic, across 2^31 and 2^32."""
    D, c = (1 << 20) + 7, 0xDEADBEEF12345
    i = np.concatenate([np.arange(5000), np.arange((1 << 31) - 3000, (1 << 31) + 3000),
                        np.arange((1 << 32) - 100, (1 << 32) + 100)]).astype(np.int64)
    if backend == "torch":
        import torch
        i = torch.from_numpy(i)
    k = S.ranked_keys(i, D, c)
    r = S.rank_of(k, c)
    assert bool(((r >= 0) & (r < D)).all()) and bool((r == i % D).all())
    want = [((x % D) * S.PHI + c) & S.MASK64 for x in np.asarray(i).tolist()]      # the modular formula, exactly
    assert np.asarray(k).view(np.uint64).tolist() == want


@pytest.mark.parametrize("n, D, R", [(50_000, 1000, 8), (3001, 1000, 7), (999, 1000, 4), (5000, 3, 16)])
def test_ranked_run_ends_match_oracle(n, D, R):
    c = 0x1234567
    keys = S.ranked_keys(np.arange(n, dtype=np.int64), D, c).view(np.uint64)
    ok, _, ps = O.sort_by_key(keys, None, R, "u64")
    ends = S.ranked_run_ends(n, D, c)
    starts = np.flatnonzero(np.r_[True, ok[1:] != ok[:-1]])
    assert np.array_equal(ends, np.r_[starts[1:], n])
    assert np.array_equal(S.cuts_from_run_ends(ends, n, R), ps.astype(np.int64))
