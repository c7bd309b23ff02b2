"""tests/f64_sum_ref.py against brute force: every result of every summation order and tree shape of small multisets
must be in the reference's outcome set, and a key that cannot overflow must have exactly one outcome class."""
import math

import numpy as np
import pytest

from tests import f64_sum_ref as F

POOL = [0.0, -0.0, math.inf, -math.inf, math.nan, -math.nan, 1.5e308, -1.5e308, 5e-324, -5e-324, 2.5e-310,
        -1.1e-315, 2.2250738585072009e-308]


def every_order(xs):
    """Every float64 result of adding xs in some order and tree shape (numpy float64 addition, round to nearest),
    NaN results as one np.nan: subset DP, each subset's results from every split into two non-empty parts."""
    n = len(xs)
    res = {1 << i: np.array([xs[i]], dtype=np.float64) for i in range(n)}
    with np.errstate(all="ignore"):
        for s in range(1, 1 << n):
            if s in res:
                continue
            out = []
            a = (s - 1) & s
            while a:
                b = s ^ a
                if a < b:                                     # each unordered split once (addition commutes)
                    out.append(np.add.outer(res[a], res[b]).ravel())
                a = (a - 1) & s
            r = np.concatenate(out)
            bits = np.unique(np.where(np.isnan(r), np.nan, r).view(np.uint64))
            res[s] = bits.view(np.float64)
    return res[(1 << n) - 1]


def draw(rng, n):
    """n values from the pool above, exact k * 2^-30 and values with low bits that round (1 + k * 2^-52, k * 2^-60)."""
    out = []
    for _ in range(n):
        c = rng.integers(0, 4)
        if c == 0:
            out.append(POOL[rng.integers(0, len(POOL))])
        elif c == 1:
            out.append(math.ldexp(float(rng.integers(-(1 << 20), 1 << 20)), -30))
        elif c == 2:
            out.append(float(rng.choice([-1, 1])) * (1 + math.ldexp(float(rng.integers(1, 1 << 10)), -52)))
        else:
            out.append(math.ldexp(float(rng.integers(-(1 << 10), 1 << 10)), -60))
    return out


def can_overflow(xs):
    return any(abs(x) == 1.5e308 for x in xs)


@pytest.mark.parametrize("seed", range(8))
def test_every_order_is_admitted(seed):
    rng = np.random.default_rng(seed)
    for _ in range(400):
        xs = draw(rng, int(rng.integers(1, 7)))
        oc, mc = F.sum_outcome(xs), F.mean_outcome(xs)
        if not can_overflow(xs):
            assert oc.classes() == 1, (xs, oc)
        for r in every_order(xs).tolist():
            assert oc.admits(r), (xs, r, oc)
            with np.errstate(all="ignore"):
                assert mc.admits(float(np.float64(r) / np.float64(len(xs)))), (xs, r, mc)


def test_special_cases():
    assert F.sum_outcome([-0.0, -0.0]).exact() == 0.0
    assert math.copysign(1, F.sum_outcome([-0.0, -0.0]).exact()) < 0
    assert not F.sum_outcome([-0.0, -0.0]).admits(0.0)
    assert F.sum_outcome([-0.0, 0.0, -0.0]).admits(0.0) and not F.sum_outcome([-0.0, 0.0]).admits(-0.0)
    assert F.sum_outcome([1.0, -1.0, -0.0]).admits(0.0) and not F.sum_outcome([1.0, -1.0, -0.0]).admits(-0.0)
    assert F.mean_outcome([-0.0] * 3).admits(-0.0) and not F.mean_outcome([-0.0] * 3).admits(0.0)
    for xs in ([math.nan, 1.0], [-math.nan], [math.inf, -math.inf, 2.0]):
        oc = F.sum_outcome(xs)
        assert oc.admits(math.nan) and oc.classes() == 1
    assert F.sum_outcome([math.inf, 1e308, 1e308]).exact() == math.inf
    oc = F.sum_outcome([math.inf, -1.5e308, -1.5e308])          # (-1.5e308 + -1.5e308) + inf is NaN
    assert oc.admits(math.inf) and oc.admits(math.nan) and not oc.admits(-math.inf)
    oc = F.sum_outcome([1.5e308, 1.5e308, -1.5e308])            # inf or 1.5e308 by order; never -inf
    assert oc.admits(math.inf) and oc.admits(1.5e308) and not oc.admits(-math.inf) and not oc.admits(math.nan)
    oc = F.sum_outcome([1.5e308, 1.5e308, -1.5e308, -1.5e308])  # both partials can overflow: NaN too
    assert oc.admits(math.nan) and oc.admits(0.0) and oc.admits(math.inf) and oc.admits(-math.inf)
    assert F.sum_outcome([1e308, 1e308]).exact() == math.inf    # the exact sum rounds to inf: no order avoids it
    top = 1.7976931348623157e308                                 # 2^1024 - 2^971
    oc = F.sum_outcome([top, math.ldexp(1.0, 970)])              # the tie at 2^1024 - 2^970 rounds up
    assert oc.admits(math.inf) and not oc.admits(math.nan) and repr(oc).startswith("{+inf, 2^1024.0000")
    oc = F.sum_outcome([top, math.ldexp(1.0, 969)])              # rounds to top; the bound also admits +inf
    assert oc.admits(top) and oc.admits(math.inf) and not oc.admits(math.nan)


def test_exact_and_bound():
    xs = [math.ldexp(k, -30) for k in (3, -7, 1 << 20, 5)]
    assert F.sum_outcome(xs).exact() == math.fsum(xs)
    xs = [1.0, 2.0 ** -53, 2.0 ** -53]                           # 1 or 1 + 2^-52 by order
    oc = F.sum_outcome(xs)
    assert oc.exact() is None and oc.classes() == 1
    assert oc.admits(1.0) and oc.admits(1.0 + 2.0 ** -52) and not oc.admits(1.0 + 2.0 ** -50)


@pytest.mark.parametrize("mean", [False, True])
def test_key_outcomes_agree_with_sum_outcome(mean):
    """The vectorized shortcuts of key_outcomes admit what sum_outcome / mean_outcome admit, on every brute-forced
    result of random keys."""
    rng = np.random.default_rng(11 + mean)
    groups = [draw(rng, int(rng.integers(1, 6))) for _ in range(300)]
    groups += [[-0.0] * 4, [0.0, -0.0], [math.ldexp(3, -30), math.ldexp(-3, -30), -0.0], [5e-324] * 3]
    keys = np.concatenate([np.full(len(g), i, np.uint64) for i, g in enumerate(groups)])
    vals = np.concatenate([np.array(g, dtype=np.float64) for g in groups])
    perm = rng.permutation(len(keys))
    ocs = F.key_outcomes(keys[perm], vals[perm], mean=mean)
    assert sorted(ocs) == list(range(len(groups)))
    for i, g in enumerate(groups):
        ref = F.mean_outcome(g) if mean else F.sum_outcome(g)
        assert ocs[i].classes() == ref.classes(), (g, ocs[i], ref)
        for r in every_order(g).tolist():
            with np.errstate(all="ignore"):
                x = float(np.float64(r) / np.float64(len(g))) if mean else r
            assert ocs[i].admits(x) == ref.admits(x) or (ocs[i].admits(x) and ref.value is None), (g, x, ocs[i], ref)
            assert ocs[i].admits(x), (g, x, ocs[i])


def test_assert_outcomes_reports():
    keys = np.array([1, 1, 2], np.uint64)
    vals = np.array([-0.0, -0.0, math.nan])
    ocs = F.key_outcomes(keys, vals)
    F.assert_outcomes({1: -0.0, 2: -math.nan}, ocs, exact=True)
    with pytest.raises(AssertionError, match="wrong"):
        F.assert_outcomes({1: 0.0, 2: math.nan}, ocs)
    with pytest.raises(AssertionError, match="missing"):
        F.assert_outcomes({1: -0.0}, ocs)
    ocs = F.key_outcomes(np.array([3, 3, 3], np.uint64), np.array([1.5e308, 1.5e308, -1.5e308]))
    with pytest.raises(AssertionError, match="cannot pin down"):
        F.assert_outcomes({3: math.inf}, ocs, lenient=set())
    F.assert_outcomes({3: math.inf}, ocs, lenient={3})
