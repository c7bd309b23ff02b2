"""What f64 SUM and MEAN may return for one key, in any summation order — TEST INFRASTRUCTURE ONLY.

The device adds a key's values with atomics in no fixed order, and through partial sums (hot-key caches, per-map
tables, other ranks' exports) that are added later: any binary tree over the values, under IEEE round-to-nearest.
`sum_outcome(values)` returns the set of results such an order can produce, computed with exact rationals
(fractions.Fraction; math.fsum loses the sign of a zero sum and raises on a finite overflow):

  * NaN if a value is NaN, or both +inf and -inf occur.  NaN is one class: its sign and payload are not compared.
  * +inf if +inf occurs (and no -inf); NaN too when the finite negative values could overflow to -inf in some order.
    The same with the signs swapped.
  * Finite values, exact sum S, P = sum of the positive values, N = -(sum of the negative ones), m values,
    gamma = (m-1)u / (1-(m-1)u), u = 2^-53:
      - when every partial sum is representable (all values are multiples of 2^q and P + N <= 2^(53+q)), the result
        is float(S) bit for bit, in every order;
      - otherwise it is finite with |result - S| <= gamma * (P + N).  The bound assumes no partial sum reaches the
        overflow threshold 2^1024 - 2^970; when P * (1 + gamma) can, +inf is admitted too, -inf when N * (1 + gamma)
        can, and NaN when both can (two overflowed partial sums of opposite signs meet).
  * A zero result is -0.0 exactly when every value is -0.0, and +0.0 otherwise: x + y rounds to -0.0 only when both
    are -0.0, and a nonzero exact sum never rounds to zero (additions do not underflow).

`mean_outcome(values)` is the SUM outcome divided by the count, as the device computes sum / (double)count.

Only keys that can overflow admit more than one class (NaN, +inf, -inf, finite)."""
import math
from fractions import Fraction

import numpy as np

U = Fraction(1, 1 << 53)
OVERFLOW = Fraction((1 << 1024) - (1 << 970))          # the smallest exact sum that rounds to infinity


def gamma(k):
    return k * U / (1 - k * U) if k > 0 else Fraction(0)


SCALE = 1 << 1074                                         # every finite f64 is an integer multiple of 2^-1074


def _scaled_sum(xs):
    """sum(xs) * 2^1074 as an exact integer (faster than adding Fractions)."""
    t = 0
    for x in xs:
        n, d = x.as_integer_ratio()
        t += n * (SCALE // d)
    return t


def _is_neg_zero(x):
    return x == 0.0 and math.copysign(1.0, x) < 0


def _low_bit_exponent(x):
    """q with x = odd * 2^q (x finite, nonzero)."""
    n, d = x.as_integer_ratio()
    n = abs(n)
    return ((n & -n).bit_length() - 1) - (d.bit_length() - 1)


def _approx(fr):
    return f"{float(fr):.17g}" if abs(fr) < OVERFLOW else f"{'-' if fr < 0 else ''}2^{math.log2(abs(fr.numerator)) - math.log2(fr.denominator):.4f}"


class Outcome:
    """The results one key may have: the classes NaN / +inf / -inf allowed or not, and the finite ones either one
    value bit for bit (`value`) or every float within `radius` of the exact sum `center`, with the sign of a zero
    fixed by `neg_zero`.  `div` divides the finite results by a count (MEAN)."""

    def __init__(self, nan=False, pinf=False, ninf=False, finite=False, value=None, center=None, radius=None,
                 neg_zero=False, div=1):
        self.nan, self.pinf, self.ninf, self.finite = nan, pinf, ninf, finite
        self.value, self.center, self.radius, self.neg_zero, self.div = value, center, radius, neg_zero, div

    def classes(self):
        return self.nan + self.pinf + self.ninf + self.finite

    def exact(self):
        """The one float it admits (None when it admits several): NaN, an infinity or a finite value."""
        if self.classes() != 1:
            return None
        if self.nan:
            return math.nan
        if self.pinf or self.ninf:
            return math.inf if self.pinf else -math.inf
        return self.value

    def admits(self, g):
        g = float(g)
        if math.isnan(g):
            return self.nan
        if math.isinf(g):
            return self.pinf if g > 0 else self.ninf
        if not self.finite:
            return False
        if self.value is not None:
            return np.float64(g).view(np.uint64) == np.float64(self.value).view(np.uint64)
        if g == 0.0 and self.div == 1 and _is_neg_zero(g) != self.neg_zero:
            return False                     # (a MEAN may round a tiny negative sum to -0.0)
        # MEAN over an inexact sum: the sum's bound divided by the count, plus the division's rounding
        slack = Fraction(math.ulp(g)) if self.div > 1 else 0
        return abs(Fraction(g) - self.center / self.div) <= self.radius / self.div + slack

    def __repr__(self):
        cls = [c for c, on in (("nan", self.nan), ("+inf", self.pinf), ("-inf", self.ninf)) if on]
        if self.finite:
            cls.append(repr(self.value) if self.value is not None else
                       f"{_approx(self.center / self.div)}+-{_approx(self.radius / self.div)}")
        return "{" + ", ".join(cls) + "}"


def sum_outcome(values):
    xs = [float(x) for x in values]
    assert xs, "a key has at least one value"
    m = len(xs)
    fin = [x for x in xs if math.isfinite(x)]
    has_nan = len(fin) < m and any(math.isnan(x) for x in xs)
    has_pinf = math.inf in xs
    has_ninf = -math.inf in xs
    P = Fraction(_scaled_sum(x for x in fin if x > 0), SCALE)
    N = -Fraction(_scaled_sum(x for x in fin if x < 0), SCALE)
    g = gamma(m - 1)
    pos_ovf = P * (1 + g) >= OVERFLOW
    neg_ovf = N * (1 + g) >= OVERFLOW
    if has_nan or (has_pinf and has_ninf):
        return Outcome(nan=True)
    if has_pinf:
        return Outcome(pinf=True, nan=neg_ovf)
    if has_ninf:
        return Outcome(ninf=True, nan=pos_ovf)
    neg_zero = all(_is_neg_zero(x) for x in xs)
    S = P - N
    nz = [x for x in xs if x != 0.0]
    if not nz or (P + N < OVERFLOW and P + N <= Fraction(2) ** (53 + min(_low_bit_exponent(x) for x in nz))):
        v = float(S)
        return Outcome(finite=True, value=-0.0 if neg_zero else v, neg_zero=neg_zero)
    r = g * (P + N)
    finite = S - r < OVERFLOW and S + r > -OVERFLOW          # else every order rounds (or overflows) to infinity
    return Outcome(finite=finite, center=S, radius=r, neg_zero=neg_zero, pinf=pos_ovf, ninf=neg_ovf,
                   nan=pos_ovf and neg_ovf)


def mean_outcome(values):
    """sum_outcome divided by the count: NaN and the infinities stay, an exact sum gives fl(sum / m) bit for bit (a
    zero keeps its sign), an inexact one its bound over m (plus the division's rounding)."""
    s, m = sum_outcome(values), len(values)
    if s.value is not None:
        s.value = float(np.float64(s.value) / np.float64(m))
    else:
        s.div = m
    return s


# ---- whole shuffles -------------------------------------------------------------------------------------------------
def _groups(keys, vals):
    keys = np.ascontiguousarray(keys).view(np.uint64)
    vals = np.ascontiguousarray(vals, dtype=np.float64)
    order = np.argsort(keys, kind="stable")
    ks, vs = keys[order], vals[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]]) if len(ks) else np.zeros(0, np.int64)
    ends = np.r_[starts[1:], len(ks)].astype(np.int64)
    return ks, vs, starts, ends


def _per_key(vs, starts, ends):
    """Vectorized over keys: (exact, sums, all_finite, abs_sum, has_nan, has_pinf, has_ninf).  exact: every value is finite and every partial sum
    is representable, so any order gives sums[i] (-0.0 when every value is -0.0); abs_sum: sum |x| rounded up enough
    to bound the exact one."""
    bits = vs.view(np.uint64)
    e = ((bits >> np.uint64(52)) & np.uint64(0x7FF)).astype(np.int64)
    mant = bits & np.uint64((1 << 52) - 1)
    mant = np.where(e > 0, mant | np.uint64(1 << 52), mant)
    low = mant & (~mant + np.uint64(1))                                  # lowest set bit (0 for zeros)
    lowexp = np.log2(np.where(low > 0, low, 1).astype(np.float64)).astype(np.int64)
    q = np.where(mant > 0, np.maximum(e, 1) - 1075 + lowexp, 900)        # x = odd * 2^q; a zero does not lower q
    finite = e < 0x7FF
    all_finite = np.logical_and.reduceat(finite, starts)
    qmin = np.minimum.reduceat(q, starts)
    m = (ends - starts).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        abs_sum = np.add.reduceat(np.where(finite, np.abs(vs), 0.0), starts) * (1 + 2 * m * 2.0 ** -53)
        lim = np.exp2(np.minimum(qmin + 53, 1023).astype(np.float64))
        exact = all_finite & (abs_sum <= lim) & (qmin + 53 <= 1023)
        sums = np.add.reduceat(np.where(finite, vs, 0.0), starts)          # exact where `exact`: any order gives it
    neg_zero = np.logical_and.reduceat(bits == np.uint64(1 << 63), starts)
    sums = np.where(neg_zero, -0.0, np.where(sums == 0, 0.0, sums))
    has_nan = np.logical_or.reduceat(np.isnan(vs), starts)
    return exact, sums, all_finite, abs_sum, has_nan, np.logical_or.reduceat(vs == np.inf, starts), \
        np.logical_or.reduceat(vs == -np.inf, starts)


def key_outcomes(keys, vals, mean=False):
    """{key (u64): Outcome} of every key of (keys, vals) for SUM (MEAN with mean=True).  Exact keys and finite keys far
    from overflow are judged without rationals: the first by the vectorized float sum, the second around math.fsum
    (correctly rounded, so half an ulp of it is added to the bound); the rest by sum_outcome."""
    ks, vs, starts, ends = _groups(keys, vals)
    out = {}
    if len(ks) == 0:
        return out
    exact, sums, all_finite, abs_sum, has_nan, has_pinf, has_ninf = _per_key(vs, starts, ends)
    counts = ends - starts
    if mean:
        sums = sums / np.maximum(counts, 1).astype(np.float64)
    vl = vs.tolist()
    for i, k in enumerate(ks[starts].tolist()):
        x, m = vl[starts[i]:ends[i]], int(counts[i])
        if exact[i]:
            out[k] = Outcome(finite=True, value=float(sums[i]))
        elif has_nan[i] or (has_pinf[i] and has_ninf[i]):
            out[k] = Outcome(nan=True)
        elif abs_sum[i] < 2.0 ** 1000 and not all_finite[i]:      # one infinity, and the finite values cannot overflow
            out[k] = Outcome(pinf=bool(has_pinf[i]), ninf=bool(has_ninf[i]))
        elif all_finite[i] and abs_sum[i] < 2.0 ** 1000:
            c = math.fsum(x)
            r = gamma(m - 1) * Fraction(float(abs_sum[i])) + Fraction(math.ulp(c)) / 2
            out[k] = Outcome(finite=True, center=Fraction(c), radius=r, div=m if mean else 1)
        else:
            out[k] = mean_outcome(x) if mean else sum_outcome(x)
    return out


def assert_outcomes(got, outcomes, what="f64 sums", exact=False, lenient=None):
    """got: {key: float}; every key of `outcomes` in it and admitted.  exact=True: every key must have a single
    bit-exact outcome.  lenient: the keys allowed more than one class (None: any key)."""
    missing = outcomes.keys() - got.keys()
    extra = got.keys() - outcomes.keys()
    assert not missing and not extra, f"{len(missing)} keys missing, {len(extra)} keys not in the input"
    bad, loose = [], []
    for k, oc in outcomes.items():
        if exact and oc.exact() is None:
            loose.append((hex(k), oc))
        elif lenient is not None and k not in lenient and oc.classes() != 1:
            loose.append((hex(k), oc))
        if not oc.admits(got[k]):
            bad.append((hex(k), got[k], oc))
    assert not loose, f"{len(loose)} keys the reference cannot pin down (input not as the case intends): {loose[:5]}"
    assert not bad, f"{len(bad)} of {len(outcomes)} {what} wrong (key, got, admitted): {bad[:5]}"
