"""Reference of the cut agreement of sort_by_key over String keys across ranks (test infrastructure).

A Python restatement of str_sort_agree_cuts (engine.cu) over W ranks, each holding its distinct keys sorted and the
row count of each: the cut key s_p of every cut p (0 < p < R) is agreed word by word, all cuts in lockstep.  A word is
str_sort_key's: bytes [7w, 7w + 7) big-endian in bits 63..8 (zero past the key's end) and min(len - 7w, 8) in bits
7..0, so comparing words compares the keys from byte 7w on, a proper prefix first.  Per cut and rank, [a, b) is the
interval of local key ranks whose earlier words equal the agreed ones.  Each round is one all-gather: either every
rank's smallest and largest word in the interval and its key count, or every rank's row count at a probed word, which
the ranks sum.
"""
from tests import str_sort_ref as SR


def word(key, w):
    """str_sort_key(key, w)"""
    pos = 7 * w
    rest = max(len(key) - pos, 0)
    return (int.from_bytes(key[pos:pos + 7].ljust(7, b"\0"), "big") << 8) | min(rest, 8)


class Rank:
    """One rank's local sort: its distinct keys in byte order and the rows' CSR by key rank."""

    def __init__(self, rows):
        rows = [SR.key_bytes(k) for k in rows]
        self.keys = sorted(set(rows))
        cnt = {}
        for k in rows:
            cnt[k] = cnt.get(k, 0) + 1
        self.row_off = [0]
        for k in self.keys:
            self.row_off.append(self.row_off[-1] + cnt[k])

    def upper(self, a, b, w, v):
        """The first rank in [a, b) whose word w is greater than v (b if none)."""
        while a < b:
            mid = (a + b) // 2
            if word(self.keys[mid], w) <= v:
                a = mid + 1
            else:
                b = mid
        return a


MINMAX, BISECT, FINAL, DONE = range(4)


def agree_cuts(ranks, R):
    """kcut[r] = [0, the local key cut of every cut p, D_r] for every rank, and the trace: rounds (all-gathers) and, per
    cut, a list of (word, bisection rounds) for every word it read."""
    N = sum(r.row_off[-1] for r in ranks)
    P = R - 1
    need = [(p * N) // R for p in range(1, R)]
    st = [MINMAX if need[i] else DONE for i in range(P)]
    w, lo, hi, v = [0] * P, [0] * P, [0] * P, [0] * P
    ab = [[[0, len(r.keys)] for _ in range(P)] for r in ranks]
    words = [[] for _ in range(P)]
    rounds = 0

    def resolve(i, x):
        v[i] = x
        if (x & 0xFF) < 8:
            st[i] = FINAL
        else:
            st[i] = MINMAX
            w[i] += 1

    while N and any(s != DONE for s in st):
        gathered = {}
        for i in range(P):
            if st[i] == FINAL:                                    # no collective: every rank's cut is upper(v)
                for r, rk in enumerate(ranks):
                    a, b = ab[r][i]
                    ab[r][i] = [rk.upper(a, b, w[i], v[i])] * 2
                st[i] = DONE
            elif st[i] == MINMAX:
                rows = []
                for r, rk in enumerate(ranks):
                    a, b = ab[r][i]
                    if w[i]:                                      # narrow to the word agreed at w - 1
                        top = rk.upper(a, b, w[i] - 1, v[i])
                        a = rk.upper(a, top, w[i] - 1, v[i] - 1) if v[i] else a
                        b = top
                        ab[r][i] = [a, b]
                    rows.append((word(rk.keys[a], w[i]), word(rk.keys[b - 1], w[i]), b - a) if a < b else (2 ** 64 - 1, 0, 0))
                gathered[i] = ("minmax", rows)
                words[i].append([w[i], 0])
            elif st[i] == BISECT:
                mid = lo[i] + (hi[i] - lo[i]) // 2
                gathered[i] = ("count", mid, [rk.row_off[rk.upper(*ab[r][i], w[i], mid)] for r, rk in enumerate(ranks)])
        if not gathered:
            continue
        rounds += 1
        for i, g in gathered.items():
            if g[0] == "minmax":
                rows = g[1]
                mn, mx, keys = min(x[0] for x in rows), max(x[1] for x in rows), sum(x[2] for x in rows)
                assert keys, "no key left for a cut"
                if keys == 1:
                    v[i], st[i] = mx, FINAL
                elif mn == mx:
                    resolve(i, mn)
                else:
                    lo[i], hi[i], st[i] = mn, mx, BISECT
            else:
                mid, counts = g[1], g[2]
                words[i][-1][1] += 1
                if sum(counts) >= need[i]:
                    hi[i] = mid
                else:
                    lo[i] = mid + 1
                if lo[i] == hi[i]:
                    resolve(i, lo[i])
    kcut = []
    for r, rk in enumerate(ranks):
        cuts = [0] + [ab[r][i][0] if need[i] else 0 for i in range(P)] + [len(rk.keys)]
        for p in range(1, R + 1):
            cuts[p] = max(cuts[p], cuts[p - 1])
        kcut.append(cuts)
    return kcut, {"rounds": rounds, "words": words}


def rank_partitions(ranks, kcut, R):
    """[rank][partition] -> the local distinct keys of that partition"""
    return [[rk.keys[kc[p]:kc[p + 1]] for p in range(R)] for rk, kc in zip(ranks, kcut)]
