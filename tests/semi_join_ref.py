"""Reference semi and anti joins of any number of parents (test infrastructure).

vega has no semi or anti join (Spark's subtractByKey and left semi join), so there is no reference output to compare
against.  This restates the rule of vb_semi_join_n over vega's cogroup of n parents (tests/cogroup_n_ref.py,
co_grouped_rdd.rs:206-249): `required` and `excluded` are masks over parents 1..n-1.  A key with lists l_0 .. l_{n-1}
in cogroup order is kept when l_0 is non-empty, every required parent has it and no excluded parent has it; a kept key
gives the rows (k, v) for v in l_0, in l_0's order.

`semi_join_n` works on Python rows (small cases).  `semi_of_parts` turns the array reference `ref_parts_n` into the
rows the GPU tests compare: per partition {key: [side-0 values in list order]}, u64 bits.  `semi_of_lists` does the same
for String keys from each side's group_by_key lists (tests/str_group_ref.py's contiguous slicing: input order).
"""
from tests import cogroup_n_ref as CN


def kept(lists, required, excluded):
    n = len(lists)
    return (bool(len(lists[0])) and all(len(lists[j]) for j in range(n) if required >> j & 1)
            and not any(len(lists[j]) for j in range(n) if excluded >> j & 1))


def semi_join_n(parents, n_reduce, required, excluded, int_width=8):
    """parents [(rows, num_slices), ...] -> [(k, v)] of the kept keys, each key's rows in its side-0 list order."""
    return [(k, v) for k, lists in CN.cogroup_n(parents, n_reduce, int_width) if kept(lists, required, excluded)
            for v in lists[0]]


def semi_of_parts(parts, required, excluded):
    """parts: CN.ref_parts_n's per-partition {key: (list per side)} -> per partition {key: [side-0 list]}."""
    return [{k: list(lists[0]) for k, lists in d.items() if kept(lists, required, excluded)} for d in parts]


def semi_of_lists(side_lists, R, required, excluded, partition):
    """side_lists [{key: [values]} per side], partition(key, R) -> per partition {key: [side-0 list]}."""
    out = [{} for _ in range(R)]
    for k, l0 in side_lists[0].items():
        lists = [l0] + [d.get(k, []) for d in side_lists[1:]]
        if kept(lists, required, excluded):
            out[partition(k, R)][k] = list(l0)
    return out
