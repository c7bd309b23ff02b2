"""Reference outer join of any number of parents (test infrastructure).

vega has no outer join, so there is no reference output to compare against.  This restates the rule of
vb_join_n_outer over vega's cogroup of n parents (tests/cogroup_n_ref.py, co_grouped_rdd.rs:206-249): bit j of
`required` marks parent j as required.  A key with lists l_0 .. l_{n-1} in cogroup order gives rows only if every
required parent has it; a parent with the key contributes l_j, an optional parent without it the single slot [None]:

    for v0 in L0 { for v1 in L1 { ... } } -> (k, [v0, v1, ..., v_{n-1}])      (the last parent varies fastest)

`join_n_outer` works on Python rows (small cases).  `outer_of_parts` turns the array reference `ref_parts_n` into the
rows the GPU tests compare: per partition {key: [(v_0, ..., v_{n-1}, valid_0, ..., valid_{n-1}), ...]} in nested order,
u64 bits, 0 and validity 0 in a None slot.
"""
import itertools

from tests import cogroup_n_ref as CN


def kept(lists, required):
    """A key is kept when every required parent has it (and, for the arrays, some parent has it at all)."""
    return any(lists) and all(lists[j] for j in range(len(lists)) if required >> j & 1)


def join_n_outer(parents, n_reduce, required, int_width=8):
    out = []
    for k, lists in CN.cogroup_n(parents, n_reduce, int_width):
        if kept(lists, required):
            out += [(k, list(row)) for row in itertools.product(*[l if l else [None] for l in lists])]
    return out


def outer_of_parts(parts, required):
    """parts: CN.ref_parts_n's per-partition {key: (list per side)} -> per partition {key: [row tuples in order]}."""
    out = []
    for d in parts:
        rows = {}
        for k, lists in d.items():
            if not kept(lists, required):
                continue
            slots = [[(v, 1) for v in l] if l else [(0, 0)] for l in lists]
            rows[k] = [tuple(v for v, _ in row) + tuple(ok for _, ok in row) for row in itertools.product(*slots)]
        out.append(rows)
    return out
