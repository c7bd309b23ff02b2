"""Restatement of vega's `repartition(n)` = `coalesce(n, shuffle = true)` (src/rdd/rdd.rs:386-418) for the tests.

Map partition m gives its item i the position start_m + 1 + i (a usize, incremented before use), and
HashPartitioner::<usize> sends the item to get_partition(position) (src/partitioner.rs:21-25, 54-57).  vega leaves the
order inside a partition to a HashMap; the library fixes it as map-id order, then input order, which this restatement
returns."""
from oracle.pyref import get_partition

MASK = (1 << 64) - 1


def position(start, i):
    """The position of item i of a map partition whose start is `start` (u64 wrap-around)."""
    return (start + 1 + i) & MASK


def repartition(map_items, starts, n_reduce):
    """map_items: per map partition, its items (any objects); starts: one start per map partition.
    Returns one list per output partition: its items in map-id, then input order."""
    out = [[] for _ in range(n_reduce)]
    for m, items in enumerate(map_items):
        for i, x in enumerate(items):
            out[get_partition(position(starts[m], i), n_reduce)].append(x)
    return out
