"""Reference of sort_by_key over String keys (test infrastructure).

The output is fully determined: the rows of the map tasks, concatenated in map-id order, stably sorted by key bytes in
Rust `String` order (`<[u8] as Ord>`: bytes compare unsigned, a proper prefix sorts first; Python's `bytes` order),
then cut into R partitions by sort_ref.cut_rule applied to the keys' ranks (partition p starts at floor(p·n/R), moved
forward past every row of the key just before it).
"""
import numpy as np

from tests import sort_ref


def key_bytes(k):
    """A key as the bytes the library sees: str keys as UTF-8 (surrogate escapes back to their bytes), bytes as is."""
    return bytes(k) if isinstance(k, (bytes, bytearray)) else k.encode("utf-8", "surrogateescape")


def sort_rows(keys, vals=None):
    """keys: str / bytes keys in map-id order; vals: a numpy array or None.  Returns (sorted keys as bytes, the values
    in the same order or None, the dense rank of every sorted key as int64)."""
    kb = [key_bytes(k) for k in keys]
    order = sorted(range(len(kb)), key=kb.__getitem__)        # list.sort is stable
    sk = [kb[i] for i in order]
    rank = {k: r for r, k in enumerate(sorted(set(kb)))}
    ranks = np.array([rank[k] for k in sk], dtype=np.int64)
    sv = None if vals is None else np.asarray(vals)[np.array(order, dtype=np.int64)]
    return sk, sv, ranks


def partitions(keys, vals, R):
    """[(keys as bytes, values or None)] for each of the R partitions."""
    sk, sv, ranks = sort_rows(keys, vals)
    starts = sort_ref.cut_rule(ranks, R).tolist()
    return [(sk[a:b], None if sv is None else sv[a:b]) for a, b in zip(starts[:-1], starts[1:])]
