"""W ranks of one shuffle in one process (test infrastructure).

Export and import are plain buffers plus host counts, so W shuffles created with set_dist(rank, W) can swap their columns
with a few torch.cat calls (swap_columns, used by the integer, String and combine_by_key harnesses): the all-to-all-v of
vega_b200/dist.py without a second process or GPU.  `run_ranks` drives
any engine with the five calls of vega_b200.dist.CudaEngine (create, map, export, import_, seal): the library itself,
or tests/fake_engine.FakeEngine on the CPU.
"""
import numpy as np
import torch

from vega_b200 import dist as vdist
from vega_b200.rdd import slice_starts


def maps_by_rank(n, M, W, place):
    """ParallelCollection slices of n rows into M map tasks, given to the ranks in map_block order.
    place(map_id, lo, hi) -> (keys, vals) as the engine's map call takes them."""
    starts = slice_starts(n, M) if n else np.zeros(M + 1, dtype=np.int64)
    out = []
    for r in range(W):
        lo, hi = vdist.map_block(r, W, M)
        out.append([(m, *place(m, int(starts[m]), int(starts[m + 1]))) for m in range(lo, hi)])
    return out


def _stats(sh):
    return sh.stats() if hasattr(sh, "stats") else None


def run_ranks(engine, W, agg, maps, R, kcode, vcode, key_width=8, hint=0, n_map=None):
    """One shuffle on W ranks: map every rank's tasks, export every rank, swap the slices, import, seal.

    maps[r]: [(map_id, keys, vals)] of rank r.  Returns (sealed shuffles by rank, stats snapshots taken after every
    export and before any seal: the map-side evidence, which the import merge of the seal would add to)."""
    n_map = n_map or max(1, sum(len(m) for m in maps))
    shs = [engine.create(n_map, R, kcode, vcode, agg, r, W, key_width=key_width, hint=hint) for r in range(W)]
    for r in range(W):
        for map_id, k, v in maps[r]:
            engine.map(shs[r], map_id, k, v)
    if W == 1:
        snaps = [_stats(shs[0])]
        engine.seal(shs[0])
        return shs, snaps
    exports = [engine.export(sh, W) for sh in shs]
    snaps = [_stats(sh) for sh in shs]
    for sh, recv in zip(shs, all_to_all_v(exports)):
        engine.import_(sh, *recv)
    for sh in shs:
        engine.seal(sh)
    return shs, snaps


def swap_columns(exports):
    """The all-to-all-v of vega_b200/dist.py in one process.  exports[src] = (columns, splits): each column (None
    allowed) destination-major along its first dimension, cut by splits[i][dst] rows per destination -> per destination
    (columns, splits[i][src] per source) with the sources concatenated in ascending order (source-rank major: map-id
    order).  The received columns are new tensors: a rank's exported buffers belong to the library and are freed by
    that rank's seal."""
    parts = [[None if c is None else torch.split(c, list(n)) for c, n in zip(cols, splits)] for cols, splits in exports]
    return [([None if p is None else torch.cat([src[i][d] for src in parts]) for i, p in enumerate(parts[0])],
             [[splits[i][d] for _, splits in exports] for i in range(len(parts[0]))]) for d in range(len(exports))]


def all_to_all_v(exports):
    """exports[src] = (counts[dst], keys, vals), destination-major -> per destination (keys, vals, counts[src])."""
    return [(k, v, n[0]) for (k, v), n in swap_columns([([k, v], [c, c]) for c, k, v in exports])]


def owned_parts(engine, shs, R):
    """Every partition of every rank: asserts that partition r has rows only on rank r % W, returns the owners'."""
    W = len(shs)
    out = [None] * R
    for d, sh in enumerate(shs):
        for r in range(R):
            p = engine.reduce(sh, r)
            if r % W == d:
                out[r] = p
            else:
                assert len(p[0]) == 0, f"rank {d} holds keys of partition {r}, owned by rank {r % W}"
    return out


def group_dict(keys, offs, vals):
    """{key (u64): [values as u64 bits, in order]} of one group partition."""
    k = np.ascontiguousarray(keys).view(np.uint64).tolist()
    o = np.asarray(offs).astype(np.int64)
    assert o[0] == 0 and o[-1] == len(vals), "offsets do not start at 0 or end at the value count"
    v = np.ascontiguousarray(vals).view(np.uint64).tolist()
    d = {kk: v[o[i]:o[i + 1]] for i, kk in enumerate(k)}
    assert len(d) == len(k), "a key appears twice in one partition"
    return d
