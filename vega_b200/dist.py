"""One-process-per-GPU shuffle: the data plane between map side and reduce side.

The reference moves shuffle blocks with one HTTP GET per (map, reduce) pair
(src/shuffle/shuffle_fetcher.rs:61-86 → src/shuffle/shuffle_manager.rs:176-251).  Here every
rank packs its map output by destination rank on the device (vb_shuffle_export_prepare: a
stable multisplit, so rows stay in map-id / encounter order) as a few columns, each split by one
vector of per-destination counts.  The ranks swap the counts and ONE all-to-all-v per column
(torch.distributed → NCCL grouped send/recv over NVLink/NVSwitch; gloo on CPU for the host-logic
tests) delivers them: all_to_all_v, the one exchange of every shuffle kind.  Reduce partition r is
owned by rank r % world; map partitions are assigned to ranks in contiguous blocks so that the
source-rank-major receive order IS map-id order (group value order, SURVEY.md F5).

The columns of each kind (run_shuffle, run_str_shuffle, run_combine_shuffle and run_str_combine_shuffle share one
driver, _exchange):
- integer rows (CudaEngine): keys and values, both split by the row counts.  Reduce ops exchange *combined* rows
  (≤ distinct keys per rank — map-side combine, src/dependency.rs:203-209), group ops raw rows.
- String keys (StrCudaEngine): u32 key lengths and u32 value counts (GROUP) split by the key counts, key bytes by the
  byte counts, u64 values by the value counts.
- combine_by_key (CombineCudaEngine): one row per distinct key, the key and the partial of every accumulator, packed
  as one [rows][1 + n_acc] column.
- combine_by_key over String keys (StrCombineCudaEngine): u32 key lengths split by the key counts, key bytes by the
  byte counts, and the partials of every accumulator packed as one [keys][n_acc] column split by the key counts.
- byte-string values (BytesCudaEngine, StrBytesCudaEngine): the columns of integer rows or of String keys without the
  values, plus u32 value lengths split by the row (or value) counts and the values' bytes split by the byte counts.
  A value's reference never leaves its rank: the receiver stores the bytes it got and issues fresh references, so the
  results of a rank are gathered through that rank's shuffle (Shuffle.gather).  sort_by_key with byte-string values
  crosses ranks inside the library only (vb_shuffle_exchange).

The exchange itself lives in libvega_b200.so (vb_ctx_comm_init + vb_shuffle_exchange: NCCL grouped
send/recv, or the fused peer-memory scatter, on the library's stream).  The run_*shuffle functions call it
whenever the context has a communicator; the torch.distributed code paths below remain for the two cases the
library's NCCL communicator cannot cover: the CPU (gloo) tests of the host logic with an oracle-backed stand-in
engine, and two ranks sharing ONE GPU on a single-GPU test box (NCCL refuses duplicate devices).
"""
import ctypes

import numpy as np

from . import _lib as L
from .rdd import Shuffle, StrKeys, StrShuffle, _BytesCol, _Col, _is_str_keys, _StrCol


def map_block(rank, world, n_map):
    """Contiguous block of map partitions owned by `rank`: [lo, hi)."""
    return (rank * n_map) // world, ((rank + 1) * n_map) // world


class _DevArray:
    """Zero-copy view of a library-owned device buffer for torch.as_tensor."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 2}


class CudaEngine:
    """libvega_b200 on this rank's GPU."""

    def __init__(self, sc):
        self.sc = sc

    def create(self, n_map, n_reduce, kcode, vcode, agg, rank, world, key_width=8, hint=0):
        return Shuffle(self.sc, n_map, n_reduce, kcode, vcode, agg, key_width=key_width, hint=hint, rank=rank, world=world)

    def map(self, sh, map_id, keys, vals):
        k = keys if isinstance(keys, _Col) else _Col(keys, allow_rows=True)
        v = None if vals is None else (vals if isinstance(vals, _Col) else _Col(vals, role="value"))
        sh.map(map_id, k, v, 0, k.n)

    def export(self, sh, world):
        import torch
        counts = (ctypes.c_uint64 * world)()
        L.check(sh._lib.vb_shuffle_export_prepare(sh._h, counts))
        counts = [int(c) for c in counts]
        kp, vp = ctypes.c_void_p(), ctypes.c_void_p()
        L.check(sh._lib.vb_shuffle_export_buffers(sh._h, ctypes.byref(kp), ctypes.byref(vp)))
        n = sum(counts)
        dev = f"cuda:{sh._lib.vb_ctx_device(self.sc._h)}"
        if n == 0:
            e = torch.empty(0, dtype=torch.int64, device=dev)
            return counts, e, e.clone()
        keys = torch.as_tensor(_DevArray(kp.value, n), device=dev)
        vals = torch.as_tensor(_DevArray(vp.value, n), device=dev)
        return counts, keys, vals

    def import_(self, sh, keys, vals, counts):
        import torch
        if keys.is_cuda:
            # NCCL collectives are stream-ordered on torch's stream; the library reads on its own stream
            torch.cuda.current_stream(keys.device).synchronize()
        sh._imported = (keys, vals)            # keep the tensors alive until seal
        c = (ctypes.c_uint64 * len(counts))(*counts)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
        L.check(sh._lib.vb_shuffle_import(sh._h, p(keys), p(vals), c))

    def seal(self, sh):
        sh.seal()
        sh._imported = None

    def reduce(self, sh, r):
        return sh.reduce(r)


def p2p_layout(allc, rank):
    """Arena layout of the fused exchange from the all-gathered count matrix allc[src][dst]:
    (total rows each rank receives, row offset of `rank`'s block inside every destination's arena,
    rows `rank` receives from every source).  Blocks are source-rank major, so the arena order is map-id order."""
    world = len(allc)
    total_recv = [sum(allc[src][dst] for src in range(world)) for dst in range(world)]
    my_off = [sum(allc[src][dst] for src in range(rank)) for dst in range(world)]
    recv_counts = [allc[src][rank] for src in range(world)]
    return total_recv, my_off, recv_counts


def p2p_exchange(engine, sh, rank, world, group=None, stats=None):
    """Fused exchange of a GROUP/COGROUP shuffle: the partition kernel of every rank stores its rows straight
    into the owners' HBM (CUDA IPC peer mappings over NVLink) — see include/vega_b200.h.  torch.distributed only
    carries the control plane: two small all-gathers (counts, IPC handles) and one barrier."""
    import torch
    import torch.distributed as dist
    lib, sc = sh._lib, engine.sc
    t0 = None
    if stats is not None:
        torch.cuda.synchronize()
        import time
        t0 = time.perf_counter()
    counts = (ctypes.c_uint64 * world)()
    L.check(lib.vb_shuffle_export_counts(sh._h, counts))
    counts = [int(c) for c in counts]
    allc = [None] * world
    dist.all_gather_object(allc, counts, group=group)            # allc[src][dst]
    total_recv, my_off, recv_counts = p2p_layout(allc, rank)
    handle = (ctypes.c_ubyte * 64)()
    gen = ctypes.c_uint64()
    L.check(lib.vb_ctx_arena_reserve(sc._h, 16 * max(total_recv[rank], 1), handle, ctypes.byref(gen)))
    allh = [None] * world
    dist.all_gather_object(allh, (bytes(handle), gen.value), group=group)   # doubles as "every arena is reserved"
    for peer, (hb, g) in enumerate(allh):
        buf = (ctypes.c_ubyte * 64).from_buffer_copy(hb)
        L.check(lib.vb_ctx_peer_open(sc._h, peer, buf, g, int(peer == rank)))
    off = (ctypes.c_uint64 * world)(*my_off)
    tot = (ctypes.c_uint64 * world)(*total_recv)
    L.check(lib.vb_shuffle_export_direct(sh._h, off, tot))        # returns when this rank's stores are done
    dist.barrier(group=group)                                     # everybody's rows have landed
    L.check(lib.vb_ctx_arena_release_retired(sc._h))              # every peer re-opened: outgrown arenas can go
    rc = (ctypes.c_uint64 * world)(*recv_counts)
    L.check(lib.vb_shuffle_import_arena(sh._h, rc))
    if stats is not None:
        torch.cuda.synchronize()
        stats["exchange_ms"] = stats.get("exchange_ms", 0.0) + (time.perf_counter() - t0) * 1e3
        stats["sent_rows"] = sum(counts) - counts[rank]
        stats["recv_rows"] = total_recv[rank] - allc[rank][rank]
        stats["exchanges"] = stats.get("exchanges", 0) + 1
        stats["exchange_kind"] = "p2p"


def all_to_all_v(cols, splits, group=None):
    """The shuffle's exchange step over torch.distributed: one all_to_all_single of the stacked counts, then one per
    column.  cols: tensors (None allowed), destination-major along their first dimension; splits[i]: the rows of
    cols[i] for every destination.  Returns (received columns, the rows of each received from every source), both
    source-rank major."""
    import torch
    import torch.distributed as dist
    dev = next(c for c in cols if c is not None).device
    cin = torch.tensor(list(zip(*splits)), dtype=torch.int64, device=dev)      # row d: what d gets of every column
    cout = torch.empty_like(cin)
    dist.all_to_all_single(cout, cin, group=group)
    rsplits = [list(r) for r in zip(*cout.tolist())]                           # rsplits[i][s]: what s sends me

    def a2a(t, sent, got):
        if t is None:
            return None
        out = torch.empty((sum(got), *t.shape[1:]), dtype=t.dtype, device=t.device)
        dist.all_to_all_single(out, t, output_split_sizes=got, input_split_sizes=list(sent), group=group)
        return out
    return [a2a(t, sent, got) for t, sent, got in zip(cols, splits, rsplits)], rsplits


_SUMMED_STATS = ("exchange_ms", "exchanges", "prepare_wall_ms", "counts_wall_ms", "post_wall_ms")


def _exchange(engine, sh, kind, rank, world, group, stats, exchange_device, mode=L.VB_XCHG_NCCL, p2p=False):
    """The exchange step of every run_*shuffle, then the seal.  kind = (the engine class that drives the library,
    export(engine, sh, world) -> (columns, splits), import_(engine, sh, columns, splits), index of the column whose
    counts are the kind's rows in `stats`).  With a communicator on the context the exchange is vb_shuffle_exchange
    (`mode`); otherwise the fused P2P exchange (p2p) or all_to_all_v (exchange_device: stage the columns there, "cpu"
    for a gloo group on a one-GPU box)."""
    cls, export, import_, rows = kind
    if world > 1 and isinstance(engine, cls) and getattr(engine.sc, "comm", None) and exchange_device is None:
        # the product path: count exchange + ONE grouped NCCL send/recv (or the fused P2P scatter) inside
        # libvega_b200, on the library's stream; torch.distributed is not involved
        sh.exchange(mode)
        engine.seal(sh)
        if stats is not None:           # after the seal: reading the event timers synchronises the stream
            for k_, v_ in sh.exchange_stats().items():
                stats[k_] = (stats.get(k_, 0) + v_) if k_ in _SUMMED_STATS else v_
        return sh
    if world > 1 and p2p:
        p2p_exchange(engine, sh, rank, world, group, stats)
    elif world > 1:
        cols, splits = export(engine, sh, world)
        home = cols[rows].device
        if exchange_device is not None:
            cols = [None if c is None else c.to(exchange_device) for c in cols]
        ev = None
        if stats is not None and cols[rows].is_cuda:
            import torch
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        rcols, rsplits = all_to_all_v(cols, splits, group)
        if ev is not None:
            ev[1].record()
            ev[1].synchronize()
            stats["exchange_ms"] = stats.get("exchange_ms", 0.0) + ev[0].elapsed_time(ev[1])
        if exchange_device is not None:
            rcols = [None if c is None else c.to(home) for c in rcols]
        if stats is not None:
            stats["sent_rows"] = sum(splits[rows]) - splits[rows][rank]
            stats["recv_rows"] = sum(rsplits[rows]) - rsplits[rows][rank]
            stats["exchanges"] = stats.get("exchanges", 0) + 1
        import_(engine, sh, rcols, rsplits)
    engine.seal(sh)
    return sh


def _rows_export(engine, sh, world):
    counts, keys, vals = engine.export(sh, world)
    return [keys, vals], [counts, counts]


def _rows_import(engine, sh, cols, splits):
    engine.import_(sh, cols[0], cols[1], splits[0])


def _set_value_order(sh, value_order):
    """vb_shuffle_set_value_order on this rank's handle, before its first map call.  Every rank of a shuffle is expected
    to pass the same order; the library does not check it."""
    if value_order != L.VB_VALORDER_INPUT:
        L.check(sh._lib.vb_shuffle_set_value_order(sh._h, value_order))


def run_shuffle(engine, local_maps, n_map, n_reduce, kcode, vcode, agg, rank, world, group=None, key_width=8, hint=0,
                stats=None, exchange_device=None, p2p=False, value_order=L.VB_VALORDER_INPUT):
    """Map side on this rank's partitions → exchange → reduce side for the partitions this rank owns.

    local_maps: [(map_id, keys, vals_or_None)], ascending map ids from map_block(rank, world, n_map).
    Returns the sealed engine handle; engine.reduce(h, r) is non-empty only for r % world == rank.
    exchange_device: move the packed buffers there for the collective (tests: "cpu" + gloo on a 1-GPU box).
    p2p: GROUP/COGROUP shuffles use the fused partition+send over peer memory instead of pack + all-to-all-v.
    value_order: VB_VALORDER_ASC sorts each key's list of a GROUP/COGROUP shuffle on the rank that owns it.
    """
    if (vcode == L.VB_BYTES) != isinstance(engine, BytesCudaEngine):
        raise TypeError("byte-string values cross ranks with dist.BytesCudaEngine, and it takes byte-string values only")
    if isinstance(engine, BytesCudaEngine):
        _bytes_checks(engine, local_maps, n_map, agg, (L.VB_AGG_GROUP, L.VB_AGG_COGROUP, L.VB_AGG_SORT), rank, world,
                      exchange_device)
    sh = engine.create(n_map, n_reduce, kcode, vcode, agg, rank, world, key_width=key_width, hint=hint)
    _set_value_order(sh, value_order)
    for map_id, keys, vals in local_maps:
        engine.map(sh, map_id, keys, vals)
    p2p = p2p and agg in (L.VB_AGG_GROUP, L.VB_AGG_COGROUP)
    if isinstance(engine, BytesCudaEngine):       # VB_XCHG_AUTO: NCCL, the one exchange of byte-string values
        return _exchange(engine, sh, (BytesCudaEngine, _bytes_export, _bytes_import, 0), rank, world, group, stats,
                         exchange_device, L.VB_XCHG_AUTO)
    return _exchange(engine, sh, (CudaEngine, _rows_export, _rows_import, 0), rank, world, group, stats, exchange_device,
                     L.VB_XCHG_P2P if p2p else L.VB_XCHG_NCCL, p2p and isinstance(engine, CudaEngine))


class StrCudaEngine:
    """libvega_b200 on this rank's GPU, for String keys: CudaEngine's calls over vb_shuffle_create_str_dist.
    export gives ((n_keys, n_key_bytes, n_vals) per destination, (key_lens, key_bytes, val_counts, vals)), the wire
    columns of include/vega_b200.h (val_counts None for reduce ops); import_ takes the same shape, source-rank major.
    agg VB_AGG_SORT is sort_by_key (vb_shuffle_create_str_sort_dist; vcode None: key-only): reduce then gives
    (key offsets, key bytes, payload or None), one key per row, and the exchange needs the library's communicator.
    key_kind VB_STRKEY_BYTES places keys as Rust hashes a Vec<u8> (vb_shuffle_set_str_key); every rank must pass the
    same kind (a reduce op's exchange inside the library refuses a rank that differs; a GROUP exchange cannot tell)."""

    def __init__(self, sc, key_kind=L.VB_STRKEY_STR):
        self.sc, self.key_kind = sc, key_kind

    def create(self, n_map, n_reduce, vcode, agg, rank, world, hint=0):
        return StrShuffle(self.sc, n_map, n_reduce, vcode, agg, hint=hint, rank=rank, world=world, sort=agg == L.VB_AGG_SORT,
                          key_kind=self.key_kind)

    def map(self, sh, map_id, keys, vals):
        """keys: a StrKeys column or a sequence of str; vals: a numpy array or torch CUDA tensor (None for count)."""
        k = keys if isinstance(keys, _StrCol) else _StrCol(keys)
        v = None if vals is None else (vals if isinstance(vals, _Col) else _Col(vals, role="value"))
        sh.map(map_id, k, v, 0, k.n)

    def export(self, sh, world):
        return sh.export()

    def import_(self, sh, cols, counts):
        sh.import_(*cols, *counts)

    def seal(self, sh):
        sh.seal()

    def reduce(self, sh, r):
        return sh.reduce_raw(r) if sh.agg == L.VB_AGG_SORT else sh.reduce(r)


def _str_export(engine, sh, world):
    (n_keys, n_key_bytes, n_vals), cols = engine.export(sh, world)
    return list(cols), [n_keys, n_key_bytes, n_keys, n_vals]     # key lengths, key bytes, value counts, values


def _str_import(engine, sh, cols, splits):
    engine.import_(sh, tuple(cols), (splits[0], splits[1], splits[3]))


def run_str_shuffle(engine, local_maps, n_map, n_reduce, vcode, agg, rank, world, group=None, hint=0, stats=None,
                    exchange_device=None, value_order=L.VB_VALORDER_INPUT):
    """run_shuffle for String keys: map side on this rank's partitions → exchange → reduce side for the partitions
    this rank owns.  local_maps: [(map_id, keys, vals_or_None)], ascending map ids from map_block(rank, world, n_map).
    With a communicator on the context the exchange is vb_shuffle_exchange (NCCL inside the library); otherwise
    all_to_all_v of the four columns (exchange_device: "cpu" for a gloo group on a one-GPU box).  agg VB_AGG_SORT
    (sort_by_key) across ranks has no such fallback: its cut keys are agreed in rounds of the library's collectives.
    value_order as for run_shuffle (GROUP only)."""
    if (vcode == L.VB_BYTES) != isinstance(engine, StrBytesCudaEngine):
        raise TypeError("byte-string values cross ranks with dist.StrBytesCudaEngine, and it takes byte-string values only")
    if isinstance(engine, StrBytesCudaEngine):
        _bytes_checks(engine, local_maps, n_map, agg, (L.VB_AGG_GROUP, L.VB_AGG_SORT), rank, world, exchange_device)
        sh = engine.create(n_map, n_reduce, vcode, agg, rank, world, hint=hint)
        _set_value_order(sh, value_order)
        for map_id, keys, vals in local_maps:
            engine.map(sh, map_id, keys, vals)
        return _exchange(engine, sh, (StrBytesCudaEngine, _str_bytes_export, _str_bytes_import, 3), rank, world, group, stats,
                         exchange_device, L.VB_XCHG_AUTO)
    if agg == L.VB_AGG_SORT and world > 1 and not (isinstance(engine, StrCudaEngine) and getattr(engine.sc, "comm", None)
                                                   and exchange_device is None):
        raise ValueError("sort_by_key over String keys across ranks needs the library's communicator (vb_ctx_comm_init, "
                         "Context.comm_init) and runs its exchange inside the library")
    sh = engine.create(n_map, n_reduce, vcode, agg, rank, world, hint=hint)
    _set_value_order(sh, value_order)
    for map_id, keys, vals in local_maps:
        engine.map(sh, map_id, keys, vals)
    return _exchange(engine, sh, (StrCudaEngine, _str_export, _str_import, 3), rank, world, group, stats, exchange_device)


class CombineCudaEngine:
    """libvega_b200 on this rank's GPU, for combine_by_key: CudaEngine's calls over vb_shuffle_create_multi_dist.
    multi is Shuffle's (value column dtype codes, [(vb_agg, column), ...]).  export gives (counts per destination, keys,
    accs), accs an (n_acc, rows) view, the wire columns of include/vega_b200.h; import_ takes the same, source-rank major."""

    def __init__(self, sc):
        self.sc = sc

    def create(self, n_map, n_reduce, kcode, multi, rank, world, key_width=8, hint=0):
        return Shuffle.combine_dist(self.sc, n_map, n_reduce, kcode, multi, rank, world, key_width=key_width, hint=hint)

    def map(self, sh, map_id, keys, cols):
        """keys and every value column: numpy arrays or torch CUDA tensors of one location."""
        k = keys if isinstance(keys, _Col) else _Col(keys)
        cs = tuple(c if isinstance(c, _Col) else _Col(c, role="value") for c in cols)
        sh.map_cols(map_id, k, cs, 0, k.n)

    def export(self, sh, world):
        return sh.export_cols()

    def import_(self, sh, keys, accs, counts):
        sh.import_cols(keys, accs, counts)

    def seal(self, sh):
        sh.seal()

    def reduce(self, sh, r, out_dtypes):
        return sh.reduce_cols(r, out_dtypes)


def _combine_pack(counts, keys, accs):
    """keys[rows] and accs[n_acc][rows] as one [rows][1 + n_acc] column: one all_to_all_single carries every row."""
    import torch
    return [torch.cat([keys.view(-1, 1), accs.t()], dim=1).contiguous()], [counts]


def _combine_unpack(cols, splits):
    """The received [rows][1 + n_acc] column as (keys[rows], accs[n_acc][rows], rows from every source)."""
    return cols[0][:, 0].contiguous(), cols[0][:, 1:].t().contiguous(), splits[0]


def _combine_export(engine, sh, world):
    return _combine_pack(*engine.export(sh, world))


def _combine_import(engine, sh, cols, splits):
    engine.import_(sh, *_combine_unpack(cols, splits))


def run_combine_shuffle(engine, local_maps, n_map, n_reduce, kcode, multi, rank, world, group=None, key_width=8, hint=0,
                        stats=None, exchange_device=None):
    """run_shuffle for combine_by_key: map side on this rank's partitions → exchange → reduce side for the partitions
    this rank owns.  local_maps: [(map_id, keys, value columns)], ascending map ids from map_block(rank, world, n_map).
    With a communicator on the context the exchange is vb_shuffle_exchange (NCCL inside the library); otherwise
    all_to_all_v of the rows, each the key and its n_acc partials (exchange_device: "cpu" for a gloo group on a one-GPU
    box)."""
    if not 0 <= rank < world <= 256:
        raise ValueError(f"rank {rank} of world {world}: 0 <= rank < world <= 256")
    lo, hi = map_block(rank, world, n_map)
    ids = [m for m, _, _ in local_maps]
    if any(not lo <= m < hi for m in ids) or ids != sorted(set(ids)):
        raise ValueError(f"rank {rank} runs map tasks {ids}: ascending ids in its block [{lo}, {hi}) expected")
    sh = engine.create(n_map, n_reduce, kcode, multi, rank, world, key_width=key_width, hint=hint)
    for map_id, keys, cols in local_maps:
        engine.map(sh, map_id, keys, cols)
    return _exchange(engine, sh, (CombineCudaEngine, _combine_export, _combine_import, 0), rank, world, group, stats,
                     exchange_device)


class StrCombineCudaEngine:
    """libvega_b200 on this rank's GPU, for combine_by_key over String keys: CudaEngine's calls over
    vb_shuffle_create_str_multi_dist.  multi is StrShuffle's (value column dtype codes, [(vb_agg, column), ...]).  export
    gives ((n_keys, n_key_bytes) per destination, (key_lens, key_bytes, accs)), accs an (n_acc, keys) view, the wire
    columns of include/vega_b200.h; import_ takes the same shape, source-rank major.  key_kind: as StrCudaEngine's."""

    def __init__(self, sc, key_kind=L.VB_STRKEY_STR):
        self.sc, self.key_kind = sc, key_kind

    def create(self, n_map, n_reduce, multi, rank, world, hint=0):
        return StrShuffle(self.sc, n_map, n_reduce, L.VB_U64, L.VB_AGG_SUM, hint=hint, rank=rank, world=world, multi=multi,
                          key_kind=self.key_kind)

    def map(self, sh, map_id, keys, cols):
        """keys: a StrKeys column or a sequence of str; cols: the value columns (numpy arrays or torch CUDA tensors of
        the keys' location)."""
        k = keys if isinstance(keys, _StrCol) else _StrCol(keys)
        cs = tuple(c if isinstance(c, _Col) else _Col(c, role="value") for c in cols)
        sh.map_cols(map_id, k, cs, 0, k.n)

    def export(self, sh, world):
        return sh.export_cols()

    def import_(self, sh, cols, counts):
        sh.import_cols(*cols, *counts)

    def seal(self, sh):
        sh.seal()

    def reduce(self, sh, r, out_dtypes):
        return sh.reduce_cols(r, out_dtypes)


def _str_combine_export(engine, sh, world):
    """The accumulators travel as one [keys][n_acc] column beside the key lengths and bytes."""
    (n_keys, n_key_bytes), (lens, data, accs) = engine.export(sh, world)
    return [lens, data, accs.t().contiguous()], [n_keys, n_key_bytes, n_keys]


def _str_combine_import(engine, sh, cols, splits):
    engine.import_(sh, (cols[0], cols[1], cols[2].t().contiguous()), (splits[0], splits[1]))


def run_str_combine_shuffle(engine, local_maps, n_map, n_reduce, multi, rank, world, group=None, hint=0, stats=None,
                            exchange_device=None):
    """run_shuffle for combine_by_key over String keys: map side on this rank's partitions → exchange → reduce side for
    the partitions this rank owns.  local_maps: [(map_id, keys, value columns)], ascending map ids from
    map_block(rank, world, n_map).  With a communicator on the context the exchange is vb_shuffle_exchange (NCCL inside
    the library); otherwise all_to_all_v of the key lengths, key bytes and the [keys][n_acc] partials (exchange_device:
    "cpu" for a gloo group on a one-GPU box)."""
    if not 0 <= rank < world <= 256:
        raise ValueError(f"rank {rank} of world {world}: 0 <= rank < world <= 256")
    lo, hi = map_block(rank, world, n_map)
    ids = [m for m, _, _ in local_maps]
    if any(not lo <= m < hi for m in ids) or ids != sorted(set(ids)):
        raise ValueError(f"rank {rank} runs map tasks {ids}: ascending ids in its block [{lo}, {hi}) expected")
    sh = engine.create(n_map, n_reduce, multi, rank, world, hint=hint)
    for map_id, keys, cols in local_maps:
        engine.map(sh, map_id, keys, cols)
    return _exchange(engine, sh, (StrCombineCudaEngine, _str_combine_export, _str_combine_import, 0), rank, world, group,
                     stats, exchange_device)


class BytesCudaEngine:
    """libvega_b200 on this rank's GPU, for byte-string values with integer keys: CudaEngine's calls over
    Shuffle.bytes_dist (vb_shuffle_create_bytes_dist; GROUP, COGROUP or SORT).  map takes the values as a sequence of str
    or bytes, or a StrKeys column.  export gives ((counts, n_val_bytes) per destination, (keys, val_lens, val_bytes)),
    the wire columns of include/vega_b200.h; import_ takes the same shape, source-rank major.  reduce gives references;
    gather them with sh.gather."""

    def __init__(self, sc):
        self.sc = sc

    def create(self, n_map, n_reduce, kcode, vcode, agg, rank, world, key_width=8, hint=0):
        return Shuffle.bytes_dist(self.sc, n_map, n_reduce, kcode, agg, rank, world, key_width=key_width, hint=hint)

    def map(self, sh, map_id, keys, vals):
        k = keys if isinstance(keys, _Col) else _Col(keys)
        v = vals if isinstance(vals, _BytesCol) else _BytesCol(vals)
        if v.n != k.n:
            raise ValueError(f"map task {map_id}: {k.n} keys and {v.n} values")
        sh.map(map_id, k, v, 0, k.n)

    def export(self, sh, world):
        return sh.export_bytes()

    def import_(self, sh, cols, counts):
        sh.import_bytes(*cols, *counts)

    def seal(self, sh):
        sh.seal()

    def reduce(self, sh, r):
        return sh.reduce(r)


class StrBytesCudaEngine:
    """libvega_b200 on this rank's GPU, for byte-string values with String keys: StrCudaEngine's calls over
    StrShuffle.bytes_dist (GROUP, or SORT: sort_by_key with a byte-string payload).  map takes str keys (or a StrKeys
    column) and the values as BytesCudaEngine does.  export gives ((n_keys, n_key_bytes, n_vals, n_val_bytes) per
    destination, (key_lens, key_bytes, val_counts, val_lens, val_bytes)); import_ takes the same shape, source-rank major.
    reduce gives references (raw: key offsets and bytes); gather them with sh.gather.  key_kind: as StrCudaEngine's."""

    def __init__(self, sc, key_kind=L.VB_STRKEY_STR):
        self.sc, self.key_kind = sc, key_kind

    def create(self, n_map, n_reduce, vcode, agg, rank, world, hint=0):
        return StrShuffle.bytes_dist(self.sc, n_map, n_reduce, rank, world, sort=agg == L.VB_AGG_SORT, hint=hint,
                                     key_kind=self.key_kind)

    def map(self, sh, map_id, keys, vals):
        if not isinstance(keys, (_StrCol, StrKeys)) and len(keys) and not _is_str_keys(keys):
            raise TypeError("String keys: a sequence of str or a StrKeys column")
        k = keys if isinstance(keys, _StrCol) else _StrCol(keys)
        v = vals if isinstance(vals, _BytesCol) else _BytesCol(vals)
        if v.n != k.n:
            raise ValueError(f"map task {map_id}: {k.n} keys and {v.n} values")
        sh.map(map_id, k, v, 0, k.n)

    def export(self, sh, world):
        return sh.export_bytes()

    def import_(self, sh, cols, counts):
        sh.import_bytes(*cols, *counts)

    def seal(self, sh):
        sh.seal()

    def reduce(self, sh, r):
        return sh.reduce_raw(r)


def _bytes_checks(engine, local_maps, n_map, agg, aggs, rank, world, exchange_device):
    """The bytes engines' refusals, before any device work: an op that computes on values (TypeError), a rank outside
    the world, map ids outside the rank's block, or a sort without the library's communicator (ValueError)."""
    if agg not in aggs:
        raise TypeError(f"agg {agg} computes on values: byte-string values cross ranks for group_by_key, cogroup, the joins "
                        "and sort_by_key")
    if not 0 <= rank < world <= 256:
        raise ValueError(f"rank {rank} of world {world}: 0 <= rank < world <= 256")
    lo, hi = map_block(rank, world, n_map)
    ids = [m for m, _, _ in local_maps]
    if any(not lo <= m < hi for m in ids) or ids != sorted(set(ids)):
        raise ValueError(f"rank {rank} runs map tasks {ids}: ascending ids in its block [{lo}, {hi}) expected")
    if agg == L.VB_AGG_SORT and world > 1 and not (getattr(engine.sc, "comm", None) and exchange_device is None):
        raise ValueError("sort_by_key with byte-string values across ranks needs the library's communicator "
                         "(Context.comm_init) and runs its exchange inside the library")


def _bytes_export(engine, sh, world):
    (counts, n_val_bytes), cols = engine.export(sh, world)
    return list(cols), [counts, counts, n_val_bytes]         # keys, value lengths, value bytes


def _bytes_import(engine, sh, cols, splits):
    engine.import_(sh, tuple(cols), (splits[0], splits[2]))


def _str_bytes_export(engine, sh, world):
    (n_keys, n_key_bytes, n_vals, n_val_bytes), cols = engine.export(sh, world)
    # key lengths, key bytes, value counts, value lengths, value bytes
    return list(cols), [n_keys, n_key_bytes, n_keys, n_vals, n_val_bytes]


def _str_bytes_import(engine, sh, cols, splits):
    engine.import_(sh, tuple(cols), (splits[0], splits[1], splits[3], splits[4]))


def owned_partitions(rank, world, n_reduce):
    return [r for r in range(n_reduce) if r % world == rank]
