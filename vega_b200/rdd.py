"""Host-side mirror of vega's operator API for the shuffle path, above the C ABI.

Same names and argument meaning as the reference for the calls on the path
(src/context.rs `Context::parallelize/make_rdd`, src/rdd/pair_rdd.rs
`group_by_key / reduce_by_key / join / cogroup / partition_by_key`, src/rdd/rdd.rs
`count_by_value / distinct / collect`), so the parity tests read like tests/test_pair_rdd.rs.
Differences forced by the boundary (SURVEY.md F4): rows are 64-bit POD (K,V) arrays
(numpy on the host or torch CUDA tensors), and `reduce_by_key` takes a *named* op
("sum" | "min" | "max") because a closure cannot cross into CUDA.  Keys may also be Rust `String`s: a
sequence of Python `str` or a `StrKeys` column (offsets + UTF-8 bytes), for reduce_by_key / count_by_key /
group_by_key / partition_by_key / combine_by_key / count_by_value / distinct; they are placed as the reference places
`String` keys.  sort_by_key / sort over them go through StrSortedRdd, which orders the keys by their bytes on the device.
Values may be byte strings (a sequence of str or bytes, or a StrKeys column) for the ops that move values without
reading them: group_by_key / partition_by_key / join / the outer joins / cogroup / CoGroupedRdd / sort_by_key, and over
String keys StrPairRdd.group_by_key / partition_by_key, StrCoGroupedRdd and StrSortedRdd.  They travel through the
shuffle as references and are gathered back into bytes on the device; they come back as numpy object arrays of str (or
bytes, as given), with None for the missing side of an outer join.

All compute happens in libvega_b200.so; this module slices the input exactly like
ParallelCollection::slice, drives map tasks → seal → reduce tasks like the scheduler does
(base_scheduler.rs:377-455), and concatenates partitions in order (rdd.rs:420-434).
"""
import ctypes
import itertools
import weakref

import numpy as np

from . import _lib as L

_AGG = {"group": L.VB_AGG_GROUP, "sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX,
        "count": L.VB_AGG_COUNT, "cogroup": L.VB_AGG_COGROUP, "sort": L.VB_AGG_SORT}
_NP_OF = {L.VB_U64: np.uint64, L.VB_I64: np.int64, L.VB_F64: np.float64, L.VB_BYTES: np.uint64}   # VB_BYTES: references
_COMBINE_OPS = {"sum": L.VB_AGG_SUM, "min": L.VB_AGG_MIN, "max": L.VB_AGG_MAX, "count": L.VB_AGG_COUNT, "mean": L.VB_AGG_MEAN}


def _is_torch(x):
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda")


def _sync_torch(*tensors):
    """The library runs on its own stream: pending torch work on buffers it is about to touch must be done
    (torch's caching allocator may hand out memory whose previous user is still running on torch's stream)."""
    for t in tensors:
        if t is not None and _is_torch(t) and t.is_cuda:
            import torch
            torch.cuda.current_stream(t.device).synchronize()
            return


class _Col:
    """One 64-bit column (or an (n,2) AoS row block): pointer + location + dtype code."""

    def __init__(self, x, allow_rows=False, role="key"):
        self.key_width = 8
        self.rows = False
        if _is_torch(x):
            import torch
            if not x.is_contiguous():
                x = x.contiguous()
            code = {torch.int64: L.VB_I64, torch.float64: L.VB_F64}.get(x.dtype)
            if code is None and hasattr(torch, "uint64") and x.dtype == torch.uint64:
                code = L.VB_U64
            if code is None:
                raise TypeError(f"unsupported tensor dtype {x.dtype}")
            self.loc = L.VB_DEVICE_BORROWED if x.is_cuda else L.VB_HOST
            if x.is_cuda:
                # the library launches on its own stream: whatever produced this tensor on torch's stream must be done
                torch.cuda.current_stream(x.device).synchronize()
            self.ptr = x.data_ptr()
            shape = tuple(x.shape)
        else:
            x = np.asarray(x)
            if x.dtype in (np.int32, np.uint32):
                self.key_width = 4          # Rust i32/u32 keys hash as 4 LE bytes
                x = x.astype(np.int64 if x.dtype.kind == "i" else np.uint64)
            elif x.dtype in (np.int16, np.uint16, np.int8, np.uint8) or x.dtype.kind == "b":
                # Rust hashes i16 as 2 bytes and i8/u8/bool as 1: the library has 4- and 8-byte key hashes only,
                # so narrow KEYS would be placed differently from the reference's HashPartitioner — refuse them.
                if role == "key":
                    raise TypeError(f"key dtype {x.dtype}: only 32- and 64-bit integer keys hash like the reference's")
                x = x.astype(np.int64 if x.dtype.kind == "i" else np.uint64)
            code = {"u": L.VB_U64, "i": L.VB_I64, "f": L.VB_F64}.get(x.dtype.kind)
            if code is None or x.dtype.itemsize != 8:
                raise TypeError(f"unsupported dtype {x.dtype}")
            x = np.ascontiguousarray(x)
            self.loc = L.VB_HOST
            self.ptr = x.ctypes.data
            shape = x.shape
        if len(shape) == 2 and shape[1] == 2 and allow_rows:
            self.rows = True
        elif len(shape) != 1:
            raise ValueError(f"expected a 1-D column{' or (n,2) rows' if allow_rows else ''}, got shape {shape}")
        self.n = shape[0]
        self.code = code
        self.owner = x

    def at(self, start):
        return ctypes.c_void_p(self.ptr + start * (16 if self.rows else 8)) if self.n else None


def slice_starts(n, num_slices):
    """ParallelCollection::slice boundaries (parallel_collection_rdd.rs:116-145) via the C ABI."""
    buf = np.zeros(min(n, num_slices) + 2, dtype=np.uint64)
    k = L.lib().vb_slice(n, num_slices, buf.ctypes.data)
    if k == 0:
        raise ValueError("Number of slices should be greater than or equal to 1")
    return buf[: k + 1].astype(np.int64)


class Context:
    """vega::Context for the shuffle path (src/context.rs:333-473): owns the device context
    and hands out shuffle ids (`new_shuffle_id`)."""

    def __init__(self, device=0, profile=False):
        self._lib = L.lib()
        h = ctypes.c_void_p()
        L.check(self._lib.vb_ctx_create(device, ctypes.byref(h)))
        self._h = h
        self._ids = itertools.count()
        self._shuffles = weakref.WeakSet()      # live shuffles are freed before the context goes away
        self.comm = None
        if profile:
            self.set_profile(True)

    @staticmethod
    def new(device=0):
        return Context(device)

    def set_profile(self, on):
        L.check(self._lib.vb_ctx_set_profile(self._h, int(bool(on))))

    def new_shuffle_id(self):
        return next(self._ids)

    def synchronize(self):
        L.check(self._lib.vb_ctx_synchronize(self._h))

    def stream(self):
        """The context's CUDA stream as a torch.cuda.ExternalStream (event timing in bench.py)."""
        import torch
        dev = self._lib.vb_ctx_device(self._h)
        return torch.cuda.ExternalStream(self._lib.vb_ctx_stream(self._h), device=f"cuda:{dev}")

    def mem_info(self):
        r, h = ctypes.c_uint64(), ctypes.c_uint64()
        L.check(self._lib.vb_ctx_mem_info(self._h, ctypes.byref(r), ctypes.byref(h)))
        return r.value, h.value

    def parallelize(self, data, num_slices, values=None):
        """`sc.parallelize(vec, num_slices)`.  data: 1-D keys (→ Rdd), (n,2) rows or
        (keys, values) (→ PairRdd).  values may also be a tuple of up to 4 value columns (combine_by_key), or byte-string
        values: a sequence or numpy array of str (returned as str), a sequence of bytes (returned as bytes) or a StrKeys
        column on the host or as CUDA tensors (returned as str).
        String keys (a sequence of str, a numpy str array or a StrKeys column) give a StrRdd / StrPairRdd; a tuple of
        value columns gives a StrPairRdd with value columns, the one kind whose combine_by_key runs."""
        if _is_bytes_vals(values):
            vals = _BytesCol(values)
            if _is_str_keys(data):
                return StrPairRdd(self, _StrCol(data), vals, num_slices)
            return PairRdd(self, _Col(data), vals, num_slices)
        if _is_str_keys(data):
            keys = _StrCol(data)
            if values is None:
                return StrRdd(self, keys, num_slices)
            if isinstance(values, tuple) and values and all(_is_torch(v) or np.ndim(v) >= 1 for v in values):
                if not 1 <= len(values) <= L.VB_MAX_VAL_COLS:
                    raise ValueError(f"{len(values)} value columns: 1 to {L.VB_MAX_VAL_COLS} are supported")
                cols = tuple(_Col(v, role="value") for v in values)
                return StrPairRdd(self, keys, cols[0] if len(cols) == 1 else None, num_slices, cols=cols)
            return StrPairRdd(self, keys, _Col(values, role="value"), num_slices)
        if values is None and isinstance(data, tuple) and len(data) == 2 and _is_str_keys(data[0]):
            return StrPairRdd(self, _StrCol(data[0]), _Col(data[1], role="value"), num_slices)
        if isinstance(values, tuple):                 # a list stays one value column, as before
            if not 1 <= len(values) <= L.VB_MAX_VAL_COLS:
                raise ValueError(f"{len(values)} value columns: 1 to {L.VB_MAX_VAL_COLS} are supported")
            cols = tuple(_Col(v, role="value") for v in values)
            return PairRdd(self, _Col(data), cols[0] if len(cols) == 1 else None, num_slices, cols=cols)
        if values is not None:
            return PairRdd(self, _Col(data), _Col(values, role="value"), num_slices)
        if isinstance(data, tuple) and len(data) == 2:
            return PairRdd(self, _Col(data[0]), _Col(data[1], role="value"), num_slices)
        col = _Col(data, allow_rows=True)
        if col.rows:
            return PairRdd(self, col, None, num_slices)
        return Rdd(self, col, num_slices)

    make_rdd = parallelize

    def range(self, start, end, step, num_slices):
        """`sc.range(start, end, step, num_slices)` (src/context.rs:419-431): (start..=end).step_by(step), generated
        ON the device (vb_range) — a source RDD with no host array and no H2D copy."""
        import torch
        n = self._lib.vb_range_len(start, end, step)
        dev = f"cuda:{self._lib.vb_ctx_device(self._h)}"
        t = torch.empty(n, dtype=torch.int64, device=dev)
        torch.cuda.current_stream(t.device).synchronize()
        L.check(self._lib.vb_range(self._h, ctypes.c_void_p(t.data_ptr()) if n else None, start, end, step))
        col = _Col(t)
        col.code = L.VB_U64
        return Rdd(self, col, num_slices)

    def gen_pairs(self, out_rows=None, out_keys=None, out_vals=None, first=0, n=0, mode="uniform", n_distinct=1,
                  rank_base=0, seed_k=1, seed_v=2, zipf_s=0.0):
        """Fill device buffers (torch CUDA tensors) with the synthetic workload of SURVEY.md §8(d)."""
        m = {"uniform": L.VB_GEN_UNIFORM, "zipf": L.VB_GEN_ZIPF, "unique": L.VB_GEN_UNIQUE}[mode]
        _sync_torch(out_rows, out_keys, out_vals)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        L.check(self._lib.vb_gen_pairs(self._h, p(out_rows), p(out_keys), p(out_vals), first, n, m, n_distinct,
                                       rank_base, seed_k, seed_v, float(zipf_s)))

    def trim(self, keep_bytes=0):
        """Return pool memory beyond keep_bytes to the device."""
        L.check(self._lib.vb_ctx_trim(self._h, keep_bytes))

    # ---- one-process-per-GPU: the NCCL communicator lives inside the library ------------------
    def comm_init(self, rank, world, unique_id=None, group=None):
        """Collective.  unique_id: the 128 bytes from `Context.comm_unique_id()` on rank 0, handed to every
        rank by any host-side bootstrap; if None, torch.distributed (already initialised) broadcasts it —
        torch is then used for this bootstrap only, the exchange itself runs inside libvega_b200."""
        if unique_id is None:
            import torch.distributed as dist
            box = [self.comm_unique_id() if rank == 0 else None]
            dist.broadcast_object_list(box, src=0, group=group)
            unique_id = box[0]
        buf = (ctypes.c_ubyte * L.VB_UNIQUE_ID_BYTES).from_buffer_copy(unique_id)
        L.check(self._lib.vb_ctx_comm_init(self._h, buf, rank, world))
        self.comm = (rank, world)

    def comm_unique_id(self):
        buf = (ctypes.c_ubyte * L.VB_UNIQUE_ID_BYTES)()
        L.check(self._lib.vb_comm_unique_id(buf))
        return bytes(buf)

    def comm_destroy(self):
        if getattr(self, "comm", None):
            L.check(self._lib.vb_ctx_comm_destroy(self._h))
            self.comm = None

    def close(self):
        if self._h:
            for sh in list(self._shuffles):
                sh.free()
            self._lib.vb_ctx_destroy(self._h)      # collective when a communicator exists
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class Shuffle:
    """Thin RAII wrapper of one vb_shuf (== one ShuffleDependency / shuffle_id)."""

    def __init__(self, sc, n_map, n_reduce, kcode, vcode, agg, key_width=8, hint=0, rank=0, world=1, multi=None,
                 value_order=L.VB_VALORDER_INPUT):
        """multi: (value column dtype codes, [(vb_agg, column), ...]) for a vb_shuffle_create_multi shuffle.
        value_order: VB_VALORDER_ASC sorts each key's list of a GROUP / COGROUP shuffle ascending on the device
        (vb_shuffle_set_value_order)."""
        self.sc, self._lib = sc, sc._lib
        self.n_map, self.n_reduce, self.agg, self.vcode, self.kcode = n_map, n_reduce, agg, vcode, kcode
        self.has_payload = True
        self._keepalive = []      # owners of VB_DEVICE_BORROWED inputs: the library reads them until seal
        h = ctypes.c_void_p()
        if multi is not None:
            codes, aggs = multi
            dts = (ctypes.c_int32 * len(codes))(*codes)
            spec = (L.vb_agg_col * len(aggs))(*[L.vb_agg_col(a, c) for a, c in aggs])
            L.check(self._lib.vb_shuffle_create_multi(sc._h, sc.new_shuffle_id(), n_map, n_reduce, kcode, len(codes), dts,
                                                      len(aggs), spec, ctypes.byref(h)))
        else:
            part = L.VB_PART_RANGE if agg == L.VB_AGG_SORT else L.VB_PART_HASH_METRO64
            L.check(self._lib.vb_shuffle_create(sc._h, sc.new_shuffle_id(), n_map, n_reduce, kcode, vcode, agg, part, ctypes.byref(h)))
        self._h = h
        sc._shuffles.add(self)
        if key_width != 8:
            L.check(self._lib.vb_shuffle_set_key_width(h, key_width))
        if hint:
            L.check(self._lib.vb_shuffle_set_hint(h, hint))
        if world > 1:
            L.check(self._lib.vb_shuffle_set_dist(h, rank, world))
        if value_order != L.VB_VALORDER_INPUT:
            L.check(self._lib.vb_shuffle_set_value_order(h, value_order))

    @classmethod
    def combine_dist(cls, sc, n_map, n_reduce, kcode, multi, rank, world, key_width=8, hint=0):
        """vb_shuffle_create_multi_dist: the multi-aggregate shuffle `multi` (as for Shuffle) on rank `rank` of `world`.
        Exchange it with export_cols / import_cols, or with exchange() when the context has a communicator."""
        self = cls.__new__(cls)
        self.sc, self._lib = sc, sc._lib
        self.n_map, self.n_reduce, self.agg, self.vcode, self.kcode = n_map, n_reduce, L.VB_AGG_SUM, L.VB_U64, kcode
        self.rank, self.world = rank, world
        self.has_payload, self._keepalive = True, []
        codes, aggs = multi
        dts = (ctypes.c_int32 * len(codes))(*codes)
        spec = (L.vb_agg_col * len(aggs))(*[L.vb_agg_col(a, c) for a, c in aggs])
        h = ctypes.c_void_p()
        L.check(self._lib.vb_shuffle_create_multi_dist(sc._h, sc.new_shuffle_id(), n_map, n_reduce, kcode, len(codes), dts,
                                                       len(aggs), spec, rank, world, ctypes.byref(h)))
        self._h = h
        sc._shuffles.add(self)
        if key_width != 8:
            L.check(self._lib.vb_shuffle_set_key_width(h, key_width))
        if hint:
            L.check(self._lib.vb_shuffle_set_hint(h, hint))
        return self

    def export_cols(self):
        """vb_shuffle_export_cols_prepare + buffers (combine_dist, world > 1): (counts, keys, accs).  counts has one entry
        per destination rank; keys (int64, rows) and accs (int64, (n_acc, rows)) are torch views of the library's device
        buffers, destination-major, in the wire format of include/vega_b200.h and valid until seal."""
        import torch
        cnt = (ctypes.c_uint64 * self.world)()
        L.check(self._lib.vb_shuffle_export_cols_prepare(self._h, cnt))
        counts = [int(x) for x in cnt]
        kp, ap, na = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint32()
        L.check(self._lib.vb_shuffle_export_cols_buffers(self._h, ctypes.byref(kp), ctypes.byref(ap), ctypes.byref(na)))
        dev = f"cuda:{self._lib.vb_ctx_device(self.sc._h)}"
        n, A = sum(counts), na.value
        if n == 0:
            return counts, torch.empty(0, dtype=torch.int64, device=dev), torch.empty((A, 0), dtype=torch.int64, device=dev)
        keys = torch.as_tensor(_DevView(kp.value, n, "<i8"), device=dev)
        accs = torch.as_tensor(_DevView(ap.value, A * n, "<i8"), device=dev).view(A, n)
        return counts, keys, accs

    def import_cols(self, keys, accs, counts):
        """vb_shuffle_import_cols: the received keys (rows) and accumulators ((n_acc, rows), both torch CUDA tensors,
        source-rank major) and the row count every source rank sent.  The tensors are kept alive until seal."""
        import torch
        if accs.dim() != 2 or accs.shape[1] != keys.numel() or len(counts) != self.world or sum(counts) != keys.numel():
            raise ValueError(f"import of {keys.numel()} keys, accumulators of shape {tuple(accs.shape)} and counts {list(counts)} "
                             f"on a world of {self.world}: (n_acc, keys) accumulators and one count per rank expected")
        accs = accs.contiguous()
        if keys.is_cuda:
            torch.cuda.current_stream(keys.device).synchronize()       # the library reads on its own stream
        self._keepalive.append((keys, accs))
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
        L.check(self._lib.vb_shuffle_import_cols(self._h, p(keys), p(accs), accs.shape[0], (ctypes.c_uint64 * len(counts))(*counts)))

    @classmethod
    def bytes_dist(cls, sc, n_map, n_reduce, kcode, agg, rank, world, key_width=8, hint=0):
        """vb_shuffle_create_bytes_dist: a GROUP / COGROUP / SORT shuffle of byte-string values on rank `rank` of `world`.
        Map it with byte-string values (a _BytesCol); exchange it with export_bytes / import_bytes (GROUP and COGROUP), or
        with exchange() when the context has a communicator.  Its results are references, gathered with gather()."""
        self = cls.__new__(cls)
        self.sc, self._lib = sc, sc._lib
        self.n_map, self.n_reduce, self.agg, self.vcode, self.kcode = n_map, n_reduce, agg, L.VB_BYTES, kcode
        self.rank, self.world = rank, world
        self.has_payload, self._keepalive = True, []
        part = L.VB_PART_RANGE if agg == L.VB_AGG_SORT else L.VB_PART_HASH_METRO64
        h = ctypes.c_void_p()
        L.check(self._lib.vb_shuffle_create_bytes_dist(sc._h, sc.new_shuffle_id(), n_map, n_reduce, kcode, agg, part, rank, world,
                                                       ctypes.byref(h)))
        self._h = h
        sc._shuffles.add(self)
        if key_width != 8:
            L.check(self._lib.vb_shuffle_set_key_width(h, key_width))
        if hint:
            L.check(self._lib.vb_shuffle_set_hint(h, hint))
        return self

    def export_bytes(self):
        """vb_shuffle_export_bytes_prepare + buffers (bytes_dist, world > 1): ((counts, n_val_bytes), (keys, val_lens,
        val_bytes)).  The counts are lists with one entry per destination rank; the columns are torch views of the
        library's device buffers (int64 keys, int32 value lengths, uint8 value bytes), destination-major, valid until seal."""
        W = self.world
        cnt, nvb = (ctypes.c_uint64 * W)(), (ctypes.c_uint64 * W)()
        L.check(self._lib.vb_shuffle_export_bytes_prepare(self._h, cnt, nvb))
        counts = ([int(x) for x in cnt], [int(x) for x in nvb])
        ptrs = [ctypes.c_void_p() for _ in range(3)]
        L.check(self._lib.vb_shuffle_export_bytes_buffers(self._h, *[ctypes.byref(p) for p in ptrs]))
        n, b = sum(counts[0]), sum(counts[1])
        return counts, (_dev_view(self, ptrs[0], n, "<i8"), _dev_view(self, ptrs[1], n, "<i4"), _dev_view(self, ptrs[2], b, "|u1"))

    def import_bytes(self, keys, val_lens, val_bytes, counts, n_val_bytes):
        """vb_shuffle_import_bytes: the received columns (torch CUDA tensors, source-rank major) and what every source rank
        sent.  The keys are kept alive until seal; the values are copied by the call."""
        _sync_torch(keys, val_lens, val_bytes)
        self._keepalive.append(keys)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
        arr = lambda c: (ctypes.c_uint64 * len(c))(*c)
        L.check(self._lib.vb_shuffle_import_bytes(self._h, p(keys), p(val_lens), p(val_bytes), arr(counts), arr(n_val_bytes)))

    @classmethod
    def narrow(cls, parent, out_col, vcode):
        """vb_shuffle_create_narrow: the sealed reduce result `parent` (output column out_col) as a sealed COGROUP side
        under the same partitioner, each key with the one-element list [its result] (vcode: the result's dtype)."""
        self = cls.__new__(cls)
        self.sc, self._lib = parent.sc, parent._lib
        self.n_map, self.n_reduce, self.agg, self.vcode, self.kcode = 0, parent.n_reduce, L.VB_AGG_COGROUP, vcode, parent.kcode
        self.has_payload, self._keepalive = True, []
        h = ctypes.c_void_p()
        L.check(self._lib.vb_shuffle_create_narrow(parent._h, out_col, ctypes.byref(h)))
        self._h = h
        self.sc._shuffles.add(self)
        return self

    def map(self, map_id, keys, vals, start, stop):
        """ShuffleMapTask::run for one map partition = rows [start, stop) of the parent."""
        n = stop - start
        if keys.loc == L.VB_DEVICE_BORROWED:
            self._keepalive.append((keys.owner, vals.owner if vals is not None else None))
        if isinstance(vals, _BytesCol):
            vals.check_loc(keys.loc)
            self.as_str = vals.as_str
            L.check(self._lib.vb_shuffle_map_bytes(self._h, map_id, keys.at(start), vals.offs_at(start), vals.data_at(), vals.n_bytes,
                                                   n, keys.loc))
            return
        if keys.rows:
            L.check(self._lib.vb_shuffle_map_aos(self._h, map_id, keys.at(start), n, keys.loc))
        else:
            if vals is not None and vals.loc != keys.loc:
                raise ValueError("keys and values must live in the same memory space")
            L.check(self._lib.vb_shuffle_map_soa(self._h, map_id, keys.at(start), vals.at(start) if vals is not None else None, n, keys.loc))

    def map_cols(self, map_id, keys, cols, start, stop):
        """One map partition of a multi-aggregate shuffle: rows [start, stop) of keys and every value column."""
        if any(c.loc != keys.loc for c in cols):
            raise ValueError("keys and values must live in the same memory space")
        if keys.loc == L.VB_DEVICE_BORROWED:
            self._keepalive.append((keys.owner,) + tuple(c.owner for c in cols))
        ptrs = (ctypes.c_void_p * len(cols))(*[c.at(start) for c in cols])
        L.check(self._lib.vb_shuffle_map_cols(self._h, map_id, keys.at(start), ptrs, stop - start, keys.loc))

    def reduce_cols(self, r, out_dtypes, dst_loc=L.VB_HOST, out_keys=None, out_aggs=None):
        """Reduce partition r of a multi-aggregate shuffle → (keys, [one array per aggregate]) on the host, or into
        caller-provided torch CUDA tensors with dst_loc=VB_DEVICE (any may be None)."""
        if dst_loc == L.VB_DEVICE:
            _sync_torch(out_keys, *(out_aggs or []))
            p = lambda t: t.data_ptr() if t is not None else None
            ptrs = (ctypes.c_void_p * len(out_aggs))(*[p(t) for t in out_aggs])
            L.check(self._lib.vb_shuffle_reduce_cols(self._h, r, p(out_keys), ptrs, L.VB_DEVICE))
            return out_keys, out_aggs
        nk, _ = self.reduce_size(r)
        keys = np.empty(nk, dtype=_NP_OF[self.kcode])
        outs = [np.empty(nk, dtype=dt) for dt in out_dtypes]
        ptrs = (ctypes.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
        L.check(self._lib.vb_shuffle_reduce_cols(self._h, r, keys.ctypes.data_as(ctypes.c_void_p), ptrs, L.VB_HOST))
        return keys, outs

    def exchange(self, mode=L.VB_XCHG_AUTO):
        """The shuffle's exchange step inside the library (collective; needs Context.comm_init)."""
        L.check(self._lib.vb_shuffle_exchange(self._h, mode))

    def exchange_stats(self):
        st = L.vb_xstats()
        L.check(self._lib.vb_shuffle_exchange_stats(self._h, ctypes.byref(st)))
        return {"sent_rows": st.sent_rows, "recv_rows": st.recv_rows, "exchanges": st.exchanges,
                "exchange_ms": st.exchange_ms, "exchange_kind": {0: None, 1: "nccl", 2: "p2p"}[st.kind],
                "prepare_wall_ms": st.prepare_wall_ms, "counts_wall_ms": st.counts_wall_ms, "post_wall_ms": st.post_wall_ms}

    def seal(self):
        L.check(self._lib.vb_shuffle_seal(self._h))
        self._keepalive = []

    def reduce_size(self, r):
        nk, nv = ctypes.c_uint64(), ctypes.c_uint64()
        L.check(self._lib.vb_shuffle_reduce_size(self._h, r, ctypes.byref(nk), ctypes.byref(nv)))
        return nk.value, nv.value

    def gather(self, refs, valid=None):
        """Byte-string values: the references refs (read from this shuffle's output) gathered into an object array of
        str or bytes, None where valid (one byte per row) is 0."""
        refs = np.ascontiguousarray(refs, dtype=np.uint64)
        n, nb = len(refs), ctypes.c_uint64()
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        L.check(self._lib.vb_shuffle_gather_bytes_size(self._h, p(refs), n, L.VB_HOST, ctypes.byref(nb)))
        offs, data = np.empty(n + 1, dtype=np.uint64), np.empty(nb.value, dtype=np.uint8)
        L.check(self._lib.vb_shuffle_gather_bytes(self._h, p(refs), n, L.VB_HOST, p(offs), p(data), L.VB_HOST))
        raw, o = data.tobytes(), offs.astype(np.int64).tolist()
        out = np.empty(n, dtype=object)
        if getattr(self, "as_str", True):
            out[:] = [raw[o[i]:o[i + 1]].decode("utf-8", "surrogateescape") for i in range(n)]
        else:
            out[:] = [raw[o[i]:o[i + 1]] for i in range(n)]
        if valid is not None:
            out[np.asarray(valid) == 0] = None
        return out

    def reduce(self, r):
        """ShuffledRdd::compute(split r) → host arrays."""
        nk, nv = self.reduce_size(r)
        keys = np.empty(nk, dtype=_NP_OF[self.kcode])
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
        if self.agg in (L.VB_AGG_GROUP, L.VB_AGG_COGROUP):
            offs = np.empty(nk + 1, dtype=np.uint64)
            vals = np.empty(nv, dtype=_NP_OF[self.vcode])
            L.check(self._lib.vb_shuffle_reduce(self._h, r, p(keys), None, p(offs), p(vals), L.VB_HOST))
            return keys, offs, _vals_out(self, vals)
        if self.agg == L.VB_AGG_SORT and not self.has_payload:
            L.check(self._lib.vb_shuffle_reduce(self._h, r, p(keys), None, None, None, L.VB_HOST))
            return keys, None
        out_dt = np.uint64 if self.agg == L.VB_AGG_COUNT else _NP_OF[self.vcode]
        comb = np.empty(nk, dtype=out_dt)
        L.check(self._lib.vb_shuffle_reduce(self._h, r, p(keys), p(comb), None, None, L.VB_HOST))
        return keys, _vals_out(self, comb)

    def reduce_device(self, r, out_keys=None, out_comb=None, out_offs=None, out_vals=None):
        """Same, into caller-provided torch CUDA tensors (any may be None)."""
        _sync_torch(out_keys, out_comb, out_offs, out_vals)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        L.check(self._lib.vb_shuffle_reduce(self._h, r, p(out_keys), p(out_comb), p(out_offs), p(out_vals), L.VB_DEVICE))

    def reduce_blob(self, r):
        """Reduce partition r as the bincode 1.2.1 blob vega stores in SHUFFLE_CACHE (bytes)."""
        n = ctypes.c_uint64()
        L.check(self._lib.vb_shuffle_reduce_blob_size(self._h, r, ctypes.byref(n)))
        buf = np.empty(n.value, dtype=np.uint8)
        L.check(self._lib.vb_shuffle_reduce_blob(self._h, r, buf.ctypes.data_as(ctypes.c_void_p), L.VB_HOST))
        return buf.tobytes()

    def reduce_blob_device(self, r, out):
        """Same, into a caller-provided torch CUDA uint8 tensor of reduce_blob_size(r) bytes (16-byte aligned for a
        string-key shuffle)."""
        _sync_torch(out)
        L.check(self._lib.vb_shuffle_reduce_blob(self._h, r, ctypes.c_void_p(out.data_ptr()), L.VB_DEVICE))

    def reduce_blob_size(self, r):
        n = ctypes.c_uint64()
        L.check(self._lib.vb_shuffle_reduce_blob_size(self._h, r, ctypes.byref(n)))
        return n.value

    def map_blob(self, map_id, blob):
        """Submit one map-side-combined bucket (bincode blob, bytes) as the output of map task `map_id`."""
        buf = np.frombuffer(blob, dtype=np.uint8)
        L.check(self._lib.vb_shuffle_map_blob(self._h, map_id, buf.ctypes.data_as(ctypes.c_void_p), len(buf), L.VB_HOST))

    def stats(self):
        st = L.vb_stats()
        L.check(self._lib.vb_shuffle_stats(self._h, ctypes.byref(st)))
        d = {f: getattr(st, f) for f, _ in st._fields_}
        kt = {}
        for i, name in enumerate(L.KERNEL_CLASSES):
            ms, n = ctypes.c_double(), ctypes.c_uint64()
            L.check(self._lib.vb_shuffle_kernel_time(self._h, i, ctypes.byref(ms), ctypes.byref(n)))
            kt[name] = {"ms": ms.value, "launches": n.value}
        d["kernels"] = kt
        return d

    def free(self):
        if self._h and self.sc._h:
            self._lib.vb_shuffle_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Grouped:
    """Result of group_by_key: CSR over all partitions in partition order.
    `to_list()` gives the reference's Vec<(K, Vec<V>)>."""

    def __init__(self, keys, offsets, vals):
        self.keys, self.offsets, self.vals = keys, offsets, vals

    def to_list(self):
        o = self.offsets
        item = lambda k: k.item() if isinstance(k, np.generic) else k      # numpy scalar keys, or str keys
        return [(item(self.keys[i]), self.vals[int(o[i]):int(o[i + 1])]) for i in range(len(self.keys))]

    def to_dict(self):
        return {k: v for k, v in self.to_list()}

    def __len__(self):
        return len(self.keys)


class _Base:
    def number_of_splits(self):
        return self.num_slices


_REDUCE_AGGS = ("sum", "min", "max", "count")


def _vals_out(sh, v, valid=None):
    """One side's values as returned to the caller: numeric values as they are (a numpy.ma.MaskedArray where validity is
    given), byte-string values gathered from the side's shuffle into an object array (None where validity is 0)."""
    if sh.vcode == L.VB_BYTES:
        return sh.gather(v, valid)
    return v if valid is None else np.ma.MaskedArray(v, mask=valid == 0)


def _value_order(sort_values, parents):
    """The vb_value_order of sort_values=... for shuffles of `parents` (TypeError, before any device work, for a
    non-bool or for byte-string values, which have no value order)."""
    if not isinstance(sort_values, (bool, np.bool_)):
        raise TypeError(f"sort_values must be a bool, got {sort_values!r}")
    if not sort_values:
        return L.VB_VALORDER_INPUT
    for r in parents:
        if isinstance(getattr(r, "vals", None), _BytesCol):
            raise TypeError("sort_values: byte-string values have no value order")
    return L.VB_VALORDER_ASC


def _refuse_bytes(parent, what):
    """TypeError, before any device work, for an op that computes on byte-string values."""
    if isinstance(getattr(parent, "vals", None), _BytesCol):
        raise TypeError(f"{what} computes on values: byte-string values support group_by_key, partition_by_key, the "
                        "joins, cogroup and sort_by_key")
_CODE_OF = {np.uint64: L.VB_U64, np.int64: L.VB_I64, np.float64: L.VB_F64}


class _AggregatedParent(_Base):
    """A reduce result (reduce_by_key / count_by_key, or one aggregate of combine_by_key) as a join or cogroup parent,
    next to PairRdds.  Its partition r already holds the keys with hash % num_splits == r, each once, so under the same
    num_splits it joins through a view of the sealed result (vb_shuffle_create_narrow: vega's OneToOneDependency,
    co_grouped_rdd.rs:103-112) with no second shuffle.  Under another num_splits each result partition is read into
    device tensors and becomes one map task of an ordinary COGROUP shuffle (vega's ShuffleDependency over the
    ShuffledRdd), with no host round trip.  Either way the key's list on this side is [its result]."""

    def join(self, other, num_splits):
        return JoinedRdd(self, other, num_splits)

    def left_outer_join(self, other, num_splits):
        return JoinedRdd(self, other, num_splits, "left")

    def right_outer_join(self, other, num_splits):
        return JoinedRdd(self, other, num_splits, "right")

    def full_outer_join(self, other, num_splits):
        return JoinedRdd(self, other, num_splits, "full")

    def cogroup(self, other, num_splits):
        return JoinedRdd(self, other, num_splits)

    def subtract_by_key(self, other, num_splits, sort_values=False):
        """PairRdd.subtract_by_key with this result as the filtered side: under the same num_splits it is read through
        a view, without a second shuffle."""
        cls = StrCoGroupedRdd if isinstance(self, StrShuffledRdd) else CoGroupedRdd
        return SemiJoinedRdd(cls([self, other], num_splits, sort_values=sort_values), 0, 0b10)

    def semi_join(self, other, num_splits, sort_values=False):
        """PairRdd.semi_join with this result as the filtered side (see subtract_by_key)."""
        cls = StrCoGroupedRdd if isinstance(self, StrShuffledRdd) else CoGroupedRdd
        return SemiJoinedRdd(cls([self, other], num_splits, sort_values=sort_values), 0b10, 0)

    def _cogroup_side(self, num_splits):
        """The sealed COGROUP-kind shuffle a cogroup over num_splits partitions reads for this parent."""
        sh = self._run()
        if num_splits == sh.n_reduce:
            col, _, vcode = self._result_col(sh)
            return Shuffle.narrow(sh, col, vcode)
        return self._reshuffled(num_splits)

    def _reshuffled(self, num_splits):
        """The result shuffled again over num_splits partitions, one map task per result partition read on the device."""
        sh = self._run()
        col, n_cols, vcode = self._result_col(sh)
        import torch
        dev = f"cuda:{sh._lib.vb_ctx_device(self.sc._h)}"
        out = Shuffle(self.sc, sh.n_reduce, num_splits, sh.kcode, vcode, L.VB_AGG_COGROUP, key_width=self.keys.key_width)
        for r in range(sh.n_reduce):
            nk = sh.reduce_size(r)[0]
            k, v = (torch.empty(nk, dtype=torch.int64, device=dev) for _ in range(2))
            if n_cols is None:
                sh.reduce_device(r, out_keys=k, out_comb=v)
            else:
                sh.reduce_cols(r, None, L.VB_DEVICE, out_keys=k, out_aggs=[v if c == col else None for c in range(n_cols)])
            out.map(r, _Col(k), _Col(v, role="value"), 0, nk)
        out.seal()
        return out


def _check_parent(r, j):
    """TypeError, before any device work, for an aggregated parent that cannot be a cogroup side."""
    if isinstance(r, StrShuffledRdd):
        raise TypeError(f"parent {j}: String keys do not support cogroup")
    if isinstance(r, ShuffledRdd) and r.agg_name not in _REDUCE_AGGS:
        raise TypeError(f"parent {j}: a {r.agg_name} result is not a join parent (reduce_by_key, count_by_key and "
                        "combine_by_key results are)")


class ShuffledRdd(_AggregatedParent):
    """ShuffledRdd<K,V,C> (src/rdd/shuffled_rdd.rs): lazy; `collect()` runs the job.  A sum / min / max / count result
    is also a join and cogroup parent (see _AggregatedParent)."""

    def __init__(self, parent, agg_name, num_splits, hint=0, sort_values=False):
        if num_splits < 1:
            raise ValueError("num_splits must be >= 1")
        if len(getattr(parent, "cols", ())) > 1:
            raise TypeError("a PairRdd with several value columns supports combine_by_key only")
        if agg_name in _REDUCE_AGGS:
            _refuse_bytes(parent, "reduce_by_key / count_by_key")
        self.value_order = _value_order(sort_values, [parent])
        self.parent, self.agg_name, self.num_slices, self.hint = parent, agg_name, num_splits, hint
        self.sc = parent.sc
        self._sh = None

    @property
    def keys(self):
        return self.parent.keys

    def _result_col(self, sh):
        return 0, None, L.VB_U64 if sh.agg == L.VB_AGG_COUNT else sh.vcode

    def _cogroup_side(self, num_splits):
        if self.agg_name == "cogroup":                  # a PairRdd parent's own shuffle (JoinedRdd, CoGroupedRdd)
            return self._run()
        return super()._cogroup_side(num_splits)

    def _run(self):
        if self._sh is not None:
            return self._sh
        p = self.parent
        starts = slice_starts(p.n, p.num_slices)
        vcode = p.vals.code if p.vals is not None else (p.keys.code if p.keys.rows else L.VB_U64)
        sh = Shuffle(self.sc, len(starts) - 1, self.num_slices, p.keys.code, vcode, _AGG[self.agg_name],
                     key_width=p.keys.key_width, hint=self.hint, value_order=self.value_order)
        sh.has_payload = p.vals is not None or p.keys.rows
        for m in range(len(starts) - 1):                    # map stage
            sh.map(m, p.keys, p.vals, int(starts[m]), int(starts[m + 1]))
        sh.seal()                                           # register_map_outputs
        self._sh = sh
        return sh

    def compute(self, split):
        return self._run().reduce(split)

    def collect(self):
        sh = self._run()
        parts = [sh.reduce(r) for r in range(self.num_slices)]     # result stage, partition order
        if self.agg_name in ("group", "cogroup"):
            keys = np.concatenate([p[0] for p in parts])
            vals = np.concatenate([p[2] for p in parts])
            offs, base = [], 0
            for p in parts:
                offs.append(p[1][:-1].astype(np.uint64) + np.uint64(base))
                base += len(p[2])
            offs.append(np.array([base], dtype=np.uint64))
            return Grouped(keys, np.concatenate(offs), vals)
        comb = None if parts[0][1] is None else np.concatenate([p[1] for p in parts])
        return np.concatenate([p[0] for p in parts]), comb

    def stats(self):
        return self._run().stats()


_JOIN_KINDS = {"left": L.VB_JOIN_LEFT, "right": L.VB_JOIN_RIGHT, "full": L.VB_JOIN_FULL}


class JoinedRdd(_Base):
    """`a.join(b, num_splits)` (src/rdd/pair_rdd.rs:104-121): cogroup of two Vec-append
    shuffles + per-key cross product, inner join.

    kind "left" / "right" / "full": the outer joins (Spark's leftOuterJoin / rightOuterJoin / fullOuterJoin, which
    vega lacks).  A key missing on the other side still gives rows, with None on that side.  compute(r) / collect()
    return (k, v, w); a side that can be None is a numpy.ma.MaskedArray (masked = None, data 0), the other side a
    plain array.  sort_values=True: each PairRdd side's lists ascending in its value dtype's order (so the rows of a
    key come in that order too); a reduce-result side has one value per key."""

    def __init__(self, left, right, num_splits, kind=None, sort_values=False):
        self.value_order = _value_order(sort_values, (left, right))
        if kind is not None:
            if kind not in _JOIN_KINDS:
                raise ValueError(f"join kind {kind!r} is not one of {sorted(_JOIN_KINDS)}")
            if num_splits < 1:
                raise ValueError("num_splits must be >= 1")
            if left.keys.key_width != right.keys.key_width:
                raise TypeError("join sides have different key types")
        sides = (left, right)
        if any(isinstance(r, _AggregatedParent) for r in sides):     # a reduce result as a parent (_AggregatedParent)
            for j, r in enumerate(sides):
                if isinstance(r, _AggregatedParent):
                    _check_parent(r, j)
                elif not isinstance(r, PairRdd) or isinstance(r, StrPairRdd):
                    raise TypeError(f"parent {j} is not an integer-key PairRdd or reduce result")
            if num_splits < 1:
                raise ValueError("num_splits must be >= 1")
            if left.keys.key_width != right.keys.key_width or left.keys.code != right.keys.code:
                raise TypeError("join sides have different key types")
        self.left, self.right, self.num_slices, self.sc = left, right, num_splits, left.sc
        self.kind = kind
        self._shs = None

    def _run(self):
        if self._shs is None:
            a, b = (r if isinstance(r, _AggregatedParent) else
                    ShuffledRdd(r, "cogroup", self.num_slices, sort_values=self.value_order == L.VB_VALORDER_ASC)
                    for r in (self.left, self.right))
            if self.left.keys.key_width != self.right.keys.key_width:
                raise TypeError("join sides have different key types")
            self._shs = (a._cogroup_side(self.num_slices), b._cogroup_side(self.num_slices))
        return self._shs

    def compute(self, split):
        a, b = self._run()
        lib = self.sc._lib
        n = ctypes.c_uint64()
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p) if x is not None else None
        if self.kind is not None:
            kind = _JOIN_KINDS[self.kind]
            L.check(lib.vb_join_outer_size(a._h, b._h, split, kind, ctypes.byref(n)))
        else:
            L.check(lib.vb_join_size(a._h, b._h, split, ctypes.byref(n)))
        k = np.empty(n.value, dtype=_NP_OF[a.kcode])
        v = np.empty(n.value, dtype=_NP_OF[a.vcode])
        w = np.empty(n.value, dtype=_NP_OF[b.vcode])
        if self.kind is None:
            L.check(lib.vb_join(a._h, b._h, split, p(k), p(v), p(w), L.VB_HOST))
            return k, _vals_out(a, v), _vals_out(b, w)
        vv = np.empty(n.value, dtype=np.uint8) if self.kind != "left" else None     # validity of the side that can be None
        wv = np.empty(n.value, dtype=np.uint8) if self.kind != "right" else None
        L.check(lib.vb_join_outer(a._h, b._h, split, kind, p(k), p(v), p(w), p(vv), p(wv), L.VB_HOST))
        return k, _vals_out(a, v, vv), _vals_out(b, w, wv)

    def collect(self):
        parts = [self.compute(r) for r in range(self.num_slices)]
        cat = lambda xs: np.ma.concatenate(xs) if isinstance(xs[0], np.ma.MaskedArray) else np.concatenate(xs)
        return tuple(cat([p[i] for p in parts]) for i in range(3))

    def cogroup_compute(self, split):
        """Partition `split` of the cogroup (co_grouped_rdd.rs:206-249), aligned on the device by vb_cogroup:
        (keys, (left_offsets, left_vals), (right_offsets, right_vals)).  Every key of either side appears once; key
        i's lists are left_vals[left_offsets[i]:left_offsets[i + 1]] and the same on the right, empty where that
        side lacks the key."""
        a, b = self._run()
        lib = self.sc._lib
        nk, nl, nr = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        L.check(lib.vb_cogroup_size(a._h, b._h, split, ctypes.byref(nk), ctypes.byref(nl), ctypes.byref(nr)))
        keys = np.empty(nk.value, dtype=_NP_OF[a.kcode])
        lo, ro = np.empty(nk.value + 1, dtype=np.uint64), np.empty(nk.value + 1, dtype=np.uint64)
        lv, rv = np.empty(nl.value, dtype=_NP_OF[a.vcode]), np.empty(nr.value, dtype=_NP_OF[b.vcode])
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
        L.check(lib.vb_cogroup(a._h, b._h, split, p(keys), p(lo), p(lv), p(ro), p(rv), L.VB_HOST))
        return keys, (lo, _vals_out(a, lv)), (ro, _vals_out(b, rv))

    def cogroup_collect(self):
        """cogroup(): per partition, the union of keys with both value lists (co_grouped_rdd.rs:206-249), as a list
        of (k, (vs, ws)) with numpy arrays."""
        out = []
        for r in range(self.num_slices):
            keys, (lo, lv), (ro, rv) = self.cogroup_compute(r)
            lo, ro = lo.tolist(), ro.tolist()
            out.extend((k, (lv[lo[i]:lo[i + 1]], rv[ro[i]:ro[i + 1]])) for i, k in enumerate(keys.tolist()))
        return out


class CoGroupedRdd(_Base):
    """CoGroupedRdd::new(rdds, HashPartitioner::new(num_splits)) (src/rdd/co_grouped_rdd.rs:75-135): the cogroup of any
    number of PairRdds (1 to 16), each shuffled with the Vec-append aggregator as JoinedRdd does.  A reduce result
    (reduce_by_key / count_by_key, or CombinedRdd.aggregate(name)) is a parent too, with the list [its result] per key;
    under the same num_splits it is not shuffled again (_AggregatedParent).

    compute(r) -> (keys, [(offsets, values) per parent]): every key of the partition once; key i's list from parent j
    is values_j[offsets_j[i]:offsets_j[i + 1]], empty where that parent lacks the key.  collect() gives the
    reference's Vec<(K, Vec<Vec<V>>)> as a list of (k, [vs_0, ..., vs_{n-1}]).  join_compute(r) / join_collect() give
    the inner join of all parents as (k, [v_0, ..., v_{n-1}]) arrays: per key, for v0 in vs_0 { for v1 in vs_1 { ... } }.
    outer_join_compute(r, required) / outer_join_collect(required) give the outer join in which only the required
    parents must have the key.  Each parent's values keep that parent's dtype.  sort_values=True: every shuffled
    parent's lists ascending in its value dtype's order (vb_shuffle_set_value_order)."""

    def __init__(self, rdds, num_splits, sort_values=False):
        rdds = list(rdds)
        if not 1 <= len(rdds) <= L.VB_MAX_COGROUP_SIDES:
            raise ValueError(f"a cogroup takes 1 to {L.VB_MAX_COGROUP_SIDES} parents, got {len(rdds)}")
        if num_splits < 1:
            raise ValueError("num_splits must be >= 1")
        for j, r in enumerate(rdds):
            if isinstance(r, StrPairRdd):
                raise TypeError(f"parent {j}: String keys do not support cogroup")
            if isinstance(r, _AggregatedParent):
                _check_parent(r, j)
                continue
            if not isinstance(r, PairRdd):
                raise TypeError(f"parent {j} is not a PairRdd")
            if len(r.cols) > 1:
                raise TypeError(f"parent {j}: a PairRdd with several value columns supports combine_by_key only")
        if any(r.sc is not rdds[0].sc for r in rdds):
            raise ValueError("the parents live on different contexts")
        k0 = rdds[0].keys
        if any(r.keys.key_width != k0.key_width or r.keys.code != k0.code for r in rdds):
            raise TypeError("the parents have different key types")
        self.value_order = _value_order(sort_values, rdds)
        self.rdds, self.num_slices, self.sc = rdds, num_splits, rdds[0].sc
        self._shs = None

    def _run(self):
        if self._shs is None:
            asc = self.value_order == L.VB_VALORDER_ASC
            self._shs = [(r if isinstance(r, _AggregatedParent) else ShuffledRdd(r, "cogroup", self.num_slices, sort_values=asc))
                         ._cogroup_side(self.num_slices) for r in self.rdds]
        return self._shs

    def _sides(self):
        shs = self._run()
        return shs, (ctypes.c_void_p * len(shs))(*[s._h.value for s in shs])

    def compute(self, split):
        """Partition `split` of the cogroup (co_grouped_rdd.rs:206-249), aligned on the device by vb_cogroup_n."""
        shs, sides = self._sides()
        n, lib = len(shs), self.sc._lib
        nk, nv = ctypes.c_uint64(), (ctypes.c_uint64 * n)()
        L.check(lib.vb_cogroup_n_size(sides, n, split, ctypes.byref(nk), nv))
        keys = np.empty(nk.value, dtype=_NP_OF[shs[0].kcode])
        offs = [np.empty(nk.value + 1, dtype=np.uint64) for _ in shs]
        vals = [np.empty(nv[j], dtype=_NP_OF[s.vcode]) for j, s in enumerate(shs)]
        ptrs = lambda xs: (ctypes.c_void_p * n)(*[x.ctypes.data for x in xs])
        L.check(lib.vb_cogroup_n(sides, n, split, keys.ctypes.data_as(ctypes.c_void_p), ptrs(offs), ptrs(vals), L.VB_HOST))
        return keys, list(zip(offs, [_vals_out(s, v) for s, v in zip(shs, vals)]))

    def collect(self):
        out = []
        for r in range(self.num_slices):
            keys, lists = self.compute(r)
            lists = [(o.tolist(), v) for o, v in lists]
            out.extend((k, [v[o[i]:o[i + 1]] for o, v in lists]) for i, k in enumerate(keys.tolist()))
        return out

    def join_compute(self, split):
        """Partition `split` of the inner join of all parents (vb_join_n): (k, [v_0, ..., v_{n-1}])."""
        shs, sides = self._sides()
        n, lib = len(shs), self.sc._lib
        nn = ctypes.c_uint64()
        L.check(lib.vb_join_n_size(sides, n, split, ctypes.byref(nn)))
        k = np.empty(nn.value, dtype=_NP_OF[shs[0].kcode])
        vs = [np.empty(nn.value, dtype=_NP_OF[s.vcode]) for s in shs]
        L.check(lib.vb_join_n(sides, n, split, k.ctypes.data_as(ctypes.c_void_p),
                              (ctypes.c_void_p * n)(*[v.ctypes.data for v in vs]), L.VB_HOST))
        return k, [_vals_out(s, v) for s, v in zip(shs, vs)]

    def join_collect(self):
        parts = [self.join_compute(r) for r in range(self.num_slices)]
        return (np.concatenate([p[0] for p in parts]),
                [np.concatenate([p[1][j] for p in parts]) for j in range(len(self.rdds))])

    def _required_mask(self, required):
        """`required` as a bitmask over the parents: an int mask, or an iterable of parent indices."""
        n = len(self.rdds)
        is_int = lambda x: isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))
        if is_int(required):
            mask = int(required)
            if not 0 <= mask < 1 << n:
                raise ValueError(f"required mask {mask:#x} names a parent outside 0..{n - 1}")
            return mask
        try:
            sides = list(required)
        except TypeError:
            raise TypeError(f"required must be a bitmask or an iterable of parent indices, got {required!r}") from None
        mask = 0
        for j in sides:
            if not is_int(j):
                raise TypeError(f"required: parent index {j!r} is not an integer")
            if not 0 <= j < n:
                raise ValueError(f"required: parent index {j} is outside 0..{n - 1}")
            mask |= 1 << int(j)
        return mask

    def _semi_masks(self, required, excluded):
        """(required, excluded) of a semi join as bitmasks over parents 1..n-1 (ValueError for parent 0 or a parent in
        both)."""
        req, exc = self._required_mask(required), self._required_mask(excluded)
        if (req | exc) & 1:
            raise ValueError("parent 0 is the parent filtered: it can be neither required nor excluded")
        if req & exc:
            raise ValueError(f"parents {req & exc:#x} are both required and excluded")
        return req, exc

    def semi_join_compute(self, split, required, excluded=0):
        """Partition `split` of the semi / anti join of parent 0 (vb_semi_join_n): (keys, values), one key per row.  A
        key of parent 0 is kept when every parent of `required` has it and no parent of `excluded` does, and gives its
        parent-0 rows in that parent's list order.  Both masks are bitmasks or iterables of parent indices, over parents
        1..n-1; the other parents' values are never read.  vega has no such op (Spark's subtractByKey: excluded = [1];
        left semi join: required = [1])."""
        req, exc = self._semi_masks(required, excluded)
        shs, sides = self._sides()
        n, lib = len(shs), self.sc._lib
        nn = ctypes.c_uint64()
        L.check(lib.vb_semi_join_n_size(sides, n, split, req, exc, ctypes.byref(nn)))
        k = np.empty(nn.value, dtype=_NP_OF[shs[0].kcode])
        v = np.empty(nn.value, dtype=_NP_OF[shs[0].vcode])
        L.check(lib.vb_semi_join_n(sides, n, split, req, exc, k.ctypes.data_as(ctypes.c_void_p), v.ctypes.data_as(ctypes.c_void_p),
                                   L.VB_HOST))
        return k, _vals_out(shs[0], v)

    def semi_join_collect(self, required, excluded=0):
        req, exc = self._semi_masks(required, excluded)
        parts = [self.semi_join_compute(r, req, exc) for r in range(self.num_slices)]
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

    def outer_join_compute(self, split, required):
        """Partition `split` of the outer join of all parents (vb_join_n_outer): (k, [v_0, ..., v_{n-1}]).  A key is
        kept if every required parent has it; an optional parent that lacks it gives one None slot, so the key gives
        prod max(len(vs_j), 1) rows, for v0 in vs_0 { for v1 in vs_1 { ... } }.  An optional parent's column is a
        numpy.ma.MaskedArray (masked = None, data 0), a required parent's a plain array.  `required` is a bitmask over
        the parents or an iterable of parent indices: all of them is join_compute, none is the full outer join."""
        mask = self._required_mask(required)
        shs, sides = self._sides()
        n, lib = len(shs), self.sc._lib
        nn = ctypes.c_uint64()
        L.check(lib.vb_join_n_outer_size(sides, n, split, mask, ctypes.byref(nn)))
        k = np.empty(nn.value, dtype=_NP_OF[shs[0].kcode])
        vs = [np.empty(nn.value, dtype=_NP_OF[s.vcode]) for s in shs]
        valid = [None if mask >> j & 1 else np.empty(nn.value, dtype=np.uint8) for j in range(n)]
        ptrs = lambda xs: (ctypes.c_void_p * n)(*[x.ctypes.data if x is not None else None for x in xs])
        L.check(lib.vb_join_n_outer(sides, n, split, mask, k.ctypes.data_as(ctypes.c_void_p), ptrs(vs), ptrs(valid),
                                    L.VB_HOST))
        return k, [_vals_out(s, v, ok) for s, v, ok in zip(shs, vs, valid)]

    def outer_join_collect(self, required):
        mask = self._required_mask(required)
        parts = [self.outer_join_compute(r, mask) for r in range(self.num_slices)]
        cat = lambda xs: np.ma.concatenate(xs) if isinstance(xs[0], np.ma.MaskedArray) else np.concatenate(xs)
        return np.concatenate([p[0] for p in parts]), [cat([p[1][j] for p in parts]) for j in range(len(self.rdds))]


class SemiJoinedRdd(_Base):
    """subtract_by_key / semi_join (Spark's subtractByKey and left semi join; vega has neither): the (k, v) rows of the
    first parent whose key the other parent lacks, or has.  Computed on the device by vb_semi_join_n(_str) over the
    cogroup of the two parents, with no cross product and without grouping the other parent; only the first parent's
    values are read.  compute(r) -> (keys, values), one key per row, a key's rows in its list order (ascending with
    sort_values=True); collect() -> the same over every partition in order.  String keys come back as str or bytes."""

    def __init__(self, cogrouped, required, excluded):
        self.cogrouped = cogrouped
        self.required, self.excluded = cogrouped._semi_masks(required, excluded)
        self.sc, self.num_slices = cogrouped.sc, cogrouped.num_slices

    def compute(self, split):
        return self.cogrouped.semi_join_compute(split, self.required, self.excluded)

    def collect(self):
        return self.cogrouped.semi_join_collect(self.required, self.excluded)


def _combine_spec(aggs, cols, num_splits):
    """combine_by_key's arguments over value columns `cols` (ValueError before any device work): the vb_agg_col spec
    [(vb_agg, column)], the aggregate names and each aggregate's output dtype, in the order given."""
    if num_splits < 1:
        raise ValueError("num_splits must be >= 1")
    if not hasattr(aggs, "items") or not aggs:
        raise ValueError("aggs must be a non-empty mapping name -> (op, column)")
    spec, names = [], []
    for name, item in aggs.items():
        if not isinstance(item, (tuple, list)) or len(item) != 2:
            raise ValueError(f"aggregate {name!r}: expected (op, column), got {item!r}")
        op, col = item
        if op not in _COMBINE_OPS:
            raise ValueError(f"aggregate {name!r}: op {op!r} is not one of {sorted(_COMBINE_OPS)}")
        if op == "count":
            col = 0
        elif not isinstance(col, (int, np.integer)) or isinstance(col, bool) or not 0 <= col < len(cols):
            raise ValueError(f"aggregate {name!r}: column {col!r} out of range for {len(cols)} value columns")
        spec.append((_COMBINE_OPS[op], int(col)))
        names.append(name)
    ops = [op for op, _ in aggs.values()]
    n_acc = len(ops) + (1 if "mean" in ops and "count" not in ops else 0)
    if n_acc > L.VB_MAX_AGGS:
        raise ValueError(f"{len(ops)} aggregates{' plus the count a mean needs' if n_acc > len(ops) else ''} "
                         f"exceed {L.VB_MAX_AGGS}")
    out_dtypes = [np.uint64 if a == L.VB_AGG_COUNT else np.float64 if a == L.VB_AGG_MEAN else _NP_OF[cols[c].code]
                  for a, c in spec]
    return spec, names, out_dtypes


class CombinedRdd(_Base):
    """`combine_by_key` with named aggregates (src/rdd/pair_rdd.rs:20-33): one shuffle, several aggregates per key.
    `compute(r)` / `collect()` return (keys, {name: array}) with the aggregates in the order they were given."""

    def __init__(self, parent, aggs, num_splits, hint=0):
        self.spec, self.names, self.out_dtypes = _combine_spec(aggs, parent.cols, num_splits)
        self.parent, self.num_slices, self.hint, self.sc = parent, num_splits, hint, parent.sc
        self._sh = None

    def _run(self):
        if self._sh is not None:
            return self._sh
        p = self.parent
        starts = slice_starts(p.n, p.num_slices)
        sh = Shuffle(self.sc, len(starts) - 1, self.num_slices, p.keys.code, L.VB_U64, L.VB_AGG_SUM, key_width=p.keys.key_width,
                     hint=self.hint, multi=([c.code for c in p.cols], self.spec))
        for m in range(len(starts) - 1):
            sh.map_cols(m, p.keys, p.cols, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        self._sh = sh
        return sh

    def aggregate(self, name):
        """The named aggregate as a join / cogroup parent: (key, that aggregate's result) rows (_AggregatedParent)."""
        if name not in self.names:
            raise ValueError(f"no aggregate named {name!r} (the aggregates are {self.names})")
        return AggregateRdd(self, name)

    def compute(self, split):
        keys, outs = self._run().reduce_cols(split, self.out_dtypes)
        return keys, dict(zip(self.names, outs))

    def collect(self):
        parts = [self.compute(r) for r in range(self.num_slices)]
        return (np.concatenate([p[0] for p in parts]),
                {name: np.concatenate([p[1][name] for p in parts]) for name in self.names})

    def stats(self):
        return self._run().stats()


class AggregateRdd(_AggregatedParent):
    """One named aggregate of a CombinedRdd as a join / cogroup parent (CombinedRdd.aggregate(name)).  The combine
    shuffle runs once and is shared by every aggregate taken from it."""

    def __init__(self, combined, name):
        self.combined, self.name = combined, name
        self.sc, self.num_slices = combined.sc, combined.num_slices

    @property
    def keys(self):
        return self.combined.parent.keys

    def _run(self):
        return self.combined._run()

    def _result_col(self, sh):
        i = self.combined.names.index(self.name)
        return i, len(self.combined.names), _CODE_OF[self.combined.out_dtypes[i]]


class RepShuffle(Shuffle):
    """vb_shuffle_create_repartition: repartition(n) = coalesce(n, shuffle=true) of items of n_cols 64-bit columns plus,
    with has_bytes, one byte-string column.  Partition r holds its items in map-id, then input order."""

    def __init__(self, sc, n_map, n_reduce, codes, has_bytes, as_str=True, rank=0, world=1):
        """codes: the dtype code of each 64-bit column (the dtype its items come back as).  world > 1: rank `rank`'s
        shuffle (vb_shuffle_create_repartition_dist); map this rank's block of map ids, then exchange() and seal()."""
        self.sc, self._lib = sc, sc._lib
        self.n_map, self.n_reduce, self.codes, self.has_bytes, self.as_str = n_map, n_reduce, tuple(codes), bool(has_bytes), as_str
        self.agg = self.vcode = self.kcode = None
        self.has_payload, self._keepalive = True, []
        h = ctypes.c_void_p()
        self.rank, self.world = rank, world
        L.check(self._lib.vb_shuffle_create_repartition_dist(sc._h, sc.new_shuffle_id(), n_map, n_reduce, len(self.codes),
                                                              int(self.has_bytes), rank, world, ctypes.byref(h)))
        self._h = h
        sc._shuffles.add(self)

    def map_items(self, map_id, first_position, cols, bcol, start, stop):
        """Map task map_id: items [start, stop) of the columns cols and of the byte-string column bcol (or None), at the
        positions first_position + 1, first_position + 2, ..."""
        host = [c.loc == L.VB_HOST for c in cols] + ([bcol.loc == L.VB_HOST] if bcol is not None else [])
        if len(set(host)) > 1:
            raise ValueError("the item columns must live in the same memory space")
        loc = cols[0].loc if cols else bcol.loc
        if loc == L.VB_DEVICE_BORROWED:
            self._keepalive.append(tuple(c.owner for c in cols))
        ptrs = (ctypes.c_void_p * len(cols))(*[c.at(start) for c in cols]) if cols else None
        offs, data, nb = (bcol.offs_at(start), bcol.data_at(), bcol.n_bytes) if bcol is not None else (None, None, 0)
        L.check(self._lib.vb_shuffle_map_repartition(self._h, map_id, int(first_position), ptrs, offs, data, nb, stop - start, loc))

    def reduce_size(self, r):
        """(items, their total bytes) of partition r."""
        n, nb = ctypes.c_uint64(), ctypes.c_uint64()
        L.check(self._lib.vb_shuffle_reduce_repartition_size(self._h, r, ctypes.byref(n), ctypes.byref(nb)))
        return n.value, nb.value

    def reduce(self, r):
        """Partition r on the host: ([one array per 64-bit column], object array of str / bytes, or None)."""
        n, nb = self.reduce_size(r)
        cols = [np.empty(n, dtype=_NP_OF[c]) for c in self.codes]
        ptrs = (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols]) if cols else None
        offs = np.empty(n + 1, dtype=np.uint64) if self.has_bytes else None
        data = np.empty(nb, dtype=np.uint8) if self.has_bytes else None
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
        L.check(self._lib.vb_shuffle_reduce_repartition(self._h, r, ptrs, p(offs), p(data), L.VB_HOST))
        if not self.has_bytes:
            return cols, None
        raw, o = data.tobytes(), offs.astype(np.int64).tolist()
        items = np.empty(n, dtype=object)
        if self.as_str:
            items[:] = [raw[o[i]:o[i + 1]].decode("utf-8", "surrogateescape") for i in range(n)]
        else:
            items[:] = [raw[o[i]:o[i + 1]] for i in range(n)]
        return cols, items

    def reduce_device(self, r, out_cols=None, out_offsets=None, out_bytes=None):
        """Partition r into caller-provided torch CUDA tensors (any may be None; sizes from reduce_size)."""
        out_cols = list(out_cols or [None] * len(self.codes))
        _sync_torch(out_offsets, out_bytes, *out_cols)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        ptrs = (ctypes.c_void_p * len(out_cols))(*[p(t) for t in out_cols]) if out_cols else None
        L.check(self._lib.vb_shuffle_reduce_repartition(self._h, r, ptrs, p(out_offsets), p(out_bytes), L.VB_DEVICE))


def _rep_starts(parent, starts):
    """One u64 start per map partition of parent (vega's start_m, drawn by the caller); 0 for every one by default."""
    n_map = len(slice_starts(parent.n, parent.num_slices)) - 1
    if starts is None:
        return [0] * n_map
    starts = [int(x) for x in (starts.tolist() if hasattr(starts, "tolist") else starts)]
    if len(starts) != n_map:
        raise ValueError(f"starts: one per map partition expected ({n_map}), got {len(starts)}")
    if any(not 0 <= x < 1 << 64 for x in starts):
        raise ValueError("starts must be u64 values")
    return starts


def _repartition(parent, num_partitions, shuffle, starts, cols, bcol=None, bytes_first=False):
    if not shuffle:
        raise NotImplementedError("coalesce(shuffle=False) (vega's narrow CoalescedRdd) is not served by the library")
    if isinstance(num_partitions, bool) or not isinstance(num_partitions, (int, np.integer)) or num_partitions < 1:
        raise ValueError("Number of partitions should be greater than or equal to 1")
    return RepartitionedRdd(parent, int(num_partitions), _rep_starts(parent, starts), cols, bcol, bytes_first)


def _split_rows(col):
    """(n,2) AoS rows as two 64-bit columns."""
    x = col.owner
    a, b = (x[:, 0].contiguous(), x[:, 1].contiguous()) if _is_torch(x) else (np.ascontiguousarray(x[:, 0]), np.ascontiguousarray(x[:, 1]))
    ka, kb = _Col(a, role="value"), _Col(b, role="value")
    ka.code = kb.code = col.code
    return ka, kb


class RepartitionedRdd(_Base):
    """`rdd.repartition(n)` = `rdd.coalesce(n, shuffle=true)` (rdd.rs:386-418): map partition m gives its items the positions
    starts[m] + 1 + i, and HashPartitioner::<usize> places each item by its position.  glom() lists the items per partition
    (in map-id, then input order), collect() concatenates them.  An item of one column comes back as an array; pairs come
    back as a tuple of two arrays, byte strings as an object array of str or bytes.
    With a communicator (Context.comm_init) every rank maps its contiguous block of map partitions, the library's NCCL
    exchange moves each partition to its owner (partition p on rank p % world), and a rank's glom() holds its own
    partitions (the others empty)."""

    def __init__(self, parent, num_partitions, starts, cols, bcol, bytes_first):
        self.sc, self.parent, self.num_slices, self.starts = parent.sc, parent, num_partitions, starts
        self.cols, self.bcol, self.bytes_first = tuple(cols), bcol, bytes_first
        self._sh = None

    def _run(self):
        if self._sh is not None:
            return self._sh
        bounds = slice_starts(self.parent.n, self.parent.num_slices)
        n_map = len(bounds) - 1
        rank, world = self.sc.comm or (0, 1)
        sh = RepShuffle(self.sc, n_map, self.num_slices, [c.code for c in self.cols], self.bcol is not None,
                        as_str=getattr(self.bcol, "as_str", True), rank=rank, world=world)
        for m in range((rank * n_map) // world, ((rank + 1) * n_map) // world):
            sh.map_items(m, self.starts[m], self.cols, self.bcol, int(bounds[m]), int(bounds[m + 1]))
        if world > 1:
            sh.exchange(L.VB_XCHG_NCCL)
        sh.seal()
        self._sh = sh
        return sh

    def _item(self, cols, items):
        parts = list(cols)
        if items is not None:
            parts.insert(0 if self.bytes_first else len(parts), items)
        return parts[0] if len(parts) == 1 else tuple(parts)

    def compute(self, split):
        return self._item(*self._run().reduce(split))

    def glom(self):
        return [self.compute(r) for r in range(self.num_slices)]

    def collect(self):
        parts = self.glom()
        if isinstance(parts[0], tuple):
            return tuple(np.concatenate([p[j] for p in parts]) for j in range(len(parts[0])))
        return np.concatenate(parts)


class PairRdd(_Base):
    """PairRdd<K,V> source (ParallelCollection of (K,V)); methods per src/rdd/pair_rdd.rs."""

    def __init__(self, sc, keys, vals, num_slices, cols=None):
        if num_slices < 1:
            raise ValueError("Number of slices should be greater than or equal to 1")
        if vals is not None and vals.n != keys.n:
            raise ValueError("keys and values differ in length")
        if cols is not None and any(c.n != keys.n for c in cols):
            raise ValueError("keys and value columns differ in length")
        if cols is not None and any(c.loc != keys.loc for c in cols):
            raise ValueError("keys and values must live in the same memory space")
        self.sc, self.keys, self.vals, self.num_slices, self.n = sc, keys, vals, num_slices, keys.n
        self.cols = cols if cols is not None else ((vals,) if vals is not None else ())

    def combine_by_key(self, aggs, num_splits, hint=0):
        """Several named aggregates per key in one shuffle.  aggs: ordered mapping name -> (op, column) with op in
        "sum" | "min" | "max" | "count" | "mean" and column an index into the value columns (ignored by "count"), e.g.
        {"n": ("count", None), "avg": ("mean", 0), "hi": ("max", 1)}."""
        if not self.cols:
            raise ValueError("combine_by_key needs value columns")
        _refuse_bytes(self, "combine_by_key")
        if self.keys.rows:
            raise ValueError("combine_by_key takes keys and value columns, not (n,2) rows")
        return CombinedRdd(self, aggs, num_splits, hint)

    def group_by_key(self, num_splits, sort_values=False):
        """sort_values=True: each key's values ascending in the value dtype's order (u64 unsigned, i64 signed, f64 as
        f64::total_cmp), sorted on the device; otherwise in map order."""
        return ShuffledRdd(self, "group", num_splits, sort_values=sort_values)

    def reduce_by_key(self, op, num_splits, hint=0):
        if op not in ("sum", "min", "max"):
            raise ValueError("reduce_by_key takes a named op: 'sum' | 'min' | 'max' (closures cannot cross the C ABI)")
        return ShuffledRdd(self, op, num_splits, hint)

    def count_by_key(self, num_splits=None, hint=0):
        return ShuffledRdd(self, "count", num_splits or self.num_slices, hint)

    def join(self, other, num_splits, sort_values=False):
        """sort_values=True: each key's rows in ascending order of both sides' values (see JoinedRdd)."""
        return JoinedRdd(self, other, num_splits, sort_values=sort_values)

    def left_outer_join(self, other, num_splits, sort_values=False):
        """(k, v, w) for every left row; w is None (masked) for a key the other side lacks."""
        return JoinedRdd(self, other, num_splits, "left", sort_values=sort_values)

    def right_outer_join(self, other, num_splits, sort_values=False):
        """(k, v, w) for every right row; v is None (masked) for a key this side lacks."""
        return JoinedRdd(self, other, num_splits, "right", sort_values=sort_values)

    def full_outer_join(self, other, num_splits, sort_values=False):
        """Rows of both sides; v or w is None (masked) for a key only the other side has."""
        return JoinedRdd(self, other, num_splits, "full", sort_values=sort_values)

    def cogroup(self, other, num_splits, sort_values=False):
        return JoinedRdd(self, other, num_splits, sort_values=sort_values)

    def subtract_by_key(self, other, num_splits, sort_values=False):
        """Spark's subtractByKey (vega has none): this PairRdd's (k, v) rows whose key `other` lacks.  other: a PairRdd
        or a reduce result of the same key type; its values are never read (SemiJoinedRdd)."""
        return SemiJoinedRdd(CoGroupedRdd([self, other], num_splits, sort_values=sort_values), 0, 0b10)

    def semi_join(self, other, num_splits, sort_values=False):
        """Left semi join (vega has none): this PairRdd's (k, v) rows whose key `other` has, each row once however many
        values `other` has for the key (SemiJoinedRdd)."""
        return SemiJoinedRdd(CoGroupedRdd([self, other], num_splits, sort_values=sort_values), 0b10, 0)

    def sort_by_key(self, num_splits):
        return ShuffledRdd(self, "sort", num_splits)

    def partition_by_key(self, num_splits):
        """partition_by_key (pair_rdd.rs:157-171): shuffle with the Vec-append aggregator, then
        flatten the values; `glom()` = values per partition."""
        return _Repartitioned(ShuffledRdd(self, "group", num_splits))

    def repartition(self, num_partitions, starts=None):
        """coalesce(num_partitions, shuffle=true) of the (k, v) items: see RepartitionedRdd."""
        return self.coalesce(num_partitions, True, starts)

    def coalesce(self, num_partitions, shuffle=False, starts=None):
        """rdd.rs:386-418 over (k, v) items: two 64-bit columns, or a key column and byte-string values.  starts: vega's
        start_m of each map partition (default 0)."""
        if isinstance(self.vals, _BytesCol):
            return _repartition(self, num_partitions, shuffle, starts, (self.keys,), self.vals)
        if len(self.cols) > 1:
            raise NotImplementedError("repartition of items with several value columns")
        keys = _split_rows(self.keys) if self.keys.rows else (self.keys,)
        return _repartition(self, num_partitions, shuffle, starts, keys + tuple(self.cols))


class _Repartitioned:
    def __init__(self, sh):
        self.sh = sh

    def glom(self):
        s = self.sh._run()
        return [s.reduce(r)[2] for r in range(self.sh.num_slices)]

    def collect(self):
        return np.concatenate(self.glom()) if self.sh.num_slices else np.empty(0)


class Rdd(_Base):
    """Key-only source RDD: the shuffle-backed ops of src/rdd/rdd.rs."""

    def __init__(self, sc, keys, num_slices):
        if num_slices < 1:
            raise ValueError("Number of slices should be greater than or equal to 1")
        self.sc, self.keys, self.num_slices, self.n = sc, keys, num_slices, keys.n

    def count_by_value(self):
        """rdd.rs:450-459: map(x → (x, 1u64)).reduce_by_key(+, number_of_splits)."""
        n_splits = len(slice_starts(self.n, self.num_slices)) - 1
        return ShuffledRdd(PairRdd(self.sc, self.keys, None, self.num_slices), "count", n_splits)

    def distinct(self, num_partitions=None):
        """rdd.rs:502-522: reduce_by_key on (Some(x), None), keys kept."""
        n_splits = num_partitions or (len(slice_starts(self.n, self.num_slices)) - 1)
        return _Distinct(ShuffledRdd(PairRdd(self.sc, self.keys, None, self.num_slices), "count", n_splits))

    distinct_with_num_partitions = distinct

    def sort(self, num_splits):
        return ShuffledRdd(PairRdd(self.sc, self.keys, None, self.num_slices), "sort", num_splits)

    def intersection(self, other, num_splits=None):
        """rdd.rs:852-946 `intersection` / `intersection_with_num_partitions`: the reference cogroups
        (x, None) of both sides and keeps the keys with `v1.len() >= 1 && v2.len() >= 1` — each key once."""
        return _SetOp(self, other, num_splits or self.number_of_splits_exact(), "and")

    intersection_with_num_partitions = intersection

    def subtract(self, other, num_splits=None):
        """rdd.rs:838-901 `subtract`: keys of self whose cogroup with `other` has exactly one non-empty side
        (`(v1.len() >= 1) ^ (v2.len() >= 1)`), intersected with self — i.e. the distinct keys of self not in other."""
        return _SetOp(self, other, num_splits or self.number_of_splits_exact(), "a_not_b")

    subtract_with_num_partition = subtract

    def group_by(self, func, num_splits=None):
        """rdd.rs:957-990 `group_by(func)`: map(x -> (func(x), x)).group_by_key(num_splits).  `func` is a
        vectorised key function over the item array (numpy / torch), e.g. `lambda x: np.sign(x) + 1`
        — a scalar closure cannot cross into CUDA (SURVEY.md F4), the key column it produces can."""
        owner = self.keys.owner
        k = func(owner)
        if not _is_torch(k):
            k = np.asarray(k)
        return PairRdd(self.sc, _Col(k), _Col(owner, role="value"), self.num_slices).group_by_key(num_splits or self.number_of_splits_exact())

    group_by_with_num_partitions = group_by

    def repartition(self, num_partitions, starts=None):
        """rdd.rs:386-390 `repartition(n)` = coalesce(n, shuffle=true): see RepartitionedRdd."""
        return self.coalesce(num_partitions, True, starts)

    def coalesce(self, num_partitions, shuffle=False, starts=None):
        """rdd.rs:392-418.  shuffle=True spreads the items evenly over num_partitions partitions; starts are vega's start_m
        of each map partition (one u64 each, default 0).  shuffle=False (the narrow CoalescedRdd) is not served."""
        return _repartition(self, num_partitions, shuffle, starts, (self.keys,))

    def number_of_splits_exact(self):
        return len(slice_starts(self.n, self.num_slices)) - 1


class _SetOp:
    """intersection / subtract as ONE tagged shuffle: side A rows carry the value 1, side B rows 2^32, the
    map-side combine + merge (hash_agg) sums them, and a key's sum says which sides it occurred on — the same
    information the reference reads off the two Vec lengths of its cogroup (rdd.rs:877-884, :925-932)."""

    def __init__(self, a, b, num_splits, mode):
        if a.keys.key_width != b.keys.key_width or a.keys.code != b.keys.code:
            raise TypeError("both sides must have the same item type")
        self.a, self.b, self.num_slices, self.mode, self.sc = a, b, num_splits, mode, a.sc
        self._sh = None

    @staticmethod
    def _const_like(col, value):
        if _is_torch(col.owner):
            import torch
            t = torch.full((col.n,), value, dtype=torch.int64, device=col.owner.device)
            return _Col(t, role="value")
        return _Col(np.full(col.n, value, dtype=np.uint64), role="value")

    def _run(self):
        if self._sh is not None:
            return self._sh
        sa, sb = slice_starts(self.a.n, self.a.num_slices), slice_starts(self.b.n, self.b.num_slices)
        na, nb = len(sa) - 1, len(sb) - 1
        sh = Shuffle(self.sc, na + nb, self.num_slices, self.a.keys.code, L.VB_U64, L.VB_AGG_SUM, key_width=self.a.keys.key_width)
        ta, tb = self._const_like(self.a.keys, 1), self._const_like(self.b.keys, 1 << 32)
        for m in range(na):
            sh.map(m, self.a.keys, ta, int(sa[m]), int(sa[m + 1]))
        for m in range(nb):
            sh.map(na + m, self.b.keys, tb, int(sb[m]), int(sb[m + 1]))
        sh.seal()
        self._sh = sh
        return sh

    def compute(self, split):
        k, c = self._run().reduce(split)
        c = c.view(np.uint64)
        in_a, in_b = (c & np.uint64(0xFFFFFFFF)) > 0, (c >> np.uint64(32)) > 0
        return k[in_a & in_b] if self.mode == "and" else k[in_a & ~in_b]

    def collect(self):
        parts = [self.compute(r) for r in range(self.num_slices)]
        return np.concatenate(parts) if parts else np.empty(0)


class _Distinct:
    def __init__(self, sh):
        self.sh = sh

    def collect(self):
        return self.sh.collect()[0]


# ---- string keys ------------------------------------------------------------------------------------------------
class StrKeys:
    """A column of byte-string keys, Arrow-style: key i is data[offsets[i]:offsets[i + 1]].  offsets has n + 1 64-bit
    integers and need not start at 0 (a slice of a larger column works as is); data holds the keys' UTF-8 bytes.
    Both are numpy arrays (data may also be `bytes`), or both torch CUDA tensors (int64 / uint64 offsets, uint8 data)."""

    def __init__(self, offsets, data):
        if _is_torch(offsets) or _is_torch(data):
            import torch
            if not (_is_torch(offsets) and _is_torch(data)) or not (offsets.is_cuda and data.is_cuda):
                raise TypeError("StrKeys: offsets and data must both be CUDA tensors, or both host arrays")
            if offsets.dtype not in (torch.int64, getattr(torch, "uint64", torch.int64)) or data.dtype != torch.uint8:
                raise TypeError("StrKeys: int64 / uint64 offsets and uint8 data expected")
            offsets, data = offsets.contiguous(), data.contiguous()
        else:
            if isinstance(data, (bytes, bytearray)):
                data = np.frombuffer(bytes(data), dtype=np.uint8)
            offsets, data = np.asarray(offsets), np.asarray(data)
            if offsets.dtype.kind not in "iu" or data.dtype != np.uint8:
                raise TypeError("StrKeys: integer offsets and uint8 data expected")
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            data = np.ascontiguousarray(data)
        if len(offsets.shape) != 1 or len(data.shape) != 1 or offsets.shape[0] < 1:
            raise ValueError("StrKeys: 1-D offsets of n + 1 entries and 1-D data expected")
        self.offsets, self.data = offsets, data

    @staticmethod
    def from_strs(strs):
        """Encode Python strs as UTF-8 into (offsets, bytes) on the host."""
        enc = [x.encode("utf-8") for x in strs]
        offsets = np.zeros(len(enc) + 1, dtype=np.uint64)
        np.cumsum(np.fromiter((len(b) for b in enc), dtype=np.uint64, count=len(enc)), out=offsets[1:])
        return StrKeys(offsets, np.frombuffer(b"".join(enc), dtype=np.uint8))

    def __len__(self):
        return self.offsets.shape[0] - 1

    def to_strs(self):
        """The keys as Python strs (bytes that are not UTF-8 are kept as surrogate escapes)."""
        return _decode_keys(np.asarray(self.offsets.cpu() if _is_torch(self.offsets) else self.offsets, dtype=np.uint64),
                            self.data.cpu().numpy() if _is_torch(self.data) else self.data)


class BytesKeys(StrKeys):
    """A column of byte-slice keys (Rust `Vec<u8>`, `&[u8]`, `Box<[u8]>`, `[u8; N]`), laid out as StrKeys.  Equality and
    order are the String ones; only the placement differs: `<[u8]>::hash` writes the length before the bytes, so key k
    goes to partition vb_get_partition_bytes(k) (MetroHash64_1(le64(len) ‖ k) % R).  Context.parallelize over it gives
    a StrPairRdd / StrRdd whose shuffles place keys so (VB_STRKEY_BYTES); their keys come back as bytes."""

    @staticmethod
    def from_bytes(items):
        """Concatenate Python bytes / bytearray keys into (offsets, bytes) on the host."""
        items = [bytes(b) for b in items]
        if not all(isinstance(b, bytes) for b in items):
            raise TypeError("BytesKeys.from_bytes takes bytes keys")
        offsets = np.zeros(len(items) + 1, dtype=np.uint64)
        np.cumsum(np.fromiter((len(b) for b in items), dtype=np.uint64, count=len(items)), out=offsets[1:])
        return BytesKeys(offsets, np.frombuffer(b"".join(items), dtype=np.uint8))

    def to_bytes(self):
        """The keys as Python bytes."""
        return _decode_keys(np.asarray(self.offsets.cpu() if _is_torch(self.offsets) else self.offsets, dtype=np.uint64),
                            self.data.cpu().numpy() if _is_torch(self.data) else self.data, L.VB_STRKEY_BYTES)


_BYTES_KEYS_MSG = ("bytes keys: a Rust Vec<u8> hashes with a length prefix, unlike a String; pass str keys, or "
                   "vb.BytesKeys.from_bytes(keys) for Vec<u8> placement")


def _key_kind(x):
    """VB_STRKEY_BYTES for a BytesKeys column (or a _StrCol / an RDD over one), else VB_STRKEY_STR."""
    return getattr(x, "key_kind", L.VB_STRKEY_BYTES if isinstance(x, BytesKeys) else L.VB_STRKEY_STR)


def _is_str_keys(x):
    """True for a StrKeys (or BytesKeys) column or a non-empty sequence / numpy array of str; a sequence of bytes is
    refused: Rust hashes a Vec<u8> with a length prefix, not like a String (BytesKeys places keys that way)."""
    if isinstance(x, StrKeys):
        return True
    if isinstance(x, np.ndarray):
        if x.dtype.kind == "S":
            raise TypeError(_BYTES_KEYS_MSG)
        if x.dtype.kind == "U":
            return True
        if x.dtype.kind != "O" or x.size == 0:
            return False
        first = x.flat[0]
    elif isinstance(x, (list, tuple)) and len(x) > 0:
        first = x[0]
    else:
        return False
    if isinstance(first, (bytes, bytearray)):
        raise TypeError(_BYTES_KEYS_MSG)
    if not isinstance(first, str):
        return False
    if not all(isinstance(k, str) for k in (x.flat if isinstance(x, np.ndarray) else x)):
        raise TypeError("a key column mixes str and other types")
    return True


def _decode_keys(offsets, data, kind=L.VB_STRKEY_STR):
    """Key bytes → numpy object array of Python str (NUL bytes survive, unlike in a numpy 'U' array), or of bytes for
    kind VB_STRKEY_BYTES (never decoded)."""
    raw = data.tobytes()
    o = offsets.astype(np.int64).tolist()
    out = np.empty(len(o) - 1, dtype=object)
    if kind == L.VB_STRKEY_BYTES:
        out[:] = [raw[o[i]:o[i + 1]] for i in range(len(o) - 1)]
    else:
        out[:] = [raw[o[i]:o[i + 1]].decode("utf-8", "surrogateescape") for i in range(len(o) - 1)]
    return out


def _is_bytes_vals(x):
    """True for byte-string values: a StrKeys column, or a non-empty sequence / numpy array of str or bytes."""
    if isinstance(x, StrKeys):
        return True
    if isinstance(x, np.ndarray):
        if x.dtype.kind in "US":
            return x.ndim == 1
        if x.dtype.kind != "O" or x.size == 0:
            return False
        first = x.flat[0]
    elif isinstance(x, (list, tuple)) and len(x) > 0:
        first = x[0]
    else:
        return False
    return isinstance(first, (str, bytes, bytearray))


class _BytesCol:
    """A column of byte-string values at the C ABI (vb_shuffle_map_bytes / vb_shuffle_map_str_bytes): Arrow-style
    offsets + bytes, on the host or as CUDA tensors.  str values (and a StrKeys column) come back as str, bytes as bytes."""

    def __init__(self, x):
        self.as_str = True
        if isinstance(x, StrKeys):
            k = x
            self.as_str = not isinstance(x, BytesKeys)
        else:
            items = x.tolist() if isinstance(x, np.ndarray) else list(x)
            if all(isinstance(v, str) for v in items):
                k = StrKeys.from_strs(items)
            elif all(isinstance(v, (bytes, bytearray)) for v in items):
                self.as_str = False
                offsets = np.zeros(len(items) + 1, dtype=np.uint64)
                np.cumsum(np.fromiter((len(b) for b in items), dtype=np.uint64, count=len(items)), out=offsets[1:])
                k = StrKeys(offsets, np.frombuffer(b"".join(bytes(b) for b in items), dtype=np.uint8))
            else:
                raise TypeError("byte-string values must be all str or all bytes")
        if _is_torch(k.offsets):
            import torch
            torch.cuda.current_stream(k.offsets.device).synchronize()
            self.loc = L.VB_DEVICE
            self.offs_ptr, self.data_ptr = k.offsets.data_ptr(), k.data.data_ptr()
        else:
            self.loc = L.VB_HOST
            self.offs_ptr, self.data_ptr = k.offsets.ctypes.data, k.data.ctypes.data
        self.n_bytes = k.data.shape[0]
        self.n = len(k)
        self.owner = k
        self.code = L.VB_BYTES

    def check_loc(self, key_loc):
        if (key_loc == L.VB_HOST) != (self.loc == L.VB_HOST):
            raise ValueError("keys and values must live in the same memory space")

    def offs_at(self, start):
        return ctypes.c_void_p(self.offs_ptr + 8 * start)

    def data_at(self):
        return ctypes.c_void_p(self.data_ptr) if self.n_bytes else None


class _StrCol:
    """A string key column at the C ABI: offsets / bytes pointers, their location and the row count."""

    def __init__(self, x):
        k = x if isinstance(x, StrKeys) else StrKeys.from_strs(x.tolist() if isinstance(x, np.ndarray) else x)
        if _is_torch(k.offsets):
            import torch
            torch.cuda.current_stream(k.offsets.device).synchronize()
            self.loc = L.VB_DEVICE_BORROWED
            self.offs_ptr, self.data_ptr = k.offsets.data_ptr(), k.data.data_ptr()
            self.n_bytes = k.data.shape[0]
        else:
            self.loc = L.VB_HOST
            self.offs_ptr, self.data_ptr = k.offsets.ctypes.data, k.data.ctypes.data
            self.n_bytes = k.data.shape[0]
        self.n = len(k)
        self.owner = k
        self.rows = False
        self.key_width = 8
        self.code = None
        self.key_kind = _key_kind(k)


class _DevView:
    """Zero-copy view of a library-owned device buffer for torch.as_tensor."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


_TORCH_OF = {"<i8": "int64", "<i4": "int32", "|u1": "uint8"}


def _dev_view(sh, p, n, typestr):
    """A torch view of n elements of a device buffer of sh's library (an empty tensor for n = 0 or a NULL pointer)."""
    import torch
    dev = f"cuda:{sh._lib.vb_ctx_device(sh.sc._h)}"
    if n == 0 or not p.value:
        return torch.empty(0, dtype=getattr(torch, _TORCH_OF[typestr]), device=dev)
    return torch.as_tensor(_DevView(p.value, n, typestr), device=dev)


class StrShuffle(Shuffle):
    """One string-key shuffle (vb_shuffle_create_str; vb_shuffle_create_str_dist for rank `rank` of `world` > 1).
    multi: (value column dtype codes, [(vb_agg, column), ...]) for a combine_by_key shuffle (vb_shuffle_create_str_multi /
    _dist; vcode and agg are then ignored), mapped with map_cols and read with reduce_cols, exchanged with export_cols /
    import_cols.  sort=True: a sort_by_key shuffle (vb_shuffle_create_str_sort; agg is ignored) with one payload column
    of dtype code vcode, or key-only with vcode None; reduce gives each row's key and its payload in key order.  With
    world > 1 (vb_shuffle_create_str_sort_dist) the rows cross ranks through exchange() only, which needs the
    library's communicator (Context.comm_init); rank r then holds the partitions p with p % world == r.
    seal / exchange / stats / free as for Shuffle.  key_kind: VB_STRKEY_STR (Rust String placement) or VB_STRKEY_BYTES
    (Vec<u8> placement, vb_shuffle_set_str_key); keys come back as str or bytes accordingly.  value_order as for Shuffle
    (GROUP shuffles only)."""

    key_kind = L.VB_STRKEY_STR

    def __init__(self, sc, n_map, n_reduce, vcode, agg, hint=0, rank=0, world=1, multi=None, sort=False, key_kind=L.VB_STRKEY_STR,
                 value_order=L.VB_VALORDER_INPUT):
        self.sc, self._lib = sc, sc._lib
        self.key_kind = key_kind
        self.n_map, self.n_reduce, self.agg, self.vcode, self.kcode = n_map, n_reduce, agg, vcode, None
        self.rank, self.world = rank, world
        self.has_payload = True
        self._keepalive = []
        h = ctypes.c_void_p()
        if sort:
            self.agg, self.has_payload = L.VB_AGG_SORT, vcode is not None
            vdt = -1 if vcode is None else vcode
            if vcode == L.VB_BYTES and world == 1:        # a byte-string payload
                L.check(self._lib.vb_shuffle_create_str_sort_bytes(sc._h, sc.new_shuffle_id(), n_map, n_reduce, ctypes.byref(h)))
            elif world > 1:
                L.check(self._lib.vb_shuffle_create_str_sort_dist(sc._h, sc.new_shuffle_id(), n_map, n_reduce, vdt, rank, world,
                                                                  ctypes.byref(h)))
            else:
                L.check(self._lib.vb_shuffle_create_str_sort(sc._h, sc.new_shuffle_id(), n_map, n_reduce, vdt, ctypes.byref(h)))
        elif multi is not None:
            self.agg, self.vcode = L.VB_AGG_SUM, L.VB_U64
            codes, aggs = multi
            dts = (ctypes.c_int32 * len(codes))(*codes)
            spec = (L.vb_agg_col * len(aggs))(*[L.vb_agg_col(a, c) for a, c in aggs])
            if world > 1:
                L.check(self._lib.vb_shuffle_create_str_multi_dist(sc._h, sc.new_shuffle_id(), n_map, n_reduce, len(codes), dts,
                                                                   len(aggs), spec, rank, world, ctypes.byref(h)))
            else:
                L.check(self._lib.vb_shuffle_create_str_multi(sc._h, sc.new_shuffle_id(), n_map, n_reduce, len(codes), dts,
                                                              len(aggs), spec, ctypes.byref(h)))
        elif world > 1:
            L.check(self._lib.vb_shuffle_create_str_dist(sc._h, sc.new_shuffle_id(), n_map, n_reduce, vcode, agg, rank, world,
                                                         ctypes.byref(h)))
        else:
            L.check(self._lib.vb_shuffle_create_str(sc._h, sc.new_shuffle_id(), n_map, n_reduce, vcode, agg, ctypes.byref(h)))
        self._h = h
        sc._shuffles.add(self)
        if key_kind != L.VB_STRKEY_STR:
            L.check(self._lib.vb_shuffle_set_str_key(h, key_kind))
        if hint:
            L.check(self._lib.vb_shuffle_set_hint(h, hint))
        if value_order != L.VB_VALORDER_INPUT:
            L.check(self._lib.vb_shuffle_set_value_order(h, value_order))

    @classmethod
    def bytes_dist(cls, sc, n_map, n_reduce, rank, world, sort=False, hint=0, key_kind=L.VB_STRKEY_STR):
        """vb_shuffle_create_str_bytes_dist (GROUP; cogroup and the joins read it), or with sort=True
        vb_shuffle_create_str_sort_bytes_dist (sort_by_key with a byte-string payload), on rank `rank` of `world`.  Map it
        with byte-string values; exchange a GROUP one with export_bytes / import_bytes or exchange(), a sort with
        exchange() only.  Its results are references, gathered with gather()."""
        self = cls.__new__(cls)
        self.sc, self._lib = sc, sc._lib
        self.n_map, self.n_reduce, self.vcode, self.kcode = n_map, n_reduce, L.VB_BYTES, None
        self.agg = L.VB_AGG_SORT if sort else L.VB_AGG_GROUP
        self.rank, self.world = rank, world
        self.has_payload, self._keepalive = True, []
        h = ctypes.c_void_p()
        create = self._lib.vb_shuffle_create_str_sort_bytes_dist if sort else self._lib.vb_shuffle_create_str_bytes_dist
        L.check(create(sc._h, sc.new_shuffle_id(), n_map, n_reduce, rank, world, ctypes.byref(h)))
        self._h = h
        sc._shuffles.add(self)
        self.key_kind = key_kind
        if key_kind != L.VB_STRKEY_STR:
            L.check(self._lib.vb_shuffle_set_str_key(h, key_kind))
        if hint:
            L.check(self._lib.vb_shuffle_set_hint(h, hint))
        return self

    def export_bytes(self):
        """vb_shuffle_export_str_bytes_prepare + buffers (bytes_dist GROUP, world > 1): ((n_keys, n_key_bytes, n_vals,
        n_val_bytes), (key_lens, key_bytes, val_counts, val_lens, val_bytes)).  The counts are lists with one entry per
        destination rank; the columns are torch views of the library's device buffers (int32 lengths and counts, uint8
        bytes), destination-major, valid until seal."""
        W = self.world
        cs = [(ctypes.c_uint64 * W)() for _ in range(4)]
        L.check(self._lib.vb_shuffle_export_str_bytes_prepare(self._h, *cs))
        counts = tuple([int(x) for x in c] for c in cs)
        ptrs = [ctypes.c_void_p() for _ in range(5)]
        L.check(self._lib.vb_shuffle_export_str_bytes_buffers(self._h, *[ctypes.byref(p) for p in ptrs]))
        K, B, V, VB = (sum(c) for c in counts)
        return counts, (_dev_view(self, ptrs[0], K, "<i4"), _dev_view(self, ptrs[1], B, "|u1"), _dev_view(self, ptrs[2], K, "<i4"),
                        _dev_view(self, ptrs[3], V, "<i4"), _dev_view(self, ptrs[4], VB, "|u1"))

    def import_bytes(self, key_lens, key_bytes, val_counts, val_lens, val_bytes, n_keys, n_key_bytes, n_vals, n_val_bytes):
        """vb_shuffle_import_str_bytes: the received columns (torch CUDA tensors, source-rank major) and what every source
        rank sent.  The key columns are kept alive until seal; the values are copied by the call."""
        _sync_torch(key_lens, key_bytes, val_counts, val_lens, val_bytes)
        self._keepalive.append((key_lens, key_bytes, val_counts))
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
        arr = lambda c: (ctypes.c_uint64 * len(c))(*c)
        L.check(self._lib.vb_shuffle_import_str_bytes(self._h, p(key_lens), p(key_bytes), p(val_counts), p(val_lens), p(val_bytes),
                                                      arr(n_keys), arr(n_key_bytes), arr(n_vals), arr(n_val_bytes)))

    @classmethod
    def narrow(cls, parent, out_col, vcode):
        """vb_shuffle_create_narrow_str: the sealed String reduce or combine result `parent` (output column out_col) as a
        sealed String GROUP side under the same partitioner, each key with the one-element list [its result] (vcode:
        the column's dtype)."""
        self = cls.__new__(cls)
        self.sc, self._lib = parent.sc, parent._lib
        self.n_map, self.n_reduce, self.agg, self.vcode, self.kcode = 0, parent.n_reduce, L.VB_AGG_GROUP, vcode, None
        self.rank, self.world = parent.rank, parent.world
        self.has_payload, self._keepalive = True, []
        self.key_kind = parent.key_kind                   # the library gives the view its parent's kind too
        h = ctypes.c_void_p()
        L.check(self._lib.vb_shuffle_create_narrow_str(parent._h, out_col, ctypes.byref(h)))
        self._h = h
        self.sc._shuffles.add(self)
        return self

    def export(self):
        """vb_shuffle_export_str_prepare + buffers (world > 1): ((n_keys, n_key_bytes, n_vals), (key_lens, key_bytes,
        val_counts, vals)).  The counts are lists with one entry per destination rank; the columns are torch views of
        the library's device buffers (int32 lengths and counts, uint8 bytes, int64 values; val_counts is None for
        reduce ops), destination-major and valid until seal."""
        import torch
        W = self.world
        nk, nb, nv = (ctypes.c_uint64 * W)(), (ctypes.c_uint64 * W)(), (ctypes.c_uint64 * W)()
        L.check(self._lib.vb_shuffle_export_str_prepare(self._h, nk, nb, nv))
        counts = tuple([int(x) for x in c] for c in (nk, nb, nv))
        ptrs = [ctypes.c_void_p() for _ in range(4)]
        L.check(self._lib.vb_shuffle_export_str_buffers(self._h, *[ctypes.byref(p) for p in ptrs]))
        dev = f"cuda:{self._lib.vb_ctx_device(self.sc._h)}"
        K, B, V = sum(counts[0]), sum(counts[1]), sum(counts[2])
        group = self.agg == L.VB_AGG_GROUP

        def view(p, n, typestr, dtype):
            if n == 0 or not p.value:
                return torch.empty(0, dtype=dtype, device=dev)
            return torch.as_tensor(_DevView(p.value, n, typestr), device=dev)
        cols = (view(ptrs[0], K, "<i4", torch.int32), view(ptrs[1], B, "|u1", torch.uint8),
                view(ptrs[2], K, "<i4", torch.int32) if group else None, view(ptrs[3], V, "<i8", torch.int64))
        return counts, cols

    def import_(self, key_lens, key_bytes, val_counts, vals, n_keys, n_key_bytes, n_vals):
        """vb_shuffle_import_str: the received columns (torch CUDA tensors, source-rank major) and the counts every
        source rank sent.  The tensors are kept alive until seal."""
        import torch
        ts = [t for t in (key_lens, key_bytes, val_counts, vals) if t is not None]
        for t in ts:
            if t.is_cuda:
                torch.cuda.current_stream(t.device).synchronize()   # the library reads on its own stream
                break
        self._keepalive.append(tuple(ts))
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None and t.numel() else None
        arr = lambda c: (ctypes.c_uint64 * len(c))(*c)
        L.check(self._lib.vb_shuffle_import_str(self._h, p(key_lens), p(key_bytes), p(val_counts), p(vals),
                                                arr(n_keys), arr(n_key_bytes), arr(n_vals)))

    def map(self, map_id, keys, vals, start, stop):
        """Rows [start, stop) of the string key column (and of the values) as map partition map_id."""
        if isinstance(vals, _BytesCol):
            vals.check_loc(keys.loc)
        elif vals is not None and vals.loc != keys.loc:
            raise ValueError("keys and values must live in the same memory space")
        if keys.loc == L.VB_DEVICE_BORROWED:
            self._keepalive.append((keys.owner, vals.owner if vals is not None else None))
        offs = ctypes.c_void_p(keys.offs_ptr + 8 * start)
        data = ctypes.c_void_p(keys.data_ptr) if keys.n_bytes else None
        if isinstance(vals, _BytesCol):
            self.as_str = vals.as_str
            L.check(self._lib.vb_shuffle_map_str_bytes(self._h, map_id, offs, data, keys.n_bytes, vals.offs_at(start), vals.data_at(),
                                                       vals.n_bytes, stop - start, keys.loc))
            return
        L.check(self._lib.vb_shuffle_map_str(self._h, map_id, offs, data, keys.n_bytes,
                                             vals.at(start) if vals is not None else None, stop - start, keys.loc))

    def reduce_size(self, r):
        nk, nb, nv = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        L.check(self._lib.vb_shuffle_reduce_str_size(self._h, r, ctypes.byref(nk), ctypes.byref(nb), ctypes.byref(nv)))
        return nk.value, nb.value, nv.value

    def reduce_raw(self, r):
        """Partition r on the host: (key offsets, key bytes, combined) or (key offsets, key bytes, offsets, values); a sort
        gives (key offsets, key bytes, payload or None), one key per row."""
        nk, nb, nv = self.reduce_size(r)
        ko, kb = np.empty(nk + 1, dtype=np.uint64), np.empty(nb, dtype=np.uint8)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        if self.agg == L.VB_AGG_SORT:
            vals = np.empty(nk, dtype=_NP_OF[self.vcode]) if self.has_payload else None
            L.check(self._lib.vb_shuffle_reduce_str(self._h, r, p(ko), p(kb), p(vals) if vals is not None else None, None, None,
                                                    L.VB_HOST))
            return ko, kb, vals if vals is None else _vals_out(self, vals)
        if self.agg == L.VB_AGG_GROUP:
            offs, vals = np.empty(nk + 1, dtype=np.uint64), np.empty(nv, dtype=_NP_OF[self.vcode])
            L.check(self._lib.vb_shuffle_reduce_str(self._h, r, p(ko), p(kb), None, p(offs), p(vals), L.VB_HOST))
            return ko, kb, offs, _vals_out(self, vals)
        comb = np.empty(nk, dtype=np.uint64 if self.agg == L.VB_AGG_COUNT else _NP_OF[self.vcode])
        L.check(self._lib.vb_shuffle_reduce_str(self._h, r, p(ko), p(kb), p(comb), None, None, L.VB_HOST))
        return ko, kb, comb

    def reduce(self, r):
        """ShuffledRdd::compute(split r): keys as a numpy object array of str, then the combined values, or the CSR
        offsets and values for GROUP."""
        out = self.reduce_raw(r)
        return (_decode_keys(out[0], out[1], self.key_kind),) + out[2:]

    def reduce_device(self, r, out_key_offsets=None, out_key_bytes=None, out_comb=None, out_offs=None, out_vals=None):
        """Partition r into caller-provided torch CUDA tensors (any may be None; sizes from reduce_size)."""
        _sync_torch(out_key_offsets, out_key_bytes, out_comb, out_offs, out_vals)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        L.check(self._lib.vb_shuffle_reduce_str(self._h, r, p(out_key_offsets), p(out_key_bytes), p(out_comb), p(out_offs),
                                                p(out_vals), L.VB_DEVICE))

    # ---- combine_by_key (multi=) ----
    def map_cols(self, map_id, keys, cols, start, stop):
        """Rows [start, stop) of the string key column and of every value column (None: a column no aggregate reads)
        as map partition map_id."""
        if any(c is not None and c.loc != keys.loc for c in cols):
            raise ValueError("keys and values must live in the same memory space")
        if keys.loc == L.VB_DEVICE_BORROWED:
            self._keepalive.append((keys.owner,) + tuple(c.owner for c in cols if c is not None))
        offs = ctypes.c_void_p(keys.offs_ptr + 8 * start)
        data = ctypes.c_void_p(keys.data_ptr) if keys.n_bytes else None
        ptrs = (ctypes.c_void_p * len(cols))(*[c.at(start) if c is not None else None for c in cols])
        L.check(self._lib.vb_shuffle_map_str_cols(self._h, map_id, offs, data, keys.n_bytes, ptrs, stop - start, keys.loc))

    def reduce_cols(self, r, out_dtypes, dst_loc=L.VB_HOST, out_key_offsets=None, out_key_bytes=None, out_aggs=None):
        """Partition r: (key offsets, key bytes, [one array per aggregate]) on the host, or into caller-provided torch
        CUDA tensors with dst_loc=VB_DEVICE (any may be None; sizes from reduce_size)."""
        if dst_loc == L.VB_DEVICE:
            _sync_torch(out_key_offsets, out_key_bytes, *(out_aggs or []))
            p = lambda t: t.data_ptr() if t is not None else None
            ptrs = (ctypes.c_void_p * len(out_aggs))(*[p(t) for t in out_aggs]) if out_aggs else None
            L.check(self._lib.vb_shuffle_reduce_str_cols(self._h, r, p(out_key_offsets), p(out_key_bytes), ptrs, L.VB_DEVICE))
            return out_key_offsets, out_key_bytes, out_aggs
        nk, nb, _ = self.reduce_size(r)
        ko, kb = np.empty(nk + 1, dtype=np.uint64), np.empty(nb, dtype=np.uint8)
        outs = [np.empty(nk, dtype=dt) for dt in out_dtypes]
        ptrs = (ctypes.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
        L.check(self._lib.vb_shuffle_reduce_str_cols(self._h, r, ko.ctypes.data_as(ctypes.c_void_p), kb.ctypes.data_as(ctypes.c_void_p),
                                                     ptrs, L.VB_HOST))
        return ko, kb, outs

    def export_cols(self):
        """vb_shuffle_export_str_cols_prepare + buffers (multi, world > 1): ((n_keys, n_key_bytes), (key_lens, key_bytes,
        accs)).  The counts are lists with one entry per destination rank; the columns are torch views of the library's
        device buffers (int32 lengths, uint8 bytes, int64 accumulators of shape (n_acc, keys)), destination-major, in the
        wire format of include/vega_b200.h and valid until seal."""
        import torch
        W = self.world
        nk, nb = (ctypes.c_uint64 * W)(), (ctypes.c_uint64 * W)()
        L.check(self._lib.vb_shuffle_export_str_cols_prepare(self._h, nk, nb))
        counts = tuple([int(x) for x in c] for c in (nk, nb))
        lp, bp, ap, na = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint32()
        L.check(self._lib.vb_shuffle_export_str_cols_buffers(self._h, ctypes.byref(lp), ctypes.byref(bp), ctypes.byref(ap),
                                                             ctypes.byref(na)))
        dev = f"cuda:{self._lib.vb_ctx_device(self.sc._h)}"
        K, B, A = sum(counts[0]), sum(counts[1]), na.value

        def view(p, n, typestr, dtype):
            if n == 0 or not p.value:
                return torch.empty(0, dtype=dtype, device=dev)
            return torch.as_tensor(_DevView(p.value, n, typestr), device=dev)
        return counts, (view(lp, K, "<i4", torch.int32), view(bp, B, "|u1", torch.uint8),
                        view(ap, A * K, "<i8", torch.int64).view(A, K))

    def import_cols(self, key_lens, key_bytes, accs, n_keys, n_key_bytes):
        """vb_shuffle_import_str_cols: the received columns (torch CUDA tensors, source-rank major; accs of shape
        (n_acc, keys)) and the key and byte counts every source rank sent.  The tensors are kept alive until seal."""
        import torch
        if accs.dim() != 2 or accs.shape[1] != key_lens.numel() or len(n_keys) != self.world or sum(n_keys) != key_lens.numel():
            raise ValueError(f"import of {key_lens.numel()} keys, accumulators of shape {tuple(accs.shape)} and counts "
                             f"{list(n_keys)} on a world of {self.world}: (n_acc, keys) accumulators and one count per rank expected")
        accs = accs.contiguous()
        for t in (key_lens, key_bytes, accs):
            if t.is_cuda:
                torch.cuda.current_stream(t.device).synchronize()   # the library reads on its own stream
                break
        self._keepalive.append((key_lens, key_bytes, accs))
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
        arr = lambda c: (ctypes.c_uint64 * len(c))(*c)
        L.check(self._lib.vb_shuffle_import_str_cols(self._h, p(key_lens), p(key_bytes), p(accs), accs.shape[0],
                                                     arr(n_keys), arr(n_key_bytes)))


def _no_str(what):
    def f(self, *a, **k):
        raise TypeError(f"{what} is not supported for string keys yet (reduce_by_key, count_by_key, group_by_key, "
                        "partition_by_key, combine_by_key, count_by_value and distinct are)")
    return f


class StrShuffledRdd(ShuffledRdd):
    """ShuffledRdd over string keys: collect() gives (keys, combined) or a Grouped whose keys are Python strs."""

    def __init__(self, parent, agg_name, num_splits, hint=0, sort_values=False):
        if num_splits < 1:
            raise ValueError("num_splits must be >= 1")
        if len(getattr(parent, "cols", ())) > 1:
            raise TypeError("a PairRdd with several value columns supports combine_by_key only")
        if agg_name in _REDUCE_AGGS:
            _refuse_bytes(parent, "reduce_by_key / count_by_key")
        self.value_order = _value_order(sort_values, [parent])
        self.parent, self.agg_name, self.num_slices, self.hint = parent, agg_name, num_splits, hint
        self.sc = parent.sc
        self._sh = None

    def _run(self):
        if self._sh is not None:
            return self._sh
        p = self.parent
        starts = slice_starts(p.n, p.num_slices)
        vcode = p.vals.code if p.vals is not None else L.VB_U64
        sh = StrShuffle(self.sc, len(starts) - 1, self.num_slices, vcode, _AGG[self.agg_name], hint=self.hint,
                        key_kind=_key_kind(p.keys), value_order=self.value_order)
        for m in range(len(starts) - 1):
            sh.map(m, p.keys, p.vals, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        self._sh = sh
        return sh

    def compute_device(self, split, **out):
        """compute(split) into caller-provided torch CUDA tensors (see StrShuffle.reduce_device)."""
        self._run().reduce_device(split, **out)

    join = _no_str("join")
    left_outer_join = _no_str("left_outer_join")
    right_outer_join = _no_str("right_outer_join")
    full_outer_join = _no_str("full_outer_join")
    cogroup = _no_str("cogroup")


class StrPairRdd(PairRdd):
    """PairRdd<String, V>: the shuffle ops string keys support; the others raise TypeError before any device work.
    combine_by_key takes value columns given as a tuple (Context.parallelize(keys, n, values=(c0, ...)), one to four
    columns); with several columns it is the only shuffle.  A PairRdd of one plain value array has no combine_by_key."""

    def __init__(self, sc, keys, vals, num_slices, cols=None):
        if vals is None and not cols and keys.n:
            raise ValueError("a PairRdd needs values")
        super().__init__(sc, keys, vals, num_slices, cols=cols)
        self.has_columns = cols is not None

    def combine_by_key(self, aggs, num_splits, hint=0):
        """PairRdd.combine_by_key over `String` keys: the same {name: (op, column)} mapping, one shuffle that encodes
        every key once.  Returns a StrCombinedRdd."""
        if not self.has_columns:
            raise TypeError("combine_by_key over String keys takes value columns given as a tuple: "
                            "Context.parallelize(keys, num_slices, values=(c0, ...))")
        return StrCombinedRdd(self, aggs, num_splits, hint)

    def group_by_key(self, num_splits, sort_values=False):
        """sort_values=True: each key's values ascending in the value dtype's order, as PairRdd.group_by_key."""
        return StrShuffledRdd(self, "group", num_splits, sort_values=sort_values)

    def reduce_by_key(self, op, num_splits, hint=0):
        if op not in ("sum", "min", "max"):
            raise ValueError("reduce_by_key takes a named op: 'sum' | 'min' | 'max' (closures cannot cross the C ABI)")
        return StrShuffledRdd(self, op, num_splits, hint)

    def count_by_key(self, num_splits=None, hint=0):
        return StrShuffledRdd(self, "count", num_splits or self.num_slices, hint)

    def partition_by_key(self, num_splits):
        return _Repartitioned(StrShuffledRdd(self, "group", num_splits))

    def coalesce(self, num_partitions, shuffle=False, starts=None):
        """rdd.rs:386-418 over (String, v) items with one 64-bit value column; returns (str keys, values) per partition."""
        if isinstance(self.vals, _BytesCol) or len(self.cols) != 1:
            raise NotImplementedError("repartition of String-key items with byte-string or several value columns")
        return _repartition(self, num_partitions, shuffle, starts, self.cols, _BytesCol(self.keys.owner), bytes_first=True)

    def subtract_by_key(self, other, num_splits, sort_values=False):
        """PairRdd.subtract_by_key over `String` keys, matched by their bytes: other is a StrPairRdd, a String reduce
        result or a StrCombinedRdd aggregate of the same key kind."""
        return SemiJoinedRdd(StrCoGroupedRdd([self, other], num_splits, sort_values=sort_values), 0, 0b10)

    def semi_join(self, other, num_splits, sort_values=False):
        """PairRdd.semi_join over `String` keys (see subtract_by_key)."""
        return SemiJoinedRdd(StrCoGroupedRdd([self, other], num_splits, sort_values=sort_values), 0b10, 0)

    join = _no_str("join")
    left_outer_join = _no_str("left_outer_join")
    right_outer_join = _no_str("right_outer_join")
    full_outer_join = _no_str("full_outer_join")
    cogroup = _no_str("cogroup")
    sort_by_key = _no_str("sort_by_key")


class StrCombinedRdd(_Base):
    """CombinedRdd over `String` keys (vb_shuffle_create_str_multi): several named aggregates per key in one shuffle.
    compute(r) / collect() give (keys as a numpy object array of str, {name: array}); compute_raw(r) gives (key offsets,
    key bytes, [one array per aggregate]); compute_device(r, ...) writes into torch CUDA tensors."""

    def __init__(self, parent, aggs, num_splits, hint=0):
        self.spec, self.names, self.out_dtypes = _combine_spec(aggs, parent.cols, num_splits)
        self.parent, self.num_slices, self.hint, self.sc = parent, num_splits, hint, parent.sc
        self._sh = None

    def _run(self):
        if self._sh is not None:
            return self._sh
        p = self.parent
        starts = slice_starts(p.n, p.num_slices)
        sh = StrShuffle(self.sc, len(starts) - 1, self.num_slices, L.VB_U64, L.VB_AGG_SUM, hint=self.hint,
                        multi=([c.code for c in p.cols], self.spec), key_kind=_key_kind(p.keys))
        for m in range(len(starts) - 1):
            sh.map_cols(m, p.keys, p.cols, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        self._sh = sh
        return sh

    def aggregate(self, name):
        """The named aggregate as a StrCoGroupedRdd parent: (key, that aggregate's result) rows (StrAggregateRdd)."""
        if name not in self.names:
            raise ValueError(f"no aggregate named {name!r} (the aggregates are {self.names})")
        return StrAggregateRdd(self, name)

    def compute_raw(self, split):
        return self._run().reduce_cols(split, self.out_dtypes)

    def compute(self, split):
        ko, kb, outs = self.compute_raw(split)
        return _decode_keys(ko, kb, self._run().key_kind), dict(zip(self.names, outs))

    def compute_device(self, split, out_key_offsets=None, out_key_bytes=None, out_aggs=None):
        """compute(split) into caller-provided torch CUDA tensors (any may be None; sizes from the shuffle's
        reduce_size): key offsets [n_keys + 1], key bytes, and one tensor per aggregate in the order given."""
        return self._run().reduce_cols(split, self.out_dtypes, L.VB_DEVICE, out_key_offsets, out_key_bytes, out_aggs)

    def collect(self):
        parts = [self.compute(r) for r in range(self.num_slices)]
        return (np.concatenate([p[0] for p in parts]),
                {name: np.concatenate([p[1][name] for p in parts]) for name in self.names})

    def stats(self):
        return self._run().stats()


class StrAggregateRdd(_Base):
    """One named aggregate of a StrCombinedRdd as a StrCoGroupedRdd parent (StrCombinedRdd.aggregate(name)), with the
    list [its result] per key.  The combine shuffle runs once and is shared by every aggregate taken from it."""

    def __init__(self, combined, name):
        self.combined, self.name = combined, name
        self.sc, self.num_slices = combined.sc, combined.num_slices

    def _run(self):
        return self.combined._run()

    _result_col = AggregateRdd._result_col


def _parent_key_kind(r):
    """The key kind of a StrCoGroupedRdd parent: of its keys, or of the keys of the shuffle that made it."""
    if isinstance(r, StrAggregateRdd):
        r = r.combined
    return _key_kind(r.parent.keys if isinstance(r, (StrShuffledRdd, StrCombinedRdd)) else r.keys)


class StrCoGroupedRdd(_Base):
    """CoGroupedRdd::new(rdds, HashPartitioner::new(num_splits)) over `String` keys (vb_cogroup_n_str / vb_join_n_str):
    the cogroup and the joins of 1 to 16 parents, with keys matched by their bytes.  A parent is a StrPairRdd, shuffled
    with the Vec-append aggregator, or a String reduce_by_key / count_by_key result or StrCombinedRdd.aggregate(name),
    with the list [its result] per key.  Such a result's partition r already holds the keys with
    vb_hash_str(key) % num_splits == r, each once, so under the same num_splits it joins through a view of the sealed
    result (vb_shuffle_create_narrow_str: vega's OneToOneDependency, co_grouped_rdd.rs:103-112) with no second shuffle;
    under another num_splits its partitions are read on the device and shuffled again.  The methods are CoGroupedRdd's,
    with keys as a numpy object array of str:
      compute(r) -> (keys, [(offsets, values) per parent]);  collect() -> [(k, [vs_0, ..., vs_{n-1}])]
      join_compute(r) / join_collect() -> (k, [v_0, ..., v_{n-1}]), one k per row
      outer_join_compute(r, required) / outer_join_collect(required): optional parents as numpy.ma.MaskedArray
    join_raw(r, required) returns the device's keyed form without decoding: (key offsets, key bytes, row offsets,
    [values], [validity or None]), each key once with its rows [row_offsets[i], row_offsets[i + 1]).
    sort_values=True: every StrPairRdd parent's lists ascending in its value dtype's order."""

    key_kind = L.VB_STRKEY_STR           # the parents' key kind (all alike: __init__ refuses a mix)

    def __init__(self, rdds, num_splits, sort_values=False):
        rdds = list(rdds)
        if not 1 <= len(rdds) <= L.VB_MAX_COGROUP_SIDES:
            raise ValueError(f"a cogroup takes 1 to {L.VB_MAX_COGROUP_SIDES} parents, got {len(rdds)}")
        if num_splits < 1:
            raise ValueError("num_splits must be >= 1")
        for j, r in enumerate(rdds):
            if isinstance(r, StrShuffledRdd):
                if r.agg_name not in _REDUCE_AGGS:
                    raise TypeError(f"parent {j}: a {r.agg_name} result is not a join parent (reduce_by_key and "
                                    "count_by_key results are)")
            elif isinstance(r, StrCombinedRdd):
                raise TypeError(f"parent {j}: a combine_by_key result joins one aggregate at a time (.aggregate(name))")
            elif not isinstance(r, (StrPairRdd, StrAggregateRdd)):
                raise TypeError(f"parent {j} is not a String-key PairRdd, reduce result or combine_by_key aggregate")
        if any(r.sc is not rdds[0].sc for r in rdds):
            raise TypeError("the parents live on different contexts")
        kinds = [_parent_key_kind(r) for r in rdds]
        if any(k != kinds[0] for k in kinds):      # equal bytes sit in different partitions under the two hashes
            raise TypeError("the parents mix String keys and BytesKeys (Vec<u8>) keys: they are placed by different hashes")
        self.key_kind = kinds[0]
        self.value_order = _value_order(sort_values, rdds)
        self.rdds, self.num_slices, self.sc = rdds, num_splits, rdds[0].sc
        self._shs = None

    _required_mask = CoGroupedRdd._required_mask

    def _side(self, r):
        """The sealed string GROUP shuffle over num_splits partitions this parent gives."""
        if isinstance(r, StrPairRdd):
            return StrShuffledRdd(r, "group", self.num_slices, sort_values=self.value_order == L.VB_VALORDER_ASC)._run()
        sh = r._run()
        col, n_cols, vcode = r._result_col(sh)
        if sh.n_reduce == self.num_slices:
            return StrShuffle.narrow(sh, col, vcode)
        return self._reshuffled(sh, col, n_cols, vcode)

    def _reshuffled(self, sh, col, n_cols, vcode):
        """Result column `col` of the sealed shuffle sh shuffled again over num_splits partitions, one map task per result
        partition read on the device."""
        import torch
        dev = f"cuda:{sh._lib.vb_ctx_device(self.sc._h)}"
        out = StrShuffle(self.sc, sh.n_reduce, self.num_slices, vcode, L.VB_AGG_GROUP, key_kind=self.key_kind)
        for p in range(sh.n_reduce):
            nk, nb, _ = sh.reduce_size(p)
            ko = torch.empty(nk + 1, dtype=torch.int64, device=dev)
            kb = torch.empty(nb, dtype=torch.uint8, device=dev)
            v = torch.empty(nk, dtype=torch.int64, device=dev)
            if n_cols is None:
                sh.reduce_device(p, out_key_offsets=ko, out_key_bytes=kb, out_comb=v)
            else:
                sh.reduce_cols(p, None, L.VB_DEVICE, ko, kb, [v if c == col else None for c in range(n_cols)])
            out.map(p, _StrCol((BytesKeys if self.key_kind == L.VB_STRKEY_BYTES else StrKeys)(ko, kb)), _Col(v, role="value"), 0, nk)
        out.seal()
        return out

    def _sides(self):
        if self._shs is None:
            self._shs = [self._side(r) for r in self.rdds]
        return self._shs, (ctypes.c_void_p * len(self._shs))(*[s._h.value for s in self._shs])

    def compute_raw(self, split):
        """Partition `split` of the cogroup without decoding: (key offsets, key bytes, [(offsets, values) per parent])."""
        shs, sides = self._sides()
        n, lib = len(shs), self.sc._lib
        nk, nb, nv = ctypes.c_uint64(), ctypes.c_uint64(), (ctypes.c_uint64 * n)()
        L.check(lib.vb_cogroup_n_str_size(sides, n, split, ctypes.byref(nk), ctypes.byref(nb), nv))
        ko, kb = np.empty(nk.value + 1, dtype=np.uint64), np.empty(nb.value, dtype=np.uint8)
        offs = [np.empty(nk.value + 1, dtype=np.uint64) for _ in shs]
        vals = [np.empty(nv[j], dtype=_NP_OF[s.vcode]) for j, s in enumerate(shs)]
        ptrs = lambda xs: (ctypes.c_void_p * n)(*[x.ctypes.data for x in xs])
        L.check(lib.vb_cogroup_n_str(sides, n, split, ko.ctypes.data_as(ctypes.c_void_p), kb.ctypes.data_as(ctypes.c_void_p),
                                     ptrs(offs), ptrs(vals), L.VB_HOST))
        return ko, kb, list(zip(offs, [_vals_out(s, v) for s, v in zip(shs, vals)]))

    def compute(self, split):
        ko, kb, lists = self.compute_raw(split)
        return _decode_keys(ko, kb, self.key_kind), lists

    def collect(self):
        out = []
        for r in range(self.num_slices):
            keys, lists = self.compute(r)
            lists = [(o.tolist(), v) for o, v in lists]
            out.extend((k, [v[o[i]:o[i + 1]] for o, v in lists]) for i, k in enumerate(keys.tolist()))
        return out

    def join_raw(self, split, required):
        """Partition `split` of the join in the device's keyed form: (key offsets, key bytes, row offsets, [values],
        [validity, None for a required parent])."""
        mask = self._required_mask(required)
        shs, sides = self._sides()
        n, lib = len(shs), self.sc._lib
        nr, nk, nb = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        L.check(lib.vb_join_n_str_size(sides, n, split, mask, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)))
        ko, kb = np.empty(nk.value + 1, dtype=np.uint64), np.empty(nb.value, dtype=np.uint8)
        ro = np.empty(nk.value + 1, dtype=np.uint64)
        vs = [np.empty(nr.value, dtype=_NP_OF[s.vcode]) for s in shs]
        valid = [None if mask >> j & 1 else np.empty(nr.value, dtype=np.uint8) for j in range(n)]
        ptrs = lambda xs: (ctypes.c_void_p * n)(*[x.ctypes.data if x is not None else None for x in xs])
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
        L.check(lib.vb_join_n_str(sides, n, split, mask, p(ko), p(kb), p(ro), ptrs(vs), ptrs(valid), L.VB_HOST))
        vs = [v if s.vcode != L.VB_BYTES else s.gather(v, ok) for s, v, ok in zip(shs, vs, valid)]   # bytes: None where invalid
        return ko, kb, ro, vs, valid

    def outer_join_compute(self, split, required):
        """Partition `split` of the outer join of all parents: (k, [v_0, ..., v_{n-1}]) with one key per row; see
        CoGroupedRdd.outer_join_compute."""
        ko, kb, ro, vs, valid = self.join_raw(split, required)
        keys = _decode_keys(ko, kb, self.key_kind)
        k = np.repeat(keys, np.diff(ro.astype(np.int64))) if len(keys) else np.empty(0, dtype=object)
        return k, [v if ok is None or v.dtype == object else np.ma.MaskedArray(v, mask=ok == 0) for v, ok in zip(vs, valid)]

    def outer_join_collect(self, required):
        mask = self._required_mask(required)
        parts = [self.outer_join_compute(r, mask) for r in range(self.num_slices)]
        cat = lambda xs: np.ma.concatenate(xs) if isinstance(xs[0], np.ma.MaskedArray) else np.concatenate(xs)
        return np.concatenate([p[0] for p in parts]), [cat([p[1][j] for p in parts]) for j in range(len(self.rdds))]

    _semi_masks = CoGroupedRdd._semi_masks

    def semi_join_raw(self, split, required, excluded=0):
        """Partition `split` of the semi / anti join of parent 0 (vb_semi_join_n_str) in the keyed form: (key offsets,
        key bytes, row offsets, values), each kept key once with its rows [row_offsets[i], row_offsets[i + 1])."""
        req, exc = self._semi_masks(required, excluded)
        shs, sides = self._sides()
        n, lib = len(shs), self.sc._lib
        nr, nk, nb = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
        L.check(lib.vb_semi_join_n_str_size(sides, n, split, req, exc, ctypes.byref(nr), ctypes.byref(nk), ctypes.byref(nb)))
        ko, kb = np.empty(nk.value + 1, dtype=np.uint64), np.empty(nb.value, dtype=np.uint8)
        ro = np.empty(nk.value + 1, dtype=np.uint64)
        v = np.empty(nr.value, dtype=_NP_OF[shs[0].vcode])
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
        L.check(lib.vb_semi_join_n_str(sides, n, split, req, exc, p(ko), p(kb), p(ro), p(v), L.VB_HOST))
        return ko, kb, ro, _vals_out(shs[0], v)

    def semi_join_compute(self, split, required, excluded=0):
        """CoGroupedRdd.semi_join_compute over `String` keys: (keys, values), one key per row."""
        ko, kb, ro, v = self.semi_join_raw(split, required, excluded)
        keys = _decode_keys(ko, kb, self.key_kind)
        return (np.repeat(keys, np.diff(ro.astype(np.int64))) if len(keys) else np.empty(0, dtype=object)), v

    def semi_join_collect(self, required, excluded=0):
        req, exc = self._semi_masks(required, excluded)
        parts = [self.semi_join_compute(r, req, exc) for r in range(self.num_slices)]
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

    def join_compute(self, split):
        """Partition `split` of the inner join of all parents: (k, [v_0, ..., v_{n-1}])."""
        return self.outer_join_compute(split, (1 << len(self.rdds)) - 1)

    def join_collect(self):
        return self.outer_join_collect((1 << len(self.rdds)) - 1)


class StrSortedRdd(_Base):
    """sort_by_key over `String` keys (PairRdd::sort_by_key, and Rdd::sort for a key-only parent) through
    vb_shuffle_create_str_sort: rows ascending by key in Rust `String` order (bytes compared unsigned, a proper prefix
    first), equal keys in input order, partitions contiguous key ranges cut as the integer sort cuts them.  parent: a
    StrPairRdd of one value column (moved bit for bit; byte-string values come back as str or bytes), or a StrRdd
    (key-only).
      compute(r) -> (keys as a numpy object array of str, values), or the keys alone;  collect(): partitions in order
      compute_raw(r) -> (key offsets, key bytes, values or None), one key per row
      compute_device(r, out_key_offsets=, out_key_bytes=, out_vals=): into torch CUDA tensors sized from the shuffle's
      reduce_size (rows, key bytes)."""

    def __init__(self, parent, num_splits):
        if isinstance(parent, StrPairRdd):
            if len(parent.cols) != 1:
                raise TypeError("sort_by_key over String keys takes one value column")
            vals = parent.cols[0]
        elif isinstance(parent, StrRdd):
            vals = None
        else:
            raise TypeError("StrSortedRdd takes a String-key PairRdd or Rdd (integer keys: PairRdd.sort_by_key / Rdd.sort)")
        if num_splits < 1:
            raise ValueError("num_splits must be >= 1")
        self.parent, self.vals, self.num_slices, self.sc = parent, vals, num_splits, parent.sc
        self._sh = None

    def _run(self):
        if self._sh is not None:
            return self._sh
        p = self.parent
        starts = slice_starts(p.n, p.num_slices)
        sh = StrShuffle(self.sc, len(starts) - 1, self.num_slices, self.vals.code if self.vals is not None else None, L.VB_AGG_SORT,
                        sort=True, key_kind=_key_kind(p.keys))
        for m in range(len(starts) - 1):
            sh.map(m, p.keys, self.vals, int(starts[m]), int(starts[m + 1]))
        sh.seal()
        self._sh = sh
        return sh

    def compute_raw(self, split):
        return self._run().reduce_raw(split)

    def compute(self, split):
        ko, kb, vals = self.compute_raw(split)
        keys = _decode_keys(ko, kb, _key_kind(self.parent.keys))
        return keys if self.vals is None else (keys, vals)

    def compute_device(self, split, out_key_offsets=None, out_key_bytes=None, out_vals=None):
        self._run().reduce_device(split, out_key_offsets=out_key_offsets, out_key_bytes=out_key_bytes, out_comb=out_vals)

    def collect(self):
        parts = [self.compute_raw(r) for r in range(self.num_slices)]
        keys = np.concatenate([_decode_keys(ko, kb, _key_kind(self.parent.keys)) for ko, kb, _ in parts])
        if self.vals is None:
            return keys
        return keys, np.concatenate([v for _, _, v in parts])

    def stats(self):
        return self._run().stats()


class StrRdd(Rdd):
    """Rdd<String>: count_by_value and distinct; the other shuffle ops raise TypeError before any device work."""

    def count_by_value(self):
        n_splits = len(slice_starts(self.n, self.num_slices)) - 1
        return StrShuffledRdd(_StrKeysOnly(self), "count", n_splits)

    def distinct(self, num_partitions=None):
        n_splits = num_partitions or (len(slice_starts(self.n, self.num_slices)) - 1)
        return _Distinct(StrShuffledRdd(_StrKeysOnly(self), "count", n_splits))

    distinct_with_num_partitions = distinct

    def coalesce(self, num_partitions, shuffle=False, starts=None):
        """rdd.rs:386-418 over String items; partitions come back as object arrays of str."""
        return _repartition(self, num_partitions, shuffle, starts, (), _BytesCol(self.keys.owner))

    sort = _no_str("sort")
    intersection = _no_str("intersection")
    intersection_with_num_partitions = intersection
    subtract = _no_str("subtract")
    subtract_with_num_partition = subtract
    group_by = _no_str("group_by")
    group_by_with_num_partitions = group_by


class _StrKeysOnly:
    """(x, ()) rows of a StrRdd: the COUNT shuffle reads no values."""

    def __init__(self, rdd):
        self.sc, self.keys, self.vals, self.num_slices, self.n = rdd.sc, rdd.keys, None, rdd.num_slices, rdd.n
