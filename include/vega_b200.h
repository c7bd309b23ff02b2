/*
 * vega_b200.h — C ABI of libvega_b200.so: an H100-native (sm_90a) shuffle + aggregation
 * engine that drops in behind rajasekarv/vega's RDD operator API for the path
 *   group_by_key / reduce_by_key / join (cogroup) / partition_by_key  (+ sort_by_key, new).
 *
 * The reference has no FFI today (SURVEY.md F4); these entry points are what a thin Rust
 * `extern "C"` shim binds at the four trait seams (INTEGRATION.md shows the shim):
 *
 *   vb_shuffle_create      <- ShuffleDependency::new              src/dependency.rs:133-149
 *                             + MapOutputTracker::register_shuffle src/map_output_tracker.rs:168
 *   vb_shuffle_map_*       <- ShuffleDependencyTrait::do_shuffle_task  src/dependency.rs:96,164-229
 *                             (called from ShuffleMapTask::run, src/shuffle/shuffle_map_task.rs:86-90)
 *   vb_get_partition       <- HashPartitioner::get_partition      src/partitioner.rs:54-57 (+ hash :21-25)
 *   vb_shuffle_seal        <- register_map_outputs ("all map outputs registered")
 *                             src/scheduler/base_scheduler.rs:304-316
 *   vb_shuffle_reduce*     <- ShuffledRdd::compute                src/rdd/shuffled_rdd.rs:149-170
 *                             + ShuffleFetcher::fetch             src/shuffle/shuffle_fetcher.rs:16-119
 *   vb_join*               <- CoGroupedRdd::compute               src/rdd/co_grouped_rdd.rs:206-249
 *                             + PairRdd::join cross product       src/rdd/pair_rdd.rs:104-121
 *   vb_join_outer*         <- nothing: vega has no outer joins (Spark's left/right/full outer join, new)
 *   vb_cogroup*            <- CoGroupedRdd::compute for PairRdd::cogroup  src/rdd/co_grouped_rdd.rs:206-249
 *   vb_cogroup_n* / vb_join_n*
 *                          <- CoGroupedRdd::compute with any number of parents (co_grouped_rdd.rs:75-135, 206-249)
 *   vb_join_n_outer*       <- nothing: vega has no outer joins (N-way, over the same cogroup, new)
 *   vb_cogroup_n_str* / vb_join_n_str*
 *                          <- the same two over `String` keys (keys matched by their bytes; join keys once per key)
 *   vb_semi_join_n*        <- nothing: vega has no semi or anti join (subtractByKey, left semi join; the rule is
 *                             restated over CoGroupedRdd::compute, src/rdd/co_grouped_rdd.rs:206-249, new)
 *   vb_shuffle_free        <- (the reference never evicts SHUFFLE_CACHE, src/env.rs:27)
 *   vb_slice               <- ParallelCollection::slice           src/rdd/parallel_collection_rdd.rs:116-145
 *   vb_shuffle_export_* / vb_shuffle_import
 *                          <- the shuffle data plane (hyper HTTP GET /shuffle/{sid}/{map}/{reduce},
 *                             src/shuffle/shuffle_manager.rs:176-251) when reduce partitions live on
 *                             other GPUs: rows packed by destination rank for one all-to-all-v.
 *
 * Conventions: plain pointers and sizes only.  Every call returns 0 (VB_OK) or a negative
 * vb_status; vb_last_error() gives a thread-local message.  No panics/exceptions cross the
 * boundary (the reference unwrap()s, dependency.rs:191-214).  Host pointers are caller-owned;
 * device memory is library-owned unless passed in as VB_DEVICE*.  Entry points may be called
 * concurrently from arbitrary OS threads (vega runs map tasks on a tokio blocking pool,
 * src/scheduler/local_scheduler.rs:336-352).  A context serialises the ENQUEUEING of its device work; a map
 * call with host input waits for its own completion with the context unlocked, its H2D copies run on a
 * separate copy stream through two staging halves, so concurrent map tasks keep PCIe and the SMs busy together.
 * Device work runs on the context's own stream (vb_ctx_stream): device buffers handed in must be complete
 * (producer stream synchronised) before the call; results are complete when a call returns.
 * There is NO CPU fallback: without a CUDA device every compute entry returns VB_ERR_CUDA.
 *
 * Rows are POD (K,V) with 64-bit K and V, or byte-string V (VB_BYTES) for the ops that only move values;
 * `Aggregator` closures (src/aggregator.rs:8-16) are replaced by named ops (vb_agg).  Arbitrary K, values that
 * are computed on, and closures stay on vega's CPU path.
 */
#ifndef VEGA_B200_H
#define VEGA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VB_API __attribute__((visibility("default")))

typedef struct vb_ctx vb_ctx;   /* one CUDA device: streams, memory pool */
typedef struct vb_shuf vb_shuf; /* one shuffle_id: map outputs + sealed reduce-side results */

enum vb_status {
    VB_OK = 0,
    VB_ERR_INVALID = -1,     /* bad argument */
    VB_ERR_CUDA = -2,        /* CUDA runtime/driver error, or no device */
    VB_ERR_OOM = -3,         /* device or host allocation failed */
    VB_ERR_STATE = -4,       /* wrong phase (map after seal, reduce of a freed shuffle, ...) */
    VB_ERR_UNSUPPORTED = -5, /* dtype/agg combination not implemented */
    VB_ERR_TOO_LARGE = -6    /* more than 2^32-2 rows in one device-local shuffle / map partition */
};

/* VB_BYTES: byte-string values (a value dtype only), see "byte-string values" below. */
enum vb_dtype { VB_U64 = 0, VB_I64 = 1, VB_F64 = 2, VB_BYTES = 3 };

/* Aggregator (src/aggregator.rs).  GROUP = Default (Vec append, :33-52); SUM/MIN/MAX =
 * reduce_by_key(f) (src/rdd/pair_rdd.rs:65-80) for the named f; COUNT = count_by_value
 * (src/rdd/rdd.rs:450-459; values ignored, combiner is u64); COGROUP = the Vec-append
 * aggregator CoGroupedRdd installs per parent (src/rdd/co_grouped_rdd.rs:78-124), same
 * layout as GROUP; SORT = sort_by_key (absent from the reference, SURVEY.md F2).
 * u64/i64 SUM wraps (two's complement); u64 MIN/MAX compare unsigned, i64 MIN/MAX signed.
 * f64 MIN/MAX fold Rust's f64::min / f64::max over a key's values: a NaN value is ignored,
 * the result is NaN only when every value of the key is NaN (payload unspecified), and
 * -0.0 < +0.0, so the result does not depend on the order of the rows.
 * f64 SUM adds a key's values in an unspecified order (any tree of IEEE round-to-nearest
 * additions), from the additive identity -0.0.  The result is NaN if a value is NaN or both
 * +inf and -inf occur; else +inf (-inf) if +inf (-inf) occurs, or NaN when the finite values
 * of the other sign can overflow in some order.  A zero sum is -0.0 exactly when every value
 * is -0.0 (vega folds from the first value: -0.0 + -0.0 = -0.0), else +0.0.  Otherwise, when
 * every partial sum is representable (all values multiples of 2^q, sum |x| <= 2^(53+q)), it
 * is the exact sum bit for bit in every order; else it is within gamma(m-1) * sum |x| of
 * the exact sum (m values, gamma(k) = k*2^-53 / (1 - k*2^-53)), and may also be +-inf (or
 * NaN, when both signs can) when the positive (negative) values' sum times 1 + gamma(m-1)
 * reaches the overflow threshold 2^1024 - 2^970.
 * SORT over f64 keys orders them by f64::total_cmp (-NaN < -inf < ... < -0.0 < +0.0 < ...
 * < +inf < +NaN); "equal keys", which a range cut never separates, are bit-equal keys.     */
enum vb_agg {
    VB_AGG_GROUP = 0,
    VB_AGG_SUM = 1,
    VB_AGG_MIN = 2,
    VB_AGG_MAX = 3,
    VB_AGG_COUNT = 4,
    VB_AGG_COGROUP = 5,
    VB_AGG_SORT = 6,
    VB_AGG_MEAN = 7     /* vb_agg_col only */
};

/* VB_PART_HASH_METRO64: MetroHash64_1(key LE bytes, seed 0) % n_reduce (src/partitioner.rs:21-25,
 * 54-57; fasthash 0.4.0).  VB_PART_RANGE: contiguous key ranges (VB_AGG_SORT only).         */
enum vb_part { VB_PART_HASH_METRO64 = 0, VB_PART_RANGE = 1 };

/* where a caller buffer lives */
enum vb_loc {
    VB_HOST = 0,           /* host memory (pageable or pinned); copied inside the call */
    VB_DEVICE = 1,         /* device memory; consumed or copied before the call returns */
    VB_DEVICE_BORROWED = 2 /* device memory the caller keeps alive and unchanged until seal */
};

typedef struct vb_stats {
    uint64_t rows_in;          /* rows submitted through vb_shuffle_map_* */
    uint64_t rows_out;         /* result rows (distinct keys, or values for group ops) */
    uint64_t kernel_launches;  /* CUDA kernels this shuffle launched (ours, not memcpy/memset) */
    uint64_t h2d_bytes;        /* host→device bytes copied by the library */
    uint64_t d2h_bytes;        /* device→host bytes copied by the library */
    uint64_t table_slots;      /* largest hash-table capacity used */
    uint64_t table_restarts;   /* map tasks restarted with a larger table */
    double hot_kernel_ms;      /* summed device time of the dominant kernel (profiling on) */
    uint64_t hot_kernel_launches;
    uint64_t hot_kernel_rows;  /* rows those launches processed */
    double map_ms;             /* device time inside vb_shuffle_map_* (profiling on) */
    double seal_ms;            /* device time inside vb_shuffle_seal (profiling on) */
    uint64_t hot_kernel_variant; /* reduce ops: 1 = bulk-staged hash_agg (cp.async.bulk + mbarrier), 0 = register-staged */
} vb_stats;

/* ---- context ------------------------------------------------------------------------- */
VB_API int32_t vb_ctx_create(int32_t device_id, vb_ctx **out);
VB_API int32_t vb_ctx_destroy(vb_ctx *ctx);
VB_API int32_t vb_ctx_synchronize(vb_ctx *ctx);
/* profiling: bracket kernels with CUDA events on the launching stream (vb_stats *_ms) */
VB_API int32_t vb_ctx_set_profile(vb_ctx *ctx, int32_t on);
VB_API int32_t vb_ctx_device(vb_ctx *ctx);
/* the cudaStream_t all device work of this context is launched on (for event timing) */
VB_API void *vb_ctx_stream(vb_ctx *ctx);
/* bytes currently held by the context's (private) device memory pool / high-water mark */
VB_API int32_t vb_ctx_mem_info(vb_ctx *ctx, uint64_t *reserved, uint64_t *high_water);
/* give pool memory beyond keep_bytes back to the device (the pool otherwise keeps everything it ever used) */
VB_API int32_t vb_ctx_trim(vb_ctx *ctx, uint64_t keep_bytes);

/* ---- shuffle lifecycle ---------------------------------------------------------------- */
VB_API int32_t vb_shuffle_create(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce,
                                 int32_t key_dtype, int32_t val_dtype, int32_t agg, int32_t part,
                                 vb_shuf **out);
/* Hash the key as 4 LE bytes (Rust i32/u32 keys, widened to 64 bits by the caller) or 8. */
VB_API int32_t vb_shuffle_set_key_width(vb_shuf *s, uint32_t bytes);
/* Optional: expected number of distinct keys (sizes the first hash table; any value is safe). */
VB_API int32_t vb_shuffle_set_hint(vb_shuf *s, uint64_t expected_distinct);
/* One-process-per-GPU mode: this process is `rank` of `world`; reduce partition r is owned by
 * rank r % world.  Must precede the first map call.  world == 1 is the default.              */
VB_API int32_t vb_shuffle_set_dist(vb_shuf *s, uint32_t rank, uint32_t world);
/* Order of the values inside each key's list of a GROUP or COGROUP shuffle.  VB_VALORDER_INPUT, the default: map-id
 * order (source-rank major across ranks).  VB_VALORDER_ASC: ascending in the value dtype's order, sorted on the device
 * right after the reduce side's CSR is built — u64 unsigned, i64 signed, f64 as f64::total_cmp (-NaN < -inf < ... <
 * -0.0 < +0.0 < ... < +inf < +NaN, NaNs by payload), so two values tie only when their bits are equal.  Keys, bucket
 * and value offsets are those of the same shuffle in input order; only the order inside each list changes, and with
 * it everything that reads the lists: vb_shuffle_reduce(_str), the blobs, vb_cogroup(_n)(_str) and every join's
 * nested-loop order (the internal sides of a join inherit the setting of the shuffle they are cut from).
 * Accepted by integer VB_AGG_GROUP / VB_AGG_COGROUP shuffles (vb_shuffle_create, the _dist creates) with u64, i64 or
 * f64 values and by GROUP shuffles of vb_shuffle_create_str(_dist) of either key kind, before the first map, blob or
 * import call (VB_ERR_STATE after one, or after seal).  VB_ERR_UNSUPPORTED for VB_BYTES values; VB_ERR_INVALID for an
 * unknown order and for any other shuffle (reduce ops, combine_by_key, sort, repartition, narrow views), checked
 * before the state.  Across ranks the setting applies where a partition is sealed, on the rank that owns it; the
 * export side does not sort.  Every rank of a shuffle is expected to set the same order: it is not checked.        */
enum vb_value_order { VB_VALORDER_INPUT = 0, VB_VALORDER_ASC = 1 };
VB_API int32_t vb_shuffle_set_value_order(vb_shuf *s, int32_t order /*vb_value_order*/);

/* do_shuffle_task for one map partition.  AoS = the reference's native Vec<(K,V)> layout
 * (16-byte rows); SoA = separate key/value arrays (vals may be NULL for VB_AGG_COUNT and
 * key-only VB_AGG_SORT).  Re-submitting a map_id overwrites it (stage resubmission,
 * src/scheduler/local_scheduler.rs:248-256).  AoS rows on the device must start on a 16-byte
 * boundary (VB_ERR_INVALID otherwise); host rows may start anywhere.                         */
VB_API int32_t vb_shuffle_map_aos(vb_shuf *s, uint32_t map_id, const void *rows, uint64_t n_rows, int32_t src_loc);
VB_API int32_t vb_shuffle_map_soa(vb_shuf *s, uint32_t map_id, const void *keys, const void *vals,
                                  uint64_t n_rows, int32_t src_loc);

/* world > 1 only.  export_prepare finishes the local map side and packs rows by destination
 * rank (combined rows for reduce ops, raw rows in map order for group ops); counts[world] gets
 * rows per destination.  export_buffers returns the packed device arrays (destination-major).
 * The host exchanges them (one all-to-all-v over NCCL) and hands the received rows, source-rank
 * major, to vb_shuffle_import (the buffers are borrowed until vb_shuffle_seal returns).  Then vb_shuffle_seal.
 * A VB_AGG_SORT shuffle is refused (VB_ERR_UNSUPPORTED): a multi-rank sort_by_key goes through vb_shuffle_exchange. */
VB_API int32_t vb_shuffle_export_prepare(vb_shuf *s, uint64_t *counts);
VB_API int32_t vb_shuffle_export_buffers(vb_shuf *s, void **keys_dev, void **vals_dev);
VB_API int32_t vb_shuffle_import(vb_shuf *s, const void *keys_dev, const void *vals_dev, const uint64_t *counts);

/* Fused exchange for GROUP/COGROUP shuffles (world > 1, one process per GPU on one NVLink/NVSwitch node):
 * the destination-rank partition kernel stores every row straight into the HBM of the rank that owns its
 * reduce partition (peer memory mapped with CUDA IPC), so there is no pack buffer and no separate
 * collective — the transfer overlaps the partitioning tile by tile.  Protocol (vega_b200/dist.py drives it):
 *   1. vb_shuffle_export_counts(s, counts[world])        rows this rank sends to each rank (histogram only)
 *   2. ranks all-gather the counts; each reserves its receive arena for sum_src counts[src][me] rows
 *      (16 B/row: keys[total] then vals[total]) with vb_ctx_arena_reserve -> 64-byte IPC handle + generation
 *   3. ranks all-gather the handles; vb_ctx_peer_open(ctx, peer, handle, generation, is_self) maps them (cached
 *      per generation; is_self != 0 for the caller's own rank)
 *   4. vb_shuffle_export_direct(s, dst_row_offset[world], dst_total_rows[world]) runs the scatter; it returns when
 *      this rank's stores are complete; the host then barriers all ranks
 *   5. vb_shuffle_import_arena(s, counts_from_each_src[world]); vb_shuffle_seal(s)
 * The arena is reused (and only grows) across shuffles of the context; a shuffle must be sealed before the
 * next one's export_direct targets the same arena.                                                            */
VB_API int32_t vb_ctx_arena_reserve(vb_ctx *ctx, uint64_t bytes, void *handle_out /*64 bytes*/, uint64_t *generation);
VB_API int32_t vb_ctx_peer_open(vb_ctx *ctx, uint32_t peer_rank, const void *handle /*64 bytes*/, uint64_t generation, int32_t is_self);
VB_API int32_t vb_shuffle_export_counts(vb_shuf *s, uint64_t *counts);
VB_API int32_t vb_shuffle_export_direct(vb_shuf *s, const uint64_t *dst_row_offset, const uint64_t *dst_total_rows);
VB_API int32_t vb_shuffle_import_arena(vb_shuf *s, const uint64_t *counts);

/* Free the arenas vb_ctx_arena_reserve outgrew.  Call after the barrier that follows the exchange: by then every
 * peer has re-opened this rank's current arena (vb_ctx_peer_open closes its mapping of the old one) — freeing an
 * exported allocation a peer still has mapped is undefined.                                                    */
VB_API int32_t vb_ctx_arena_release_retired(vb_ctx *ctx);

/* ---- the exchange itself, behind the C ABI (ShuffleFetcher::fetch, src/shuffle/shuffle_fetcher.rs:16-119;
 *      the tracker hand-shake it replaces: src/map_output_tracker.rs:168-265) ---------------------------------
 * One process per GPU.  vb_comm_unique_id (rank 0) produces the 128-byte NCCL unique id; the host bootstrap
 * (vega's tracker channel, torch.distributed, the TCP rendezvous in vega_b200/rendezvous.py, ...) hands it to every rank; vb_ctx_comm_init is
 * collective over the `world` ranks.  Then, per shuffle, instead of export_prepare / buffers / import:
 *
 *     vb_shuffle_map_*(...)  ...  vb_shuffle_exchange(s, VB_XCHG_AUTO);  vb_shuffle_seal(s);
 *
 * vb_shuffle_exchange is collective and runs entirely on the library's stream:
 *   VB_XCHG_NCCL  pack rows by destination rank (combined rows for reduce ops), all-gather the world x world
 *                 count matrix (one small collective + one D2H), then ONE ncclGroupStart .. ncclSend/ncclRecv
 *                 .. ncclGroupEnd carrying keys and values of every peer (a single all-to-all-v).
 *   VB_XCHG_P2P   GROUP/COGROUP: the fused exchange above — the partition kernel stores into the peers'
 *                 arenas; counts, arena sizes/generations ride one all-gather, IPC handles a second one only
 *                 when some arena had to grow; a stream-ordered all-gather is the closing barrier.
 *   VB_XCHG_AUTO  P2P for group ops, NCCL for reduce ops.
 * NCCL is dlopen'ed (libnccl.so.2) on first use.  vb_ctx_destroy / vb_ctx_comm_destroy are collective when a
 * communicator exists (peer mappings are closed before the arenas are freed).                                 */
#define VB_UNIQUE_ID_BYTES 128
enum vb_xchg { VB_XCHG_AUTO = 0, VB_XCHG_NCCL = 1, VB_XCHG_P2P = 2 };
typedef struct vb_xstats {
    uint64_t sent_rows;     /* rows that left this rank (excluding rows it keeps) */
    uint64_t recv_rows;
    uint64_t exchanges;
    double exchange_ms;     /* device time of the exchange (profiling on): NCCL group, or counts+scatter+barrier for P2P */
    int32_t kind;           /* vb_xchg actually used */
    int32_t pad;
    double prepare_wall_ms; /* host wall clock: finish the map side + pack by destination (merge, multisplit, their syncs) */
    double counts_wall_ms;  /* host wall clock: count all-gather + D2H */
    double post_wall_ms;    /* host wall clock: buffers + enqueueing the grouped send/recv (or handles + scatter + barrier) */
} vb_xstats;
VB_API int32_t vb_comm_unique_id(void *id_out /*VB_UNIQUE_ID_BYTES*/);
VB_API int32_t vb_ctx_comm_init(vb_ctx *ctx, const void *unique_id, uint32_t rank, uint32_t world);
VB_API int32_t vb_ctx_comm_destroy(vb_ctx *ctx);
VB_API int32_t vb_ctx_comm_info(vb_ctx *ctx, uint32_t *rank, uint32_t *world, int32_t *nccl_version);
VB_API int32_t vb_shuffle_exchange(vb_shuf *s, int32_t mode);
VB_API int32_t vb_shuffle_exchange_stats(vb_shuf *s, vb_xstats *out);

/* All map outputs are registered: run the reduce side for every partition this rank owns.
 * world == 1: every map_id in [0, n_map) must have been submitted.                          */
VB_API int32_t vb_shuffle_seal(vb_shuf *s);
VB_API int32_t vb_shuffle_is_sealed(vb_shuf *s);

/* ShuffledRdd::compute for one reduce partition.  Both calls BLOCK until the shuffle is sealed
 * (the reference polls the map-output tracker, src/map_output_tracker.rs:122-132,220-231).
 *   reduce ops : out_keys[n_keys], out_combined[n_keys]            (n_vals == 0)
 *   group ops  : out_keys[n_keys], out_offsets[n_keys+1], out_vals[n_vals]  (CSR; each key's
 *                values in input order: map-id order, then encounter order — tests/test_pair_rdd.rs:30-36)
 *   sort       : out_keys[n_keys] ascending, out_combined[n_keys] = payload (if any)
 * Key order within a partition is unspecified (the reference's is HashMap order).
 * NULL output pointers are skipped.  dst_loc: VB_HOST or VB_DEVICE.                          */
VB_API int32_t vb_shuffle_reduce_size(vb_shuf *s, uint32_t reduce_id, uint64_t *n_keys, uint64_t *n_vals);
VB_API int32_t vb_shuffle_reduce(vb_shuf *s, uint32_t reduce_id, void *out_keys, void *out_combined,
                                 uint64_t *out_offsets, void *out_vals, int32_t dst_loc);

/* ---- combine_by_key: several named aggregates per key in one shuffle (PairRdd::combine_by_key,
 *      src/rdd/pair_rdd.rs:20-33, with a combiner of up to VB_MAX_AGGS named fields) --------------------------
 * Rows are a key column plus n_val_cols value columns (SoA only) of dtypes val_dtypes[].  Aggregate a is op
 * aggs[a].agg folded over input column aggs[a].src, independently for every key:
 *   SUM / MIN / MAX follow the vb_agg rules of that column's dtype (wrapping integer sums, unsigned / signed
 *         compares, f64 MIN/MAX as f64::min / f64::max with NaN ignored); output dtype = the column's dtype.
 *   COUNT rows of the key (src ignored); output u64.
 *   MEAN  f64: for u64 / i64 columns (double)S / (double)n, S = the 64-bit wrapping sum read with the column's
 *         signedness, so it is exact only while the key's sum does not wrap; for f64 columns the f64 SUM (the
 *         vb_agg rules: NaN, +-inf and a zero's sign included) / (double)n, so an all -0.0 key averages to -0.0.
 * A MEAN keeps a SUM accumulator and shares one COUNT accumulator (the spec's own COUNT if it has one, else an
 * internal one); that internal COUNT counts against VB_MAX_AGGS.  Keys are placed by MetroHash64_1(k) % n_reduce,
 * the same partition as any single-column shuffle of the same keys; vb_shuffle_set_key_width / set_hint apply.
 * VB_ERR_INVALID: more than VB_MAX_VAL_COLS columns or VB_MAX_AGGS aggregates, src out of range, or a GROUP /
 * COGROUP / SORT op.  Several ranks: vb_shuffle_create_multi_dist and the _cols export / import calls below.  Not
 * supported (VB_ERR_UNSUPPORTED): vb_shuffle_set_dist with world > 1, the single-column export / import and P2P calls,
 * the bincode blob calls, AoS rows (vb_shuffle_map_aos).  vb_shuffle_map_soa returns VB_ERR_INVALID;
 * vb_shuffle_reduce returns the keys only (VB_ERR_INVALID with out_combined != NULL); the join calls return
 * VB_ERR_INVALID; vb_shuffle_reduce_size / seal / stats / kernel_time / free work as for any reduce shuffle.   */
#define VB_MAX_VAL_COLS 4
#define VB_MAX_AGGS 8
typedef struct vb_agg_col {
    int32_t agg; /* VB_AGG_SUM / MIN / MAX / COUNT / MEAN */
    int32_t src; /* input value column (ignored by COUNT) */
} vb_agg_col;
VB_API int32_t vb_shuffle_create_multi(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t key_dtype,
                                       uint32_t n_val_cols, const int32_t *val_dtypes, uint32_t n_aggs, const vb_agg_col *aggs,
                                       vb_shuf **out);
/* one map partition: keys[n_rows] and vals[c][n_rows] for c < n_val_cols (a column no aggregate reads may be NULL) */
VB_API int32_t vb_shuffle_map_cols(vb_shuf *s, uint32_t map_id, const void *keys, const void *const *vals, uint64_t n_rows,
                                   int32_t src_loc);
/* one reduce partition: out_keys[n_keys] and out_aggs[a][n_keys] per aggregate (NULL entries are skipped) */
VB_API int32_t vb_shuffle_reduce_cols(vb_shuf *s, uint32_t reduce_id, void *out_keys, void *const *out_aggs, int32_t dst_loc);
/* combine_by_key across ranks (one process per GPU; ShuffleFetcher::fetch of the combiners, shuffle_fetcher.rs:16-119).
 * vb_shuffle_create_multi_dist is vb_shuffle_create_multi for rank `rank` of `world` (1 <= world <= 256, VB_ERR_INVALID
 * otherwise); world == 1 gives the same shuffle as vb_shuffle_create_multi.  Placement is unchanged: partition
 * MetroHash64_1(k) % n_reduce with the shuffle's key width, owned by rank r % world.  Each rank runs its map tasks
 * (vb_shuffle_map_cols, any src_loc, resubmission allowed), then:
 *   vb_shuffle_export_cols_prepare  finishes the local map side (merges the map tables) and packs one row per distinct
 *                                   key by destination rank; counts[world] gets the rows going to each rank.
 *   vb_shuffle_export_cols_buffers  the device columns, destination-major, owned by the library until seal (NULL output
 *                                   pointers are skipped); n_acc gets the accumulator count.  This is the wire format:
 *                                     keys  u64 [rows]
 *                                     accs  u64 [n_acc][rows]   accumulator a of row i at accs[a * rows + i], rows = the
 *                                                               sum of counts; each the rank's partial in plain value form:
 *                                       SUM, and a MEAN's sum   the wrapping u64 sum, or the f64 sum
 *                                       COUNT (the spec's, or   the partial count
 *                                       the internal one a MEAN adds after the aggregates)
 *                                       MIN / MAX               the rank's result in the column's dtype; f64: NaN when all
 *                                                               the rank's values of the key were NaN
 *                                   Accumulator a is aggregate a's; n_acc = n_aggs, plus 1 for the internal COUNT.
 *   vb_shuffle_import_cols          the received columns, source-rank major, accs as [n_acc][n] with n = the sum of
 *                                   counts (what each source sent); borrowed until vb_shuffle_seal returns.  Then seal.
 * The seal merges the partials with merge_combiners (partial COUNTs summed, SUM added, MIN / MAX by their vb_agg rules)
 * and finalizes as the one-process seal does, so every owner's partitions equal those of the one-process
 * vb_shuffle_create_multi shuffle over the same map tasks, whatever `world` is (f64 SUM and MEAN up to summation
 * order).  Partitions a rank does not own are empty on it.
 * vb_shuffle_exchange(s, VB_XCHG_AUTO or VB_XCHG_NCCL) does all of it on the library's stream: export, one all-gather of
 * the counts and a fingerprint of the spec (n_acc, every accumulator's op and order transform, key width, n_reduce),
 * one grouped send/recv of the key column and the n_acc accumulator columns.  Ranks whose specs differ all return
 * VB_ERR_INVALID before any send; VB_XCHG_P2P, and any exchange of a world-1 shuffle, is VB_ERR_UNSUPPORTED.
 * Errors: the _cols calls on a multi-aggregate shuffle of world 1: VB_ERR_STATE (VB_ERR_INVALID on any other shuffle);
 * import before export, twice, or after seal: VB_ERR_STATE; map after export: VB_ERR_STATE; seal without import:
 * VB_ERR_STATE; an n_acc that differs from the shuffle's, or a NULL column with a non-zero count: VB_ERR_INVALID; an
 * import of 2^32 - 2 rows or more: VB_ERR_TOO_LARGE, from the counts.                                                  */
VB_API int32_t vb_shuffle_create_multi_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t key_dtype,
                                            uint32_t n_val_cols, const int32_t *val_dtypes, uint32_t n_aggs, const vb_agg_col *aggs,
                                            uint32_t rank, uint32_t world, vb_shuf **out);
VB_API int32_t vb_shuffle_export_cols_prepare(vb_shuf *s, uint64_t *counts /*[world]*/);
VB_API int32_t vb_shuffle_export_cols_buffers(vb_shuf *s, void **keys, void **accs, uint32_t *n_acc);
VB_API int32_t vb_shuffle_import_cols(vb_shuf *s, const void *keys, const void *accs, uint32_t n_acc, const uint64_t *counts /*[world]*/);

/* A sealed reduce-op or combine_by_key shuffle as a cogroup / join parent under the same partitioner, without a
 * shuffle (CoGroupedRdd::new's OneToOneDependency, co_grouped_rdd.rs:103-112).  *out is a new sealed COGROUP-kind
 * shuffle: its partition r holds partition r of `parent`, each key once, with the one-element list [its result].
 * out_col: the combine_by_key output column (0 for a single-column shuffle).  Blocks until `parent` is sealed.
 *   parents   SUM / MIN / MAX / COUNT shuffles, and any output column of a vb_shuffle_create_multi shuffle (MEAN too).
 *             The view's values are the results bit for bit: the parent's value dtype for SUM / MIN / MAX, u64 for COUNT
 *             and f64 for MEAN.
 *   refused   VB_ERR_INVALID, the parent staying usable: NULL arguments, GROUP / COGROUP parents (their lists are
 *             cogroup sides already; a view is one of them), SORT and string-key parents, out_col out of range.
 *   use       an ordinary sealed group shuffle: vb_shuffle_reduce* gives the parent's keys, offsets 0..n and the
 *             results, and every join / cogroup call takes it as any side, next to COGROUP shuffles and other views.
 *             It has the parent's n_reduce, key width, rank and world: on a rank of a multi-rank shuffle it holds the
 *             partitions that rank owns.
 *   memory    the view owns copies of the keys and of the column (16 B per key) and its key dictionary, so the parent
 *             and the view may be freed in either order; free it with vb_shuffle_free.                              */
VB_API int32_t vb_shuffle_create_narrow(vb_shuf *parent, uint32_t out_col, vb_shuf **out);

/* Inner join of two sealed GROUP/COGROUP shuffles with equal n_reduce, for one partition:
 * per key `for v in left { for w in right }` (src/rdd/pair_rdd.rs:109-115).                  */
VB_API int32_t vb_join_size(vb_shuf *left, vb_shuf *right, uint32_t reduce_id, uint64_t *n_out);
VB_API int32_t vb_join(vb_shuf *left, vb_shuf *right, uint32_t reduce_id, void *out_k, void *out_v, void *out_w,
                       int32_t dst_loc);

/* Outer joins (Spark's leftOuterJoin / rightOuterJoin / fullOuterJoin; the reference has none, so there is no
 * reference output to compare against).  Same arguments and rules as vb_join, plus the kind (VB_ERR_INVALID for any
 * other value: the inner join is vb_join).  For a key with left values vs and right values ws, each in cogroup order:
 *   key on both sides     for v in vs { for w in ws } -> (k, v, w)          every kind
 *   key only on the left  (k, v, None) for each v                           LEFT, FULL
 *   key only on the right (k, None, w) for each w                           RIGHT, FULL
 * so a key gives max(|vs|,1) * max(|ws|,1) rows on the kept sides.  A key's rows are contiguous, in that order; the
 * order of keys within the partition is unspecified.  A None slot holds 0 and its validity byte is 0.
 * out_v_valid / out_w_valid (one byte per row, same dst_loc) are optional: when given, they are written for every
 * row, including the 1s of a side that is always present.  On a rank of a multi-rank shuffle only the partitions
 * that rank owns have rows.                                                                                       */
enum vb_join_kind { VB_JOIN_LEFT = 1, VB_JOIN_RIGHT = 2, VB_JOIN_FULL = 3 };
VB_API int32_t vb_join_outer_size(vb_shuf *left, vb_shuf *right, uint32_t reduce_id, int32_t kind, uint64_t *n_out);
VB_API int32_t vb_join_outer(vb_shuf *left, vb_shuf *right, uint32_t reduce_id, int32_t kind,
                             void *out_k, void *out_v, void *out_w,
                             uint8_t *out_v_valid, uint8_t *out_w_valid, int32_t dst_loc);

/* CoGroupedRdd::compute for PairRdd::cogroup (src/rdd/pair_rdd.rs:123-155, src/rdd/co_grouped_rdd.rs:206-249):
 * partition reduce_id of the cogroup of two sealed GROUP/COGROUP shuffles, as one key list with two CSR value lists.
 *   keys     every key that occurs on either side in the partition, exactly once; the order of keys within the
 *            partition is unspecified (as for vb_shuffle_reduce).
 *   lists    a key's left list is exactly the value list vb_shuffle_reduce of the left shuffle gives for it (map-id
 *            order, then encounter order), and the same holds for the right list.  A key a side lacks has an empty
 *            list on that side.  left == right is allowed and gives two equal lists.
 *   offsets  out_left_offsets / out_right_offsets [n_keys + 1] are relative to the partition and start at 0, as
 *            vb_shuffle_reduce's do: key i's left values are out_left_vals[out_left_offsets[i] .. [i + 1]).
 * The argument rules are vb_join's (two sealed GROUP/COGROUP shuffles with equal n_reduce and key width on the same
 * context, reduce_id < n_reduce; anything else is VB_ERR_INVALID), and the call blocks until both sides are sealed.
 * vb_cogroup_size gives the output sizes (NULL pointers skipped); vb_cogroup writes to dst_loc VB_HOST or VB_DEVICE
 * and skips NULL outputs.  On a rank of a multi-rank shuffle only the partitions that rank owns have keys.         */
VB_API int32_t vb_cogroup_size(vb_shuf *left, vb_shuf *right, uint32_t reduce_id,
                               uint64_t *n_keys, uint64_t *n_left_vals, uint64_t *n_right_vals);
VB_API int32_t vb_cogroup(vb_shuf *left, vb_shuf *right, uint32_t reduce_id, void *out_keys,
                          uint64_t *out_left_offsets /*n_keys+1*/, void *out_left_vals,
                          uint64_t *out_right_offsets /*n_keys+1*/, void *out_right_vals, int32_t dst_loc);

/* CoGroupedRdd::compute with n_sides parents (src/rdd/co_grouped_rdd.rs:75-135, 206-249): partition reduce_id of the
 * cogroup of sides[0 .. n_sides), as one key list with one CSR value list per side, in side order.
 *   keys     every key that occurs on any side in the partition, exactly once; the order of keys within the partition
 *            is unspecified.
 *   lists    side j's list for a key is exactly the value list vb_shuffle_reduce of side j gives for it (map-id order,
 *            then encounter order), and empty where side j lacks the key.
 *   offsets  out_offsets[j] [n_keys + 1] is relative to the partition and starts at 0: key i's values on side j are
 *            out_vals[j][out_offsets[j][i] .. [i + 1]).
 * For n_sides = 2 the keys and lists are those of vb_cogroup(sides[0], sides[1]); for n_sides = 1 those of
 * vb_shuffle_reduce(sides[0]).
 * Argument rules: vb_cogroup's, for every side.  Each side is a sealed GROUP or COGROUP shuffle (the calls block until
 * every side is sealed); all sides have the same n_reduce and key width and live on the same context; none is a
 * string, multi-column or reduce-op shuffle; reduce_id < n_reduce; 1 <= n_sides <= VB_MAX_COGROUP_SIDES.  The same
 * shuffle may appear more than once and then gives equal lists.  Anything else, including a NULL sides array or a NULL
 * entry in it, is VB_ERR_INVALID.  A COGROUP side that was not grouped yet is grouped whole by these calls.
 * vb_cogroup_n_size gives n_keys and the value count of every side (n_vals[n_sides]; NULL pointers skipped);
 * vb_cogroup_n writes to dst_loc VB_HOST or VB_DEVICE and skips NULL outputs: out_offsets / out_vals themselves, or
 * single entries in them.  The size call keeps the partition's plan on sides[0] for the write call, which frees it (so
 * does vb_shuffle_free of sides[0]).  On a rank of a multi-rank shuffle only the partitions that rank owns have keys. */
#define VB_MAX_COGROUP_SIDES 16
VB_API int32_t vb_cogroup_n_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint64_t *n_keys,
                                 uint64_t *n_vals /*[n_sides], may be NULL*/);
VB_API int32_t vb_cogroup_n(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, void *out_keys,
                            uint64_t *const *out_offsets /*[n_sides] arrays of n_keys+1*/,
                            void *const *out_vals /*[n_sides]*/, int32_t dst_loc);

/* Inner join of all sides, for one partition, with vb_cogroup_n's argument rules: a key on every side with lists
 * l_0 .. l_{n-1} (each in cogroup order) gives prod |l_j| rows, contiguous, in the order
 *   for v0 in l0 { for v1 in l1 { ... } } -> (k, v0, v1, ..., v_{n-1})
 * (the last side varies fastest; for n_sides = 2 this is vb_join's per-key order).  A key missing on any side gives no
 * rows; the order of keys within the partition is unspecified.  Row i is (out_k[i], out_vals[0][i], ...,
 * out_vals[n_sides-1][i]).  Once the partition has rows, out_k, out_vals and every entry of it must be non-NULL
 * (VB_ERR_INVALID).  A key's product, or the partition's total, of 2^63 rows or more is VB_ERR_TOO_LARGE from the size
 * call.                                                                                                              */
VB_API int32_t vb_join_n_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint64_t *n_out);
VB_API int32_t vb_join_n(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, void *out_k,
                         void *const *out_vals /*[n_sides]*/, int32_t dst_loc);

/* Outer join of all sides, for one partition (CoGroupedRdd::compute, src/rdd/co_grouped_rdd.rs:206-249, expanded as
 * PairRdd::join does, src/rdd/pair_rdd.rs:104-121; the reference has no outer join, so there is no reference output to
 * compare against).  Bit j of `required` marks side j as required.  A key of the partition, with lists l_0 .. l_{n-1}
 * in cogroup order, gives rows only if every required side has it.  A side that has the key contributes l_j; an
 * optional side that lacks it contributes the single slot [None].  So the key gives prod_j max(|l_j|, 1) rows,
 * contiguous, in the order
 *   for v0 in L0 { for v1 in L1 { ... } } -> (k, v0, v1, ..., v_{n-1})      (the last side varies fastest)
 * and the order of keys within the partition is unspecified.  A None slot holds 0 and its validity byte is 0.
 * required = all sides is vb_join_n; for two sides 0b01 is vb_join_outer LEFT, 0b10 RIGHT and 0 FULL.  For more sides
 * required = 1 is `a LEFT JOIN b LEFT JOIN c ...` on the same key, and 0 the chained full outer join.
 * Argument rules: vb_cogroup_n's, and a required bit at n_sides or above is VB_ERR_INVALID.  Once the partition has
 * rows, out_k, out_vals and every entry of it must be non-NULL (VB_ERR_INVALID).  out_valid [n_sides] (one byte per
 * row, same dst_loc) is optional, and so is each entry: an entry given is written for every row, including the 1s.  A
 * key's product, or the partition's total, of 2^63 rows or more is VB_ERR_TOO_LARGE from the size call.  The size call
 * keeps the plan on sides[0] for the write call, as vb_join_n_size does.  On a rank of a multi-rank shuffle only the
 * partitions that rank owns have rows.                                                                               */
VB_API int32_t vb_join_n_outer_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                                    uint64_t *n_out);
VB_API int32_t vb_join_n_outer(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                               void *out_k, void *const *out_vals /*[n_sides]*/,
                               uint8_t *const *out_valid /*[n_sides] or NULL; entries may be NULL*/, int32_t dst_loc);

/* Semi and anti join of side 0 by the other sides, for one partition.  vega has no such op (Spark's subtractByKey and
 * left semi join); the rule is restated over CoGroupedRdd::compute, src/rdd/co_grouped_rdd.rs:206-249, so there is no
 * reference output to compare against.  `required` and `excluded` are masks over sides 1 .. n_sides-1.  A key of the
 * partition, with cogroup lists l_0 .. l_{n-1}, is kept when l_0 is non-empty, every side of `required` has it and no
 * side of `excluded` has it; a kept key gives the rows (k, v) for v in l_0, contiguous and in l_0's order (map-id order,
 * or ascending under vb_shuffle_set_value_order).  The order of keys within the partition is unspecified.
 *   subtract_by_key(a, b) = {a, b} with excluded = 0b10;  semi_join(a, b) = {a, b} with required = 0b10;
 *   both masks 0 gives side 0's rows as vb_shuffle_reduce gives them.
 * Only side 0's values are read or moved: the other sides' value dtypes are free.  out_v has side 0's value dtype
 * (VB_BYTES: references that vb_shuffle_gather_bytes of side 0 resolves).  Sides: those vb_cogroup_n takes.  A lazy
 * COGROUP filter side gives its rows' keys and is not grouped; a lazy side 0 has only its kept rows grouped.  The
 * filter (one presence dictionary of the filter sides' keys) is built once per (sides, masks) and kept on sides[0].
 * Argument rules: vb_cogroup_n's; and VB_ERR_INVALID, before any device work and with every side staying usable, for a
 * mask bit at n_sides or above, bit 0 in either mask, a side in both masks, or (once the partition has rows) a NULL
 * out_k or out_v.  The size call keeps the partition's plan on sides[0] for the write call, as vb_join_n_size does.  On
 * a rank of a multi-rank shuffle only the partitions that rank owns have rows.                                      */
VB_API int32_t vb_semi_join_n_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                                   uint32_t excluded, uint64_t *n_rows);
VB_API int32_t vb_semi_join_n(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                              uint32_t excluded, void *out_k, void *out_v, int32_t dst_loc);

/* ---- string keys: byte-string keys that hash like Rust `String` (reduce_by_key / count_by_key / count_by_value /
 *      distinct / group_by_key / partition_by_key over `String` keys, examples/group_by.rs, tests/test_pair_rdd.rs:8-37)
 * Key i of a map partition is key_bytes[key_offsets[i] .. key_offsets[i+1]) (Arrow-style: key_offsets has n_rows + 1
 * entries and need not start at 0, so a slice of a larger column is passed as is).  The bytes are not checked for
 * UTF-8; equal keys are byte-equal keys; the empty key and keys containing NUL bytes are ordinary keys.
 *   placement  MetroHash64_1(bytes ‖ 0xFF, seed 0) % n_reduce: `str::hash` (the bytes, then write_u8(0xff)) fed to
 *              the buffering MetroHasher the integer keys already assume (vb_hash_str / vb_get_partition_str).
 *   reduce ops per key, the results and rules of the integer-key shuffle with the same agg and val_dtype (wrapping
 *              integer sums, unsigned / signed MIN and MAX, f64 MIN / MAX as f64::min / f64::max with NaN ignored,
 *              COUNT as u64, vals may be NULL for COUNT).
 *   GROUP      per key, the values in input order (map-id order, then encounter order).
 * Re-submitting a map_id overwrites it: a key only the replaced submission had is not in the output.
 * Limits: fewer than 2^32 - 2 rows per map partition and per shuffle, fewer than 2^31 distinct keys, every key shorter
 * than 2^32 bytes (VB_ERR_TOO_LARGE beyond them).  Key offsets that decrease or exceed n_bytes are VB_ERR_INVALID,
 * for device input too (checked on the device).  Several ranks: vb_shuffle_create_str_dist and the string export /
 * import calls below (vb_shuffle_set_dist with world > 1, the integer export / import / P2P calls, the blob calls on a
 * GROUP shuffle and vb_shuffle_map_blob with world > 1 return VB_ERR_UNSUPPORTED on a string shuffle; the blob calls
 * of the reduce ops are described with them below); vb_shuffle_set_key_width, the integer map and
 * reduce calls and the join / cogroup calls return VB_ERR_INVALID on a string shuffle (vb_cogroup_n_str / vb_join_n_str
 * below join and cogroup string GROUP shuffles), and the string calls return
 * VB_ERR_INVALID on any other shuffle.  seal / is_sealed / stats / kernel_time / set_hint / free work as for any
 * shuffle (table_slots: largest dictionary index, table_restarts: index growths).
 * vb_shuffle_reduce_str_size / vb_shuffle_reduce_str block until the shuffle is sealed and skip NULL outputs; the
 * order of keys within a partition is unspecified.  out_key_offsets [n_keys + 1] start at 0 and index
 * out_key_bytes [n_key_bytes]; out_combined [n_keys] for reduce ops; out_offsets [n_keys + 1] (from 0) and out_vals
 * [n_vals] for GROUP.  dst_loc: VB_HOST or VB_DEVICE.                                                                */
VB_API int32_t vb_shuffle_create_str(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce,
                                     int32_t val_dtype, int32_t agg, vb_shuf **out);
VB_API int32_t vb_shuffle_map_str(vb_shuf *s, uint32_t map_id, const uint64_t *key_offsets /*n_rows+1*/,
                                  const void *key_bytes, uint64_t n_bytes, const void *vals /*NULL for COUNT*/,
                                  uint64_t n_rows, int32_t src_loc);
VB_API int32_t vb_shuffle_reduce_str_size(vb_shuf *s, uint32_t reduce_id, uint64_t *n_keys, uint64_t *n_key_bytes,
                                          uint64_t *n_vals);
VB_API int32_t vb_shuffle_reduce_str(vb_shuf *s, uint32_t reduce_id, uint64_t *out_key_offsets /*n_keys+1*/,
                                     void *out_key_bytes, void *out_combined, uint64_t *out_offsets /*n_keys+1*/,
                                     void *out_vals, int32_t dst_loc);
/* Byte-slice keys: the string-key shuffle placing keys as Rust hashes `Vec<u8>` (HashPartitioner::get_partition,
 * src/partitioner.rs:29-60, over `Vec<u8>`, `&[u8]`, `Box<[u8]>` or `[u8; N]` keys).  `<[u8] as Hash>` writes the
 * length as a usize and then the bytes, so
 *   placement  VB_STRKEY_BYTES: MetroHash64_1(le64(len) ‖ bytes, seed 0) % n_reduce (vb_hash_bytes /
 *              vb_get_partition_bytes); VB_STRKEY_STR, the default: the `String` placement above.
 * Nothing else depends on the kind: keys are equal when their bytes are, sort in `<[u8] as Ord>` order (the `String`
 * order), and bincode writes `Vec<u8>`, `&[u8]` and `Box<[u8]>` as u64 len | bytes, as it writes a `String`, so the
 * reduce-op blobs below are the same bytes for both kinds (a `[u8; N]` is written with no length: not a blob of these).
 * vb_shuffle_set_str_key sets the kind of a shuffle of any vb_shuffle_create_str* call (plain, _dist, _multi(_dist),
 * _sort(_dist), _sort_bytes(_dist), _bytes_dist) before its first map, blob or import call (VB_ERR_STATE after one, or
 * after seal); VB_ERR_INVALID for any other shuffle or kind.  Checked: vb_cogroup_n_str / vb_join_n_str (and _size)
 * refuse sides of different kinds (VB_ERR_INVALID, every side staying usable); vb_shuffle_create_narrow_str gives the
 * view its parent's kind; vb_shuffle_exchange of a reduce-op or combine_by_key shuffle refuses, on every rank and before
 * any send, a rank whose kind differs (VB_ERR_INVALID).  Not checked: the GROUP exchanges and the export / import calls
 * carry no kind, so every rank of a shuffle must set the same one.  A sort places rows by cut keys, not by hash: the
 * kind changes none of its output.                                                                                   */
enum vb_str_key { VB_STRKEY_STR = 0, VB_STRKEY_BYTES = 1 };
VB_API int32_t vb_shuffle_set_str_key(vb_shuf *s, int32_t kind /*vb_str_key*/);
/* Cogroup and join of string-key shuffles, for one partition: vb_cogroup_n and vb_join_n_outer with keys compared as
 * byte strings (CoGroupedRdd::compute over `String` keys, co_grouped_rdd.rs:75-135, 206-249).  Each side is a sealed
 * GROUP shuffle of vb_shuffle_create_str (the calls block until every side is sealed); 1 <= n_sides <=
 * VB_MAX_COGROUP_SIDES, all sides with the same n_reduce on the same context; value dtypes may differ and the same
 * shuffle may appear more than once.  Integer shuffles, string reduce-op shuffles, NULL or out-of-range arguments and
 * a `required` bit at n_sides or above are VB_ERR_INVALID.  The first call that reads a side builds an index of its
 * keys, kept until vb_shuffle_free.
 *   cogroup  vb_cogroup_n's keys and lists: every key of any side in the partition exactly once, in unspecified
 *            order, as out_key_offsets [n_keys + 1] (from 0) into out_key_bytes [n_key_bytes]; side j's list is the
 *            one vb_shuffle_reduce_str of side j gives for the key, empty where side j lacks it.  NULL outputs, or
 *            NULL entries of out_offsets / out_vals, are skipped.
 *   join     vb_join_n_outer's rows: a key gives rows only if every side of `required` has it (all bits set: the inner
 *            join); a side that lacks it gives one None slot (value 0, validity 0); the key's prod max(|l_j|, 1) rows
 *            are contiguous, the last side varying fastest.  The keys are written once each, not once per row: the
 *            n_keys keys of the partition that have rows, in row order, as out_key_offsets / out_key_bytes, and key
 *            i's rows are [out_row_offsets[i], out_row_offsets[i + 1]) of out_vals[j] (out_row_offsets [n_keys + 1],
 *            ending at n_rows).  A caller that wants one (key, v_0, ..., v_{n-1}) per row repeats key i over its
 *            range.  Once the partition has rows, out_key_offsets, out_row_offsets, out_vals and every entry of it,
 *            and out_key_bytes unless n_key_bytes is 0, must be non-NULL (VB_ERR_INVALID); out_valid and its entries
 *            are optional.  A key's product, or the partition's total, of 2^63 rows or more is VB_ERR_TOO_LARGE from
 *            the size call.
 * The size calls keep the partition's plan on sides[0] for the write call, which frees it.  dst_loc: VB_HOST or
 * VB_DEVICE.  Limit: fewer than 2^32 - 1 keys over all sides of one partition.                                     */
VB_API int32_t vb_cogroup_n_str_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint64_t *n_keys,
                                     uint64_t *n_key_bytes, uint64_t *n_vals /*[n_sides], may be NULL*/);
VB_API int32_t vb_cogroup_n_str(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id,
                                uint64_t *out_key_offsets /*n_keys+1*/, void *out_key_bytes,
                                uint64_t *const *out_offsets /*[n_sides] arrays of n_keys+1*/,
                                void *const *out_vals /*[n_sides]*/, int32_t dst_loc);
VB_API int32_t vb_join_n_str_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                                  uint64_t *n_rows, uint64_t *n_keys, uint64_t *n_key_bytes);
VB_API int32_t vb_join_n_str(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                             uint64_t *out_key_offsets /*n_keys+1*/, void *out_key_bytes,
                             uint64_t *out_row_offsets /*n_keys+1*/, void *const *out_vals /*[n_sides] of n_rows*/,
                             uint8_t *const *out_valid /*[n_sides] or NULL; entries may be NULL*/, int32_t dst_loc);
/* vb_semi_join_n over string GROUP shuffles and vb_shuffle_create_narrow_str views, all of one key kind (the same rule,
 * restated over CoGroupedRdd::compute, src/rdd/co_grouped_rdd.rs:206-249; vega has no such op).  Side 0's keys of the
 * partition are looked up in each filter side's key index by their hash, then their bytes, so keys that share a hash
 * stay apart.  The output is vb_join_n_str's with one value column: each kept key once (out_key_offsets [n_keys + 1],
 * out_key_bytes), out_row_offsets [n_keys + 1] its rows, out_vals [n_rows] side 0's values.  Argument rules:
 * vb_join_n_str's and vb_semi_join_n's masks; once the partition has rows out_key_offsets, out_row_offsets, out_vals
 * and (with key bytes) out_key_bytes must be non-NULL.                                                               */
VB_API int32_t vb_semi_join_n_str_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                                       uint32_t excluded, uint64_t *n_rows, uint64_t *n_keys, uint64_t *n_key_bytes);
VB_API int32_t vb_semi_join_n_str(vb_shuf *const *sides, uint32_t n_sides, uint32_t reduce_id, uint32_t required,
                                  uint32_t excluded, uint64_t *out_key_offsets /*n_keys+1*/, void *out_key_bytes,
                                  uint64_t *out_row_offsets /*n_keys+1*/, void *out_vals /*n_rows*/, int32_t dst_loc);
/* A sealed string reduce-op or combine_by_key shuffle as a cogroup / join parent under the same partitioner, without a
 * shuffle: vb_shuffle_create_narrow for string keys.  *out is a new sealed string GROUP-kind shuffle: its partition r
 * holds partition r of `parent` (the keys with vb_hash_str(key) % n_reduce == r), each key once, with the one-element
 * list [its result].  out_col: the combine_by_key output column (0 for a single-aggregate shuffle).  Blocks until
 * `parent` is sealed.
 *   parents   SUM / MIN / MAX / COUNT shuffles of vb_shuffle_create_str(_dist), and any output column of a
 *             vb_shuffle_create_str_multi(_dist) shuffle (MEAN and COUNT too).  The view's values are the column bit for
 *             bit, of the column's output dtype: the value dtype for SUM / MIN / MAX, u64 for COUNT, f64 for MEAN.
 *   refused   VB_ERR_INVALID, the parent staying usable: NULL arguments, integer-key parents (vb_shuffle_create_narrow
 *             takes those), string GROUP parents (a view is one), string sort parents, out_col out of range.  A string
 *             reduce shuffle itself stays refused by vb_cogroup_n_str / vb_join_n_str: the view is the side.
 *   use       an ordinary sealed string GROUP shuffle: vb_shuffle_reduce_str(_size) gives the parent's keys, offsets
 *             0..n and the column's values, and vb_cogroup_n_str(_size) / vb_join_n_str(_size) take it as any side, next
 *             to GROUP shuffles and other views.  It has the parent's n_reduce, rank and world: on a rank of a multi-rank
 *             shuffle it holds the partitions that rank owns, and the others are empty.  Like any side, its key index is
 *             built by the first cogroup or join that reads it.
 *   memory    the view owns copies of the key offsets, the key bytes and the column (24 B per key plus the key bytes)
 *             and its key index, so the parent and the view may be freed in either order; free it with
 *             vb_shuffle_free.                                                                                        */
VB_API int32_t vb_shuffle_create_narrow_str(vb_shuf *parent, uint32_t out_col, vb_shuf **out);
/* String keys across ranks (one process per GPU; ShuffleFetcher::fetch over `String` keys, shuffle_fetcher.rs:16-119).
 * vb_shuffle_create_str_dist is vb_shuffle_create_str for rank `rank` of `world` (1 <= world <= 256, VB_ERR_INVALID
 * otherwise); world == 1 gives the same shuffle as vb_shuffle_create_str.  Placement is unchanged: partition
 * vb_hash_str(key) % n_reduce, owned by rank r % world.  Each rank runs its map tasks (vb_shuffle_map_str, any src_loc,
 * resubmission allowed), then:
 *   vb_shuffle_export_str_prepare  finishes the local map side and packs it by destination rank; n_keys / n_key_bytes /
 *                                  n_vals [world] get what goes to each rank.  Reduce ops send combined rows: one
 *                                  accumulator per distinct live key (n_vals == n_keys); GROUP sends raw values.
 *   vb_shuffle_export_str_buffers  the four device columns, destination-major, owned by the library until seal (NULL
 *                                  output pointers are skipped).  This is the wire format:
 *                                    key_lens   u32 [keys]    each key's length in bytes
 *                                    key_bytes  u8  [bytes]   the keys' bytes, concatenated in key order
 *                                    val_counts u32 [keys]    GROUP: each key's value count (NULL for reduce ops)
 *                                    vals       u64 [vals]    reduce ops: one accumulator per key (the op's result for
 *                                                             the rank's rows; COUNT: a partial count); GROUP: the
 *                                                             values key by key, each key's run in map order
 *                                  Lengths and counts rather than offsets: slices concatenate without rebasing.
 *   vb_shuffle_import_str          the received columns, source-rank major (concatenated in ascending source rank), with
 *                                  the counts each source sent; borrowed until vb_shuffle_seal returns.  Then seal.
 * The seal merges the received accumulators with merge_combiners (partial COUNTs summed, MIN / MAX / SUM by their
 * vb_agg rules), so every owner's partitions equal those of the one-process shuffle over the same map tasks, whatever
 * `world` is (f64 SUM up to summation order).  GROUP value lists are in source-rank order, which is map-id order when
 * rank r's map ids precede rank r + 1's (vega_b200/dist.py map_block).  Partitions a rank does not own are empty on it;
 * a sealed GROUP shuffle is a side of vb_cogroup_n_str / vb_join_n_str for the partitions the calling rank owns.
 * vb_shuffle_exchange(s, VB_XCHG_AUTO or VB_XCHG_NCCL) does all of it on the library's stream: export, one all-gather of
 * counts per rank, one grouped send/recv of the columns; VB_XCHG_P2P is VB_ERR_UNSUPPORTED.  GROUP gathers 3 x world
 * counts (keys, key bytes, values).  Reduce ops gather 2 x world counts (keys, key bytes) and a fingerprint of the op
 * and its order transform, as vb_shuffle_create_str_multi_dist does: ranks whose op or transform differ all return
 * VB_ERR_INVALID before any send.
 * Errors: the export / import calls on a string shuffle of world 1: VB_ERR_STATE (VB_ERR_INVALID on a non-string
 * shuffle); import before export, twice, or after seal: VB_ERR_STATE; map after export: VB_ERR_STATE; a NULL column
 * whose count is non-zero, or reduce-op counts with n_vals != n_keys: VB_ERR_INVALID; an import of 2^32 - 2 rows or
 * more (keys for reduce ops, values for GROUP) or of 2^31 keys or more: VB_ERR_TOO_LARGE, from the counts; key lengths
 * or value counts that do not add up to the announced totals: VB_ERR_INVALID from the seal.                         */
VB_API int32_t vb_shuffle_create_str_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce,
                                          int32_t val_dtype, int32_t agg, uint32_t rank, uint32_t world, vb_shuf **out);
VB_API int32_t vb_shuffle_export_str_prepare(vb_shuf *s, uint64_t *n_keys /*[world]*/, uint64_t *n_key_bytes /*[world]*/,
                                             uint64_t *n_vals /*[world]*/);
VB_API int32_t vb_shuffle_export_str_buffers(vb_shuf *s, uint32_t **key_lens, void **key_bytes, uint32_t **val_counts,
                                             uint64_t **vals);
VB_API int32_t vb_shuffle_import_str(vb_shuf *s, const uint32_t *key_lens, const void *key_bytes, const uint32_t *val_counts,
                                     const uint64_t *vals, const uint64_t *n_keys /*[world]*/,
                                     const uint64_t *n_key_bytes /*[world]*/, const uint64_t *n_vals /*[world]*/);
/* ---- combine_by_key over string keys: several named aggregates per `String` key in one shuffle (PairRdd::combine_by_key,
 *      src/rdd/pair_rdd.rs:20-33, over `String` keys) -----------------------------------------------------------------
 * vb_shuffle_create_str_multi takes the spec of vb_shuffle_create_multi (1 to VB_MAX_VAL_COLS value columns of VB_U64 /
 * VB_I64 / VB_F64, 1 to VB_MAX_AGGS aggregates of SUM / MIN / MAX / COUNT / MEAN, a MEAN's internal COUNT counted against
 * VB_MAX_AGGS; VB_ERR_INVALID otherwise) and places keys as any string shuffle does: vb_hash_str(key) % n_reduce.  For
 * every key, aggregate a is what vb_shuffle_create_str with op aggs[a].agg over column aggs[a].src gives (integer ops,
 * COUNT and f64 MIN / MAX bit for bit, NaN rules included; f64 SUM up to summation order), and a MEAN is (double)S / n
 * with S read with the column's signedness, as the integer-key combine computes it.  Every key of the input appears
 * exactly once, in its partition; the order of keys within a partition is unspecified.  Re-submitting a map_id replaces
 * its rows (a key only the replaced rows had is dropped).  Limits: those of vb_shuffle_create_str (fewer than 2^32 - 2
 * rows per map partition and per shuffle, fewer than 2^31 distinct keys, keys shorter than 2^32 bytes).
 *   vb_shuffle_map_str_cols    keys as for vb_shuffle_map_str (Arrow-style offsets that may start anywhere, any src_loc)
 *                              and vals[c][n_rows] for c < n_val_cols; a column no aggregate reads may be NULL and is not
 *                              copied (VB_ERR_INVALID for a NULL column that one reads).
 *   vb_shuffle_reduce_str_cols one partition: out_key_offsets [n_keys + 1] (from 0) into out_key_bytes [n_key_bytes], and
 *                              out_aggs[a][n_keys] per aggregate in the output dtype of vb_shuffle_reduce_cols; sizes from
 *                              vb_shuffle_reduce_str_size (n_vals == n_keys); NULL outputs are skipped; blocks until sealed.
 * On this shuffle kind vb_shuffle_map_str, the integer map / reduce / join calls, vb_shuffle_set_key_width,
 * vb_cogroup_n_str / vb_join_n_str, vb_shuffle_create_narrow and the single-column string export / import calls return
 * VB_ERR_INVALID; vb_shuffle_reduce_str returns the keys only (VB_ERR_INVALID with out_combined, out_offsets or out_vals
 * non-NULL); vb_shuffle_set_dist with world > 1, VB_XCHG_P2P and the bincode blob calls return VB_ERR_UNSUPPORTED.  The
 * calls below return VB_ERR_INVALID on any other shuffle.  seal / stats / kernel_time / set_hint / free work as for any
 * string shuffle.
 * Several ranks (one process per GPU): vb_shuffle_create_str_multi_dist is vb_shuffle_create_str_multi for rank `rank` of
 * `world` (1 <= world <= 256, VB_ERR_INVALID otherwise; world == 1 gives the same shuffle as the plain call).  Partition
 * r is owned by rank r % world.  Each rank runs its map tasks, then:
 *   vb_shuffle_export_str_cols_prepare  finishes the local map side and packs one row per distinct live key by
 *                                       destination rank; n_keys / n_key_bytes [world] get what goes to each rank.
 *   vb_shuffle_export_str_cols_buffers  the device columns, destination-major, owned by the library until seal (NULL
 *                                       output pointers are skipped); n_acc gets the accumulator count.  Wire format:
 *                                         key_lens   u32 [keys]          each key's length in bytes
 *                                         key_bytes  u8  [bytes]         the keys' bytes, concatenated in key order
 *                                         accs       u64 [n_acc][keys]   accumulator a of key i at accs[a * keys + i],
 *                                                                        keys = the sum of n_keys; the rank's partials in
 *                                                                        the plain value form of vb_shuffle_export_cols_buffers
 *   vb_shuffle_import_str_cols          the received columns, source-rank major, with the key and byte counts each
 *                                       source sent; borrowed until vb_shuffle_seal returns.  Then seal.
 * The seal merges the partials with merge_combiners and finalizes as the one-process seal does, so every owner's
 * partitions equal those of the one-process shuffle over the same map tasks, whatever `world` is (f64 SUM and MEAN up to
 * summation order); partitions a rank does not own are empty on it.  vb_shuffle_exchange(s, VB_XCHG_AUTO or
 * VB_XCHG_NCCL) does all of it on the library's stream: export, one all-gather of 2 x world counts and the spec's
 * fingerprint (n_acc, every accumulator's op and order transform, n_reduce), one grouped send/recv of the 2 + n_acc
 * columns; ranks whose specs differ all return VB_ERR_INVALID before any send.
 * Errors: the _str_cols export / import calls on a world-1 shuffle, import before export, twice or after seal, map after
 * export, and seal without import: VB_ERR_STATE; an n_acc that differs from the shuffle's, or a NULL column with a
 * non-zero count: VB_ERR_INVALID; an import of 2^31 keys or more: VB_ERR_TOO_LARGE, from the counts; key lengths that do
 * not add up to the announced bytes: VB_ERR_INVALID from the seal.                                                     */
VB_API int32_t vb_shuffle_create_str_multi(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce,
                                           uint32_t n_val_cols, const int32_t *val_dtypes, uint32_t n_aggs,
                                           const vb_agg_col *aggs, vb_shuf **out);
VB_API int32_t vb_shuffle_create_str_multi_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce,
                                                uint32_t n_val_cols, const int32_t *val_dtypes, uint32_t n_aggs,
                                                const vb_agg_col *aggs, uint32_t rank, uint32_t world, vb_shuf **out);
VB_API int32_t vb_shuffle_map_str_cols(vb_shuf *s, uint32_t map_id, const uint64_t *key_offsets /*n_rows+1*/,
                                       const void *key_bytes, uint64_t n_bytes, const void *const *vals /*[n_val_cols]*/,
                                       uint64_t n_rows, int32_t src_loc);
VB_API int32_t vb_shuffle_reduce_str_cols(vb_shuf *s, uint32_t reduce_id, uint64_t *out_key_offsets /*n_keys+1*/,
                                          void *out_key_bytes, void *const *out_aggs /*[n_aggs]*/, int32_t dst_loc);
VB_API int32_t vb_shuffle_export_str_cols_prepare(vb_shuf *s, uint64_t *n_keys /*[world]*/, uint64_t *n_key_bytes /*[world]*/);
VB_API int32_t vb_shuffle_export_str_cols_buffers(vb_shuf *s, uint32_t **key_lens, void **key_bytes, uint64_t **accs,
                                                  uint32_t *n_acc);
VB_API int32_t vb_shuffle_import_str_cols(vb_shuf *s, const uint32_t *key_lens, const void *key_bytes, const uint64_t *accs,
                                          uint32_t n_acc, const uint64_t *n_keys /*[world]*/,
                                          const uint64_t *n_key_bytes /*[world]*/);
/* ---- sort_by_key over string keys (PairRdd::sort_by_key / Rdd::sort over `String` keys, one process) ----------------
 * vb_shuffle_create_str_sort: a sort shuffle of byte-string keys with one payload column of val_dtype (VB_U64 / VB_I64
 * / VB_F64), or key-only with val_dtype -1 (VB_ERR_INVALID otherwise).  The semantics of the integer sort_by_key, with
 * keys in `String` order (`<[u8] as Ord>`: bytes compare unsigned, a proper prefix sorts first; the bytes are not
 * checked for UTF-8):
 *   order      rows ascending by key; equal keys stay in input order (map-id order, then row order).
 *   partitions contiguous ranges: with n rows, cut p (0 < p < n_reduce) is the first row at or after floor(p·n/n_reduce)
 *              where the key changes, so no key is split; partitions may be empty and n_reduce may exceed n.
 *   payload    moved bit for bit (NaN payloads survive).
 * Re-submitting a map_id overwrites it (a key only the replaced rows had is gone).  Limits: those of
 * vb_shuffle_create_str (fewer than 2^32 - 2 rows, fewer than 2^31 distinct keys, keys shorter than 2^32 bytes:
 * VB_ERR_TOO_LARGE beyond them); bad key offsets are VB_ERR_INVALID as for vb_shuffle_map_str.
 *   map     vb_shuffle_map_str; vals must be NULL on a key-only shuffle, and non-NULL with rows otherwise (VB_ERR_INVALID).
 *   read    vb_shuffle_reduce_str_size: n_keys = the partition's rows, n_key_bytes = the bytes of their keys (each row
 *           carries its own copy), n_vals = 0.  vb_shuffle_reduce_str: out_key_offsets [n_keys + 1] (from 0) into
 *           out_key_bytes, and out_combined [n_keys] the payload (NULL outputs are skipped); out_offsets / out_vals must
 *           be NULL, and so must out_combined on a key-only shuffle (VB_ERR_INVALID).  dst_loc: VB_HOST or VB_DEVICE.
 * set_hint / seal / stats / kernel_time / free work as for any shuffle; kernel_time class 8 is the ordering of the
 * distinct keys.  On this kind the integer map / reduce / join calls, vb_cogroup_n_str / vb_join_n_str,
 * vb_shuffle_create_narrow, vb_shuffle_set_key_width and the _str_cols calls return VB_ERR_INVALID; vb_shuffle_set_dist
 * with world > 1 and the export / import / exchange / blob calls return VB_ERR_UNSUPPORTED (across ranks:
 * vb_shuffle_create_str_sort_dist). */
VB_API int32_t vb_shuffle_create_str_sort(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce,
                                          int32_t val_dtype /*VB_U64 / VB_I64 / VB_F64, or -1: key-only*/, vb_shuf **out);
/* vb_shuffle_create_str_sort_dist: vb_shuffle_create_str_sort for rank `rank` of `world` (1 <= world <= 256; world 1
 * is the one-process shuffle), with the same limits and argument checks.  Each rank maps its own map tasks (ascending
 * blocks of map ids, rank order = map-id order); vb_shuffle_exchange(s, VB_XCHG_AUTO or VB_XCHG_NCCL) on a context
 * with vb_ctx_comm_init then sorts locally, agrees on the exact cut keys with the other ranks word by word (only u64
 * words and counts cross), and sends every rank's rows of output partition p to rank p % world in one grouped
 * send/recv; seal re-sorts what arrived.  The partitions a rank owns are then identical, key bytes and payload bits
 * row for row, to those of the one-process shuffle over the same map tasks; the other partitions are empty.
 * Errors, the same on every rank: ranks whose val_dtype or n_reduce differ VB_ERR_INVALID; n_reduce > 4096
 * VB_ERR_UNSUPPORTED; a rank that would receive 2^32 - 2 rows or more, or 2^31 keys or more, VB_ERR_TOO_LARGE.
 * VB_XCHG_P2P, the _str / _str_cols export and import calls and vb_shuffle_set_dist return VB_ERR_UNSUPPORTED (agreeing
 * on the cuts takes several collective rounds); seal at world > 1 without the exchange returns VB_ERR_STATE.
 * vb_shuffle_exchange_stats: prepare_wall_ms the local sort, counts_wall_ms the all-gathers and the cut agreement,
 * post_wall_ms the send/recv; sent_rows / recv_rows count rows.                                                     */
VB_API int32_t vb_shuffle_create_str_sort_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce,
                                               int32_t val_dtype /*VB_U64 / VB_I64 / VB_F64, or -1: key-only*/, uint32_t rank,
                                               uint32_t world, vb_shuf **out);
/* ---- byte-string values: `String` values as their UTF-8 bytes, any `V: Serialize` as its bincode bytes, for the ops
 *      that move values without reading them: group_by_key / partition_by_key / cogroup / the joins (CoGroupedRdd::compute,
 *      src/rdd/co_grouped_rdd.rs:206-249, PairRdd::join, src/rdd/pair_rdd.rs:104-121) and the sort_by_key payload ----
 * VB_BYTES is accepted as the value dtype of vb_shuffle_create with VB_AGG_GROUP / VB_AGG_COGROUP / VB_AGG_SORT and of
 * vb_shuffle_create_str with VB_AGG_GROUP; vb_shuffle_create_str_sort_bytes is sort_by_key over string keys with a
 * byte-string payload (vb_shuffle_create_str_sort's rules; vb_shuffle_create_str_sort keeps refusing val_dtype 3 with
 * VB_ERR_INVALID, as it always has).  Refused: with a reduce op or COUNT (VB_ERR_UNSUPPORTED); as a key dtype, in
 * vb_agg_col specs or _multi value columns (VB_ERR_INVALID); vb_shuffle_create_str_dist and
 * vb_shuffle_create_str_sort_dist with VB_BYTES, vb_shuffle_set_dist with world > 1, the export / import / exchange / P2P
 * calls and the blob calls (VB_ERR_UNSUPPORTED).  Across ranks: the _bytes_dist creates below.
 *   map     vb_shuffle_map_bytes (integer keys, read as by vb_shuffle_map_soa, VB_DEVICE_BORROWED included) and
 *           vb_shuffle_map_str_bytes (string keys, read as by vb_shuffle_map_str).  Value i is val_bytes[val_offsets[i] ..
 *           val_offsets[i + 1]) (Arrow-style: n_rows + 1 offsets that need not start at 0).  The values and their offsets
 *           are always COPIED, whatever src_loc is (VB_DEVICE_BORROWED applies to the keys only).  Offsets that decrease or
 *           exceed n_val_bytes are VB_ERR_INVALID and a value of 2^32 bytes or more VB_ERR_TOO_LARGE, for device input
 *           too.  Re-submitting a map_id replaces its values.  vb_shuffle_map_soa / _aos / _str on a bytes shuffle, and
 *           the bytes calls on any other shuffle, are VB_ERR_INVALID.
 *   values  every output call is unchanged and, where it writes values of a bytes shuffle, writes REFERENCES: opaque
 *           64-bit words (vb_shuffle_reduce(_str) out_vals / out_combined, vb_join*, vb_cogroup*, vb_join_n*_str ...).  A
 *           side's references are gathered from that side's shuffle.  References stay valid until vb_shuffle_free;
 *           the reference 0 is never issued, so the 0 of an outer join's None slot gathers as an empty value (its validity
 *           byte tells None from an empty value).
 *   gather  vb_shuffle_gather_bytes_size gives the total bytes of n references; vb_shuffle_gather_bytes writes
 *           out_offsets [n + 1] (from 0) and out_bytes, value i at out_bytes[out_offsets[i] .. [i + 1]).  Both block until
 *           s is sealed.  refs come from src_loc (VB_HOST or VB_DEVICE); dst_loc is VB_HOST or VB_DEVICE.  A reference s
 *           did not issue, or a NULL out_bytes with bytes to write, is VB_ERR_INVALID before anything is written, and s
 *           stays usable.                           */
VB_API int32_t vb_shuffle_map_bytes(vb_shuf *s, uint32_t map_id, const void *keys, const uint64_t *val_offsets /*n_rows+1*/,
                                    const void *val_bytes, uint64_t n_val_bytes, uint64_t n_rows, int32_t src_loc);
VB_API int32_t vb_shuffle_map_str_bytes(vb_shuf *s, uint32_t map_id, const uint64_t *key_offsets /*n_rows+1*/, const void *key_bytes,
                                        uint64_t n_key_bytes, const uint64_t *val_offsets /*n_rows+1*/, const void *val_bytes,
                                        uint64_t n_val_bytes, uint64_t n_rows, int32_t src_loc);
VB_API int32_t vb_shuffle_create_str_sort_bytes(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, vb_shuf **out);
VB_API int32_t vb_shuffle_gather_bytes_size(vb_shuf *s, const uint64_t *refs, uint64_t n, int32_t src_loc, uint64_t *n_bytes);
VB_API int32_t vb_shuffle_gather_bytes(vb_shuf *s, const uint64_t *refs, uint64_t n, int32_t src_loc,
                                       uint64_t *out_offsets /*n+1, from 0*/, void *out_bytes, int32_t dst_loc);
/* ---- repartition(n) = coalesce(n, shuffle = true) (Rdd::coalesce, src/rdd/rdd.rs:386-418): any item, spread evenly ----
 * The map task of parent partition m gives its items the positions start_m + 1 + i (i = 0, 1, ...; u64 arithmetic mod
 * 2^64), and item i goes to reduce partition vb_get_partition(position, 8, n_reduce), as vega's HashPartitioner::<usize>
 * places it.  start_m is vega's own draw (rdd.rs:393-398), made by the caller; the library draws nothing.  The library
 * fixes the order that vega leaves to a HashMap: partition r holds its items in map-id order, then input order (a stable
 * split), which is one of the orders vega can produce.
 * Items are only moved, never read: n_cols (0 to 2) 64-bit columns, plus one byte-string column if has_bytes (a String
 * as its UTF-8 bytes, any T: Serialize as its bincode bytes); at least one column in all, else VB_ERR_INVALID.
 *   create  vb_shuffle_create_repartition: one process.  n_reduce 1 .. 65536 (VB_ERR_INVALID for 0, VB_ERR_UNSUPPORTED
 *           above).  has_bytes is 0 or 1.  vb_shuffle_create_repartition_dist is the same for rank `rank` of `world`
 *           (1 <= world <= 256, rank < world, VB_ERR_INVALID otherwise; world 1 is the one-process create).  Rank r owns
 *           the partitions p with p % world == r; map ids are assigned in contiguous blocks by rank, and each rank maps its
 *           own block (the maps it never submits are empty).
 *   exchange  world > 1: vb_shuffle_exchange with VB_XCHG_AUTO or VB_XCHG_NCCL (needs vb_ctx_comm_init) between the map
 *           calls and the seal: each partition's items go to their owner, which keeps them in source-rank order, i.e.
 *           map-id order.  VB_XCHG_P2P is VB_ERR_UNSUPPORTED, an exchange of a world-1 shuffle VB_ERR_STATE.  Ranks that
 *           disagree on n_cols or has_bytes, or a rank that would receive 2^32 - 2 items or more, make every rank return
 *           the same code (VB_ERR_INVALID / VB_ERR_TOO_LARGE) before any send; each shuffle can still be freed.  A seal
 *           before the exchange, or a map call after it, is VB_ERR_STATE.
 *   map     vb_shuffle_map_repartition: map task map_id, its items' positions from first_position + 1.  The 64-bit
 *           columns cols[n_cols] follow vb_shuffle_map_soa's rules, VB_DEVICE_BORROWED included (read until seal); the
 *           bytes follow vb_shuffle_map_bytes's rules (Arrow-style offsets, always copied, the same offset checks and
 *           2^32-byte limit; ignored without has_bytes).  Re-submitting a map_id replaces it.  A map task of 2^32 - 2
 *           items or more, or a shuffle of as many, is VB_ERR_TOO_LARGE.
 *   seal    vb_shuffle_seal, once every map id was submitted (VB_ERR_STATE otherwise).
 *   reduce  vb_shuffle_reduce_repartition_size gives partition r's items and, with has_bytes, their total bytes;
 *           vb_shuffle_reduce_repartition writes out_cols[k] (n_rows words each), out_offsets [n_rows + 1] (from 0) and
 *           out_bytes, item i's bytes at out_bytes[out_offsets[i] .. [i + 1]), to dst_loc (VB_HOST or VB_DEVICE; a device
 *           out_bytes may have any alignment).  Any output may be NULL to skip it, except out_bytes when the partition has
 *           bytes and the offsets or bytes are asked for (VB_ERR_INVALID, nothing written).  Both block until s is sealed.
 *   refused VB_ERR_INVALID before any device work, the shuffle staying usable: the repartition calls on any other
 *           shuffle; on a repartition shuffle every other map call (vb_shuffle_map_soa / _aos / _cols / _bytes / _str* /
 *           _blob), reduce call (vb_shuffle_reduce* / _blob*), join, cogroup, narrow, gather and export / import call,
 *           vb_shuffle_set_key_width and vb_shuffle_set_dist.  Seal, stats, kernel_time and free work as for
 *           any shuffle.  A partition a rank does not own has 0 items.                                                    */
VB_API int32_t vb_shuffle_create_repartition(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t n_cols,
                                             int32_t has_bytes, vb_shuf **out);
VB_API int32_t vb_shuffle_create_repartition_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t n_cols,
                                                  int32_t has_bytes, uint32_t rank, uint32_t world, vb_shuf **out);
VB_API int32_t vb_shuffle_map_repartition(vb_shuf *s, uint32_t map_id, uint64_t first_position, const void *const *cols /*n_cols*/,
                                          const uint64_t *val_offsets /*n_rows+1*/, const void *val_bytes, uint64_t n_val_bytes,
                                          uint64_t n_rows, int32_t src_loc);
VB_API int32_t vb_shuffle_reduce_repartition_size(vb_shuf *s, uint32_t r, uint64_t *n_rows, uint64_t *n_bytes);
VB_API int32_t vb_shuffle_reduce_repartition(vb_shuf *s, uint32_t r, void *const *out_cols /*n_cols*/,
                                             uint64_t *out_offsets /*n_rows+1, from 0*/, void *out_bytes, int32_t dst_loc);
/* ---- byte-string values across ranks: each value's bytes are sent once, never its reference --------------------------
 * vb_shuffle_create_bytes_dist        vb_shuffle_create(key_dtype, VB_BYTES, agg, part) for rank `rank` of `world`:
 *                                     agg VB_AGG_GROUP / VB_AGG_COGROUP / VB_AGG_SORT (a reduce op or COUNT is
 *                                     VB_ERR_UNSUPPORTED); vb_shuffle_set_key_width applies.
 * vb_shuffle_create_str_bytes_dist    vb_shuffle_create_str(VB_BYTES, VB_AGG_GROUP) for rank `rank` of `world`; String
 *                                     cogroup and the joins (vb_cogroup_n_str, vb_join_n_str) read such shuffles.
 * vb_shuffle_create_str_sort_bytes_dist  vb_shuffle_create_str_sort_bytes for rank `rank` of `world`.
 * 1 <= world <= 256 (VB_ERR_INVALID otherwise); world 1 is the one-process create.  Map with vb_shuffle_map_bytes /
 * vb_shuffle_map_str_bytes, map ids in contiguous blocks by rank as for every multi-rank shuffle; rank r owns the
 * partitions p with p % world == r.  The exchange, for GROUP and COGROUP, is the export / import pair below (any
 * all-to-all-v moves the columns) or vb_shuffle_exchange; the sorts cross ranks through vb_shuffle_exchange only.
 * vb_shuffle_exchange(VB_XCHG_AUTO or VB_XCHG_NCCL) runs the whole exchange with NCCL on the library's stream; it counts
 * rows in stats as integer rows do (String GROUP: values).  VB_XCHG_P2P, vb_shuffle_set_dist with world > 1, the plain,
 * _str and _cols export / import calls, vb_shuffle_export_counts / export_direct / import_arena and the blob calls return
 * VB_ERR_UNSUPPORTED.
 * Wire format: the kind's columns without the value references, plus two columns for the values:
 *   val_lens   u32 [values]   each value's length in bytes, split by the kind's value counts (integer rows: counts)
 *   val_bytes  u8  [bytes]    the values' bytes, concatenated in row order, split by n_val_bytes
 * integer GROUP / COGROUP  keys (i64) [rows] by counts, then val_lens and val_bytes; the gathered count row is counts[W]
 *                          and n_val_bytes[W].
 * String GROUP             key_lens, key_bytes and val_counts as for vb_shuffle_export_str_*, then val_lens (by n_vals)
 *                          and val_bytes; the gathered count row is n_keys, n_key_bytes, n_vals and n_val_bytes [W] each.
 * sorts                    per output partition as their numeric forms, val_lens and val_bytes in place of the payload,
 *                          with each partition's value bytes added to the gathered segment table.
 * Receive side: the received bytes become one more value store of the shuffle, and the received rows get fresh
 * references into it in receive order, so everything downstream (seal, cogroup, joins, gather) runs as on one process.
 * The map stores are freed once the export has packed them: a reference read before the exchange is refused by the
 * gather from then on (VB_ERR_INVALID).  Memory: during the exchange a rank holds its map stores, the packed copy of
 * its values and what it receives, about three times its share of value bytes; afterwards only what it received.
 *   vb_shuffle_export_bytes_prepare  finishes the local map side and packs it by destination rank; counts / n_val_bytes
 *                                    [world] get the rows and value bytes that go to each rank.
 *   vb_shuffle_export_bytes_buffers  the packed columns (library-owned device buffers, destination-major, valid until
 *                                    seal).
 *   vb_shuffle_import_bytes          the received columns, source-rank major, with what every source sent.  keys are
 *                                    borrowed until seal; val_lens and val_bytes are read (and the bytes copied) during
 *                                    the call.
 *   vb_shuffle_export_str_bytes_prepare / _buffers / vb_shuffle_import_str_bytes: the same for String GROUP; the key
 *                                    columns and val_counts are borrowed until seal.
 * Errors: the export / import calls on a bytes shuffle of world 1: VB_ERR_STATE (VB_ERR_INVALID on a shuffle the matching
 * create did not make, VB_ERR_UNSUPPORTED on a sort); import before export, twice, or after seal, map after export, and
 * seal without import: VB_ERR_STATE; a NULL column with a non-zero count: VB_ERR_INVALID; value lengths that do not add
 * up to the byte counts: VB_ERR_INVALID, the import keeps nothing and the shuffle can still be imported; a rank that
 * would receive 2^32 - 2 rows or more: VB_ERR_TOO_LARGE, decided from the counts so that, in vb_shuffle_exchange, every
 * rank returns it alike. */
VB_API int32_t vb_shuffle_create_bytes_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t key_dtype,
                                            int32_t agg, int32_t part, uint32_t rank, uint32_t world, vb_shuf **out);
VB_API int32_t vb_shuffle_create_str_bytes_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t rank,
                                                uint32_t world, vb_shuf **out);
VB_API int32_t vb_shuffle_create_str_sort_bytes_dist(vb_ctx *ctx, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t rank,
                                                     uint32_t world, vb_shuf **out);
VB_API int32_t vb_shuffle_export_bytes_prepare(vb_shuf *s, uint64_t *counts /*[world]*/, uint64_t *n_val_bytes /*[world]*/);
VB_API int32_t vb_shuffle_export_bytes_buffers(vb_shuf *s, void **keys, uint32_t **val_lens, void **val_bytes);
VB_API int32_t vb_shuffle_import_bytes(vb_shuf *s, const void *keys, const uint32_t *val_lens, const void *val_bytes,
                                       const uint64_t *counts /*[world]*/, const uint64_t *n_val_bytes /*[world]*/);
VB_API int32_t vb_shuffle_export_str_bytes_prepare(vb_shuf *s, uint64_t *n_keys /*[world]*/, uint64_t *n_key_bytes /*[world]*/,
                                                   uint64_t *n_vals /*[world]*/, uint64_t *n_val_bytes /*[world]*/);
VB_API int32_t vb_shuffle_export_str_bytes_buffers(vb_shuf *s, uint32_t **key_lens, void **key_bytes, uint32_t **val_counts,
                                                   uint32_t **val_lens, void **val_bytes);
VB_API int32_t vb_shuffle_import_str_bytes(vb_shuf *s, const uint32_t *key_lens, const void *key_bytes, const uint32_t *val_counts,
                                           const uint32_t *val_lens, const void *val_bytes, const uint64_t *n_keys /*[world]*/,
                                           const uint64_t *n_key_bytes /*[world]*/, const uint64_t *n_vals /*[world]*/,
                                           const uint64_t *n_val_bytes /*[world]*/);

/* MetroHash64_1(bytes ‖ 0xFF, seed 0): the reference's hash of a `String` / `&str` key */
VB_API uint64_t vb_hash_str(const void *bytes, uint64_t len);
VB_API uint32_t vb_get_partition_str(const void *bytes, uint64_t len, uint32_t n_reduce);
/* MetroHash64_1(le64(len) ‖ bytes, seed 0): the reference's hash of a `Vec<u8>` / `&[u8]` / `[u8; N]` key */
VB_API uint64_t vb_hash_bytes(const void *bytes, uint64_t len);
VB_API uint32_t vb_get_partition_bytes(const void *bytes, uint64_t len, uint32_t n_reduce);

/* ---- SURVEY §8(f) N1: bincode blobs — the payload format of SHUFFLE_CACHE ------------------------
 * The reference serialises every (map, reduce) bucket with bincode 1.2.1 defaults (src/dependency.rs:213-214:
 * little-endian, fixed-width integers, u64 length prefixes) and decodes it in the fetcher
 * (src/shuffle/shuffle_fetcher.rs:85).  These entry points speak that format so GPU results can be
 * served to, and CPU-produced buckets consumed from, unmodified vega executors:
 *   Vec<(u64,u64)>      = u64 n | n x (u64 k, u64 c)                       (reduce ops, sort)
 *   Vec<(u64,Vec<u64>)> = u64 n | n x (u64 k, u64 len, len x u64)          (group ops)
 *   Vec<(String,u64)>   = u64 n | n x (u64 len, len key bytes, u64 c)      (string-key SUM / MIN / MAX / COUNT)
 * vb_shuffle_reduce_blob encodes one sealed reduce partition; vb_shuffle_map_blob submits one
 * map-side-COMBINED bucket as the output of map task `map_id` (combiners are merged with
 * merge_combiners, so partial counts are summed).  A blob whose length field disagrees with its
 * size is rejected with VB_ERR_INVALID (the reference's DeserializationError).
 * String keys (vb_shuffle_create_str / _str_dist with a reduce op): records are unaligned, so a blob
 * is 8 + 16 n + key bytes long; c is the op's combiner (the value's bits, a u64 count for COUNT).
 * vb_shuffle_reduce_blob gives the rows of vb_shuffle_reduce_str in the same key order (a partition
 * this rank does not own: 8 zero bytes); its device destination must be 16-byte aligned
 * (VB_ERR_INVALID otherwise).  vb_shuffle_map_blob (world == 1 only, VB_ERR_UNSUPPORTED otherwise)
 * takes any src_loc; a map id may be submitted as rows or as a blob, the last submission wins.
 * Rejected before any allocation or device work: fewer than 8 bytes, more records than the bytes
 * can hold, a record whose key or value runs past the end, trailing bytes (VB_ERR_INVALID); a key
 * of 2^32 bytes or more (VB_ERR_TOO_LARGE).  Key bytes are not UTF-8-validated.  String GROUP,
 * sort and combine_by_key shuffles and byte-string values return VB_ERR_UNSUPPORTED.            */
VB_API int32_t vb_shuffle_reduce_blob_size(vb_shuf *s, uint32_t reduce_id, uint64_t *n_bytes);
VB_API int32_t vb_shuffle_reduce_blob(vb_shuf *s, uint32_t reduce_id, void *out_blob, int32_t dst_loc);
VB_API int32_t vb_shuffle_map_blob(vb_shuf *s, uint32_t map_id, const void *blob, uint64_t n_bytes, int32_t src_loc);

VB_API int32_t vb_shuffle_free(vb_shuf *s);
VB_API int32_t vb_shuffle_stats(vb_shuf *s, vb_stats *out);
VB_API const char *vb_last_error(void);

/* ---- host-side pieces of the path ------------------------------------------------------ */
/* MetroHash64_1 of the key's 4 or 8 LE bytes, seed 0 (src/partitioner.rs:21-25). */
VB_API uint64_t vb_hash_key(uint64_t key, uint32_t key_width);
/* HashPartitioner::get_partition (src/partitioner.rs:54-57). */
VB_API uint32_t vb_get_partition(uint64_t key, uint32_t key_width, uint32_t n_reduce);
/* ParallelCollection::slice: writes slice starts (and n as the last entry) into
 * starts[min(n,num_slices)+2] and returns the number of slices (n+1 when n < num_slices).  */
VB_API uint64_t vb_slice(uint64_t n, uint64_t num_slices, uint64_t *starts);

/* Context::range (src/context.rs:419-431): the u64 sequence (start..=end).step_by(step) as a device-resident
 * source — SURVEY §8(f) N3: no host array, no H2D.  vb_range_len = number of elements; out_dev holds that many. */
VB_API uint64_t vb_range_len(uint64_t start, uint64_t end, uint64_t step);
VB_API int32_t vb_range(vb_ctx *ctx, void *out_dev, uint64_t start, uint64_t end, uint64_t step);

/* ---- synthetic input, generated on the device (bench / parity tests) -------------------- */
/* Row i (i = first .. first+n-1):
 *   VB_GEN_UNIFORM  rank = splitmix64(seed_k+i) % n_distinct
 *   VB_GEN_ZIPF     rank = Zipf(zipf_s) over [0,n_distinct) by inverse CDF, u = splitmix64(seed_k+i)/2^64
 *   VB_GEN_UNIQUE   rank = rank_base + i   (each rank exactly once: join inputs)
 * key = splitmix64(rank ^ 0xA5A5A5A5A5A5A5A5) (a bijection: distinct ranks give distinct keys);
 * val = splitmix64(seed_v+i) & 0xFFFFF.  Writes AoS rows (rows_dev) if non-NULL, else SoA
 * keys_dev / vals_dev (vals_dev may be NULL).  Same stream as oracle/vega_oracle.c:vo_gen_uniform. */
enum vb_gen { VB_GEN_UNIFORM = 0, VB_GEN_ZIPF = 1, VB_GEN_UNIQUE = 2 };
VB_API int32_t vb_gen_pairs(vb_ctx *ctx, void *rows_dev, void *keys_dev, void *vals_dev, uint64_t first, uint64_t n,
                            int32_t mode, uint64_t n_distinct, uint64_t rank_base, uint64_t seed_k, uint64_t seed_v,
                            double zipf_s);

/* Device time and launch count per kernel class (profiling on): 0 hash_agg (map-side combine),
 * 1 dict build, 2 merge, 3 rp_hist, 4 rp_scan, 5 rp_scatter, 6 misc, 7 join, 8 str_order (the ordering of a
 * string sort's distinct keys, its radix passes included).                                     */
VB_API int32_t vb_shuffle_kernel_time(vb_shuf *s, int32_t klass, double *ms, uint64_t *launches);

/* library build info: "vega_b200 <version> sm_90a" */
VB_API const char *vb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* VEGA_B200_H */
