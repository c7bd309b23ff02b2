//! vega_b200_sys.rs — `extern "C"` declarations of libvega_b200.so for vega (Rust).
//!
//! SOURCE ONLY: this image has no rustc/cargo (and vega needs nightly-2020-05-31 + capnpc), so
//! this file has never been compiled.  It is the binding a vega maintainer would add as
//! `src/gpu/sys.rs`; see INTEGRATION.md for the four call-site patches that use it.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_void};

#[repr(C)] pub struct vb_ctx { _p: [u8; 0] }
#[repr(C)] pub struct vb_shuf { _p: [u8; 0] }
/// include/vega_b200.h `vb_agg_col`: aggregate `agg` (VB_AGG_SUM / MIN / MAX / COUNT / MEAN) over value column `src`
#[repr(C)] pub struct vb_agg_col { pub agg: i32, pub src: i32 }

pub const VB_OK: i32 = 0;
pub const VB_U64: i32 = 0; pub const VB_I64: i32 = 1; pub const VB_F64: i32 = 2; pub const VB_BYTES: i32 = 3;
pub const VB_STRKEY_STR: i32 = 0; pub const VB_STRKEY_BYTES: i32 = 1;   // vb_shuffle_set_str_key
pub const VB_VALORDER_INPUT: i32 = 0; pub const VB_VALORDER_ASC: i32 = 1;   // vb_shuffle_set_value_order
pub const VB_AGG_GROUP: i32 = 0; pub const VB_AGG_SUM: i32 = 1; pub const VB_AGG_MIN: i32 = 2;
pub const VB_AGG_MAX: i32 = 3; pub const VB_AGG_COUNT: i32 = 4; pub const VB_AGG_COGROUP: i32 = 5;
pub const VB_AGG_MEAN: i32 = 7;   // vb_agg_col only
pub const VB_PART_HASH_METRO64: i32 = 0;
pub const VB_HOST: i32 = 0;
/// include/vega_b200.h `vb_join_kind` (vb_join_outer; the inner join is vb_join)
pub const VB_JOIN_LEFT: i32 = 1; pub const VB_JOIN_RIGHT: i32 = 2; pub const VB_JOIN_FULL: i32 = 3;
pub const VB_MAX_COGROUP_SIDES: usize = 16;

#[link(name = "vega_b200")]
extern "C" {
    pub fn vb_ctx_create(device_id: i32, out: *mut *mut vb_ctx) -> i32;
    pub fn vb_ctx_destroy(ctx: *mut vb_ctx) -> i32;
    pub fn vb_shuffle_create(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, key_dtype: i32,
                             val_dtype: i32, agg: i32, part: i32, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_set_key_width(s: *mut vb_shuf, bytes: u32) -> i32;
    pub fn vb_shuffle_map_aos(s: *mut vb_shuf, map_id: u32, rows: *const c_void, n_rows: u64, src_loc: i32) -> i32;
    pub fn vb_shuffle_map_soa(s: *mut vb_shuf, map_id: u32, keys: *const c_void, vals: *const c_void,
                              n_rows: u64, src_loc: i32) -> i32;
    pub fn vb_shuffle_seal(s: *mut vb_shuf) -> i32;
    pub fn vb_shuffle_reduce_size(s: *mut vb_shuf, reduce_id: u32, n_keys: *mut u64, n_vals: *mut u64) -> i32;
    pub fn vb_shuffle_reduce(s: *mut vb_shuf, reduce_id: u32, out_keys: *mut c_void, out_combined: *mut c_void,
                             out_offsets: *mut u64, out_vals: *mut c_void, dst_loc: i32) -> i32;
    pub fn vb_join_size(left: *mut vb_shuf, right: *mut vb_shuf, reduce_id: u32, n_out: *mut u64) -> i32;
    pub fn vb_join(left: *mut vb_shuf, right: *mut vb_shuf, reduce_id: u32, out_k: *mut c_void, out_v: *mut c_void,
                   out_w: *mut c_void, dst_loc: i32) -> i32;
    // left / right / full outer joins: a None slot holds 0 and its validity byte (optional arrays) is 0
    pub fn vb_join_outer_size(left: *mut vb_shuf, right: *mut vb_shuf, reduce_id: u32, kind: i32, n_out: *mut u64) -> i32;
    pub fn vb_join_outer(left: *mut vb_shuf, right: *mut vb_shuf, reduce_id: u32, kind: i32, out_k: *mut c_void,
                         out_v: *mut c_void, out_w: *mut c_void, out_v_valid: *mut u8, out_w_valid: *mut u8,
                         dst_loc: i32) -> i32;
    // CoGroupedRdd::compute for PairRdd::cogroup: every key once, left and right value lists as two CSRs
    pub fn vb_cogroup_size(left: *mut vb_shuf, right: *mut vb_shuf, reduce_id: u32, n_keys: *mut u64,
                           n_left_vals: *mut u64, n_right_vals: *mut u64) -> i32;
    pub fn vb_cogroup(left: *mut vb_shuf, right: *mut vb_shuf, reduce_id: u32, out_keys: *mut c_void,
                      out_left_offsets: *mut u64, out_left_vals: *mut c_void, out_right_offsets: *mut u64,
                      out_right_vals: *mut c_void, dst_loc: i32) -> i32;
    // CoGroupedRdd::compute with n_sides parents (1 ..= VB_MAX_COGROUP_SIDES): one CSR value list per side, and the
    // inner join of all sides as (k, v_0, ..., v_{n-1}) rows
    pub fn vb_cogroup_n_size(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, n_keys: *mut u64,
                             n_vals: *mut u64) -> i32;
    pub fn vb_cogroup_n(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, out_keys: *mut c_void,
                        out_offsets: *const *mut u64, out_vals: *const *mut c_void, dst_loc: i32) -> i32;
    pub fn vb_join_n_size(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, n_out: *mut u64) -> i32;
    pub fn vb_join_n(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, out_k: *mut c_void,
                     out_vals: *const *mut c_void, dst_loc: i32) -> i32;
    // outer join of all sides: bit j of `required` marks side j required; a missing optional side is one None slot
    // (value 0, validity byte 0).  out_valid and its entries may be NULL
    pub fn vb_join_n_outer_size(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32,
                                n_out: *mut u64) -> i32;
    pub fn vb_join_n_outer(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32, out_k: *mut c_void,
                           out_vals: *const *mut c_void, out_valid: *const *mut u8, dst_loc: i32) -> i32;
    // semi / anti join of side 0 (subtractByKey, left semi join; vega has none): a side-0 key is kept when every side of
    // `required` has it and no side of `excluded` does (masks over sides 1..n-1), and gives its side-0 rows
    pub fn vb_semi_join_n_size(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32, excluded: u32,
                               n_rows: *mut u64) -> i32;
    pub fn vb_semi_join_n(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32, excluded: u32,
                          out_k: *mut c_void, out_v: *mut c_void, dst_loc: i32) -> i32;
    // N1: bincode blobs (the payload format of SHUFFLE_CACHE)
    pub fn vb_shuffle_reduce_blob_size(s: *mut vb_shuf, reduce_id: u32, n_bytes: *mut u64) -> i32;
    pub fn vb_shuffle_reduce_blob(s: *mut vb_shuf, reduce_id: u32, out_blob: *mut c_void, dst_loc: i32) -> i32;
    pub fn vb_shuffle_map_blob(s: *mut vb_shuf, map_id: u32, blob: *const c_void, n_bytes: u64, src_loc: i32) -> i32;
    // one process per GPU: pack + all-to-all-v, or the fused exchange over peer memory
    pub fn vb_shuffle_set_dist(s: *mut vb_shuf, rank: u32, world: u32) -> i32;
    pub fn vb_shuffle_export_prepare(s: *mut vb_shuf, counts: *mut u64) -> i32;
    pub fn vb_shuffle_export_buffers(s: *mut vb_shuf, keys_dev: *mut *mut c_void, vals_dev: *mut *mut c_void) -> i32;
    pub fn vb_shuffle_import(s: *mut vb_shuf, keys_dev: *const c_void, vals_dev: *const c_void, counts: *const u64) -> i32;
    pub fn vb_ctx_arena_reserve(ctx: *mut vb_ctx, bytes: u64, handle_out: *mut c_void, generation: *mut u64) -> i32;
    pub fn vb_ctx_peer_open(ctx: *mut vb_ctx, peer_rank: u32, handle: *const c_void, generation: u64, is_self: i32) -> i32;
    pub fn vb_shuffle_export_counts(s: *mut vb_shuf, counts: *mut u64) -> i32;
    pub fn vb_shuffle_export_direct(s: *mut vb_shuf, dst_row_offset: *const u64, dst_total_rows: *const u64) -> i32;
    pub fn vb_shuffle_import_arena(s: *mut vb_shuf, counts: *const u64) -> i32;
    // the exchange inside the library: NCCL communicator per context (unique id handed out by vega's tracker channel)
    pub fn vb_comm_unique_id(id_out: *mut c_void /* 128 bytes */) -> i32;
    pub fn vb_ctx_comm_init(ctx: *mut vb_ctx, unique_id: *const c_void, rank: u32, world: u32) -> i32;
    pub fn vb_ctx_comm_destroy(ctx: *mut vb_ctx) -> i32;
    pub fn vb_shuffle_exchange(s: *mut vb_shuf, mode: i32 /* VB_XCHG_AUTO = 0 */) -> i32;
    pub fn vb_ctx_arena_release_retired(ctx: *mut vb_ctx) -> i32;
    pub fn vb_ctx_trim(ctx: *mut vb_ctx, keep_bytes: u64) -> i32;
    // device-resident source (Context::range)
    pub fn vb_range_len(start: u64, end: u64, step: u64) -> u64;
    pub fn vb_range(ctx: *mut vb_ctx, out_dev: *mut c_void, start: u64, end: u64, step: u64) -> i32;
    // combine_by_key: several named aggregates per key in one shuffle (SoA columns)
    pub fn vb_shuffle_create_multi(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, key_dtype: i32, n_val_cols: u32,
                                   val_dtypes: *const i32, n_aggs: u32, aggs: *const vb_agg_col, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_map_cols(s: *mut vb_shuf, map_id: u32, keys: *const c_void, vals: *const *const c_void, n_rows: u64, src_loc: i32) -> i32;
    pub fn vb_shuffle_reduce_cols(s: *mut vb_shuf, reduce_id: u32, out_keys: *mut c_void, out_aggs: *const *mut c_void, dst_loc: i32) -> i32;
    // combine_by_key across ranks: export packs one row per distinct key by destination rank (u64 keys, u64 accumulator
    // columns [n_acc][rows] in plain value form), import takes them source-rank major (borrowed until seal)
    pub fn vb_shuffle_create_multi_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, key_dtype: i32, n_val_cols: u32,
                                        val_dtypes: *const i32, n_aggs: u32, aggs: *const vb_agg_col, rank: u32, world: u32,
                                        out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_export_cols_prepare(s: *mut vb_shuf, counts: *mut u64) -> i32;
    pub fn vb_shuffle_export_cols_buffers(s: *mut vb_shuf, keys: *mut *mut c_void, accs: *mut *mut c_void, n_acc: *mut u32) -> i32;
    pub fn vb_shuffle_import_cols(s: *mut vb_shuf, keys: *const c_void, accs: *const c_void, n_acc: u32, counts: *const u64) -> i32;
    // a sealed reduce-op / combine_by_key shuffle as a cogroup or join side under the same partitioner (OneToOneDependency)
    pub fn vb_shuffle_create_narrow(parent: *mut vb_shuf, out_col: u32, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_create_narrow_str(parent: *mut vb_shuf, out_col: u32, out: *mut *mut vb_shuf) -> i32;
    // String keys (Arrow-style offsets + bytes; placed by MetroHash64_1(bytes ‖ 0xFF) like `str::hash`)
    pub fn vb_shuffle_create_str(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, val_dtype: i32, agg: i32,
                                 out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_map_str(s: *mut vb_shuf, map_id: u32, key_offsets: *const u64, key_bytes: *const c_void, n_bytes: u64,
                              vals: *const c_void, n_rows: u64, src_loc: i32) -> i32;
    pub fn vb_shuffle_reduce_str_size(s: *mut vb_shuf, reduce_id: u32, n_keys: *mut u64, n_key_bytes: *mut u64,
                                      n_vals: *mut u64) -> i32;
    pub fn vb_shuffle_reduce_str(s: *mut vb_shuf, reduce_id: u32, out_key_offsets: *mut u64, out_key_bytes: *mut c_void,
                                 out_combined: *mut c_void, out_offsets: *mut u64, out_vals: *mut c_void, dst_loc: i32) -> i32;
    // CoGroupedRdd::compute over String GROUP shuffles: the cogroup, and the join with a `required` mask whose keys
    // come once per key (key i's rows are out_row_offsets[i] .. [i + 1])
    pub fn vb_cogroup_n_str_size(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, n_keys: *mut u64,
                                 n_key_bytes: *mut u64, n_vals: *mut u64) -> i32;
    pub fn vb_cogroup_n_str(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, out_key_offsets: *mut u64,
                            out_key_bytes: *mut c_void, out_offsets: *const *mut u64, out_vals: *const *mut c_void,
                            dst_loc: i32) -> i32;
    pub fn vb_join_n_str_size(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32, n_rows: *mut u64,
                              n_keys: *mut u64, n_key_bytes: *mut u64) -> i32;
    pub fn vb_join_n_str(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32, out_key_offsets: *mut u64,
                         out_key_bytes: *mut c_void, out_row_offsets: *mut u64, out_vals: *const *mut c_void,
                         out_valid: *const *mut u8, dst_loc: i32) -> i32;
    pub fn vb_semi_join_n_str_size(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32, excluded: u32,
                                   n_rows: *mut u64, n_keys: *mut u64, n_key_bytes: *mut u64) -> i32;
    pub fn vb_semi_join_n_str(sides: *const *mut vb_shuf, n_sides: u32, reduce_id: u32, required: u32, excluded: u32,
                              out_key_offsets: *mut u64, out_key_bytes: *mut c_void, out_row_offsets: *mut u64,
                              out_vals: *mut c_void, dst_loc: i32) -> i32;
    // String keys across ranks: export packs by destination rank as four columns (u32 key lengths, key bytes, u32 value
    // counts for GROUP, u64 values), import takes them source-rank major (borrowed until seal)
    pub fn vb_shuffle_create_str_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, val_dtype: i32, agg: i32,
                                      rank: u32, world: u32, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_export_str_prepare(s: *mut vb_shuf, n_keys: *mut u64, n_key_bytes: *mut u64, n_vals: *mut u64) -> i32;
    pub fn vb_shuffle_export_str_buffers(s: *mut vb_shuf, key_lens: *mut *mut u32, key_bytes: *mut *mut c_void,
                                         val_counts: *mut *mut u32, vals: *mut *mut u64) -> i32;
    pub fn vb_shuffle_import_str(s: *mut vb_shuf, key_lens: *const u32, key_bytes: *const c_void, val_counts: *const u32,
                                 vals: *const u64, n_keys: *const u64, n_key_bytes: *const u64, n_vals: *const u64) -> i32;
    // combine_by_key over String keys: the combine spec of vb_shuffle_create_multi, keys as for vb_shuffle_map_str; across
    // ranks the wire is u32 key lengths, key bytes and u64 accumulators [n_acc][keys] in plain value form
    pub fn vb_shuffle_create_str_multi(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, n_val_cols: u32,
                                       val_dtypes: *const i32, n_aggs: u32, aggs: *const vb_agg_col, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_create_str_multi_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, n_val_cols: u32,
                                            val_dtypes: *const i32, n_aggs: u32, aggs: *const vb_agg_col, rank: u32, world: u32,
                                            out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_map_str_cols(s: *mut vb_shuf, map_id: u32, key_offsets: *const u64, key_bytes: *const c_void, n_bytes: u64,
                                   vals: *const *const c_void, n_rows: u64, src_loc: i32) -> i32;
    pub fn vb_shuffle_reduce_str_cols(s: *mut vb_shuf, reduce_id: u32, out_key_offsets: *mut u64, out_key_bytes: *mut c_void,
                                      out_aggs: *const *mut c_void, dst_loc: i32) -> i32;
    pub fn vb_shuffle_export_str_cols_prepare(s: *mut vb_shuf, n_keys: *mut u64, n_key_bytes: *mut u64) -> i32;
    pub fn vb_shuffle_export_str_cols_buffers(s: *mut vb_shuf, key_lens: *mut *mut u32, key_bytes: *mut *mut c_void,
                                              accs: *mut *mut u64, n_acc: *mut u32) -> i32;
    pub fn vb_shuffle_import_str_cols(s: *mut vb_shuf, key_lens: *const u32, key_bytes: *const c_void, accs: *const u64, n_acc: u32,
                                      n_keys: *const u64, n_key_bytes: *const u64) -> i32;
    // byte-string values (VB_BYTES = 3): a String as its UTF-8 bytes, any V: Serialize as its bincode bytes, for
    // group / cogroup / join / sort; the output calls return opaque references, gathered back into bytes here
    pub fn vb_shuffle_map_bytes(s: *mut vb_shuf, map_id: u32, keys: *const c_void, val_offsets: *const u64, val_bytes: *const c_void,
                                n_val_bytes: u64, n_rows: u64, src_loc: i32) -> i32;
    pub fn vb_shuffle_map_str_bytes(s: *mut vb_shuf, map_id: u32, key_offsets: *const u64, key_bytes: *const c_void, n_key_bytes: u64,
                                    val_offsets: *const u64, val_bytes: *const c_void, n_val_bytes: u64, n_rows: u64,
                                    src_loc: i32) -> i32;
    pub fn vb_shuffle_create_str_sort_bytes(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32,
                                            out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_gather_bytes_size(s: *mut vb_shuf, refs: *const u64, n: u64, src_loc: i32, n_bytes: *mut u64) -> i32;
    pub fn vb_shuffle_gather_bytes(s: *mut vb_shuf, refs: *const u64, n: u64, src_loc: i32, out_offsets: *mut u64,
                                   out_bytes: *mut c_void, dst_loc: i32) -> i32;
    // repartition(n) = coalesce(n, shuffle = true): items of 0-2 u64 columns plus optional bytes, placed by position
    pub fn vb_shuffle_create_repartition(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, n_cols: u32, has_bytes: i32,
                                         out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_create_repartition_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, n_cols: u32, has_bytes: i32,
                                              rank: u32, world: u32, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_map_repartition(s: *mut vb_shuf, map_id: u32, first_position: u64, cols: *const *const c_void,
                                      val_offsets: *const u64, val_bytes: *const c_void, n_val_bytes: u64, n_rows: u64,
                                      src_loc: i32) -> i32;
    pub fn vb_shuffle_reduce_repartition_size(s: *mut vb_shuf, r: u32, n_rows: *mut u64, n_bytes: *mut u64) -> i32;
    pub fn vb_shuffle_reduce_repartition(s: *mut vb_shuf, r: u32, out_cols: *const *mut c_void, out_offsets: *mut u64,
                                         out_bytes: *mut c_void, dst_loc: i32) -> i32;
    // byte-string values across ranks: the rows' bytes travel as u32 lengths + bytes, never their references
    pub fn vb_shuffle_create_bytes_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, key_dtype: i32, agg: i32,
                                        part: i32, rank: u32, world: u32, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_create_str_bytes_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, rank: u32, world: u32,
                                            out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_create_str_sort_bytes_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, rank: u32,
                                                 world: u32, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_shuffle_export_bytes_prepare(s: *mut vb_shuf, counts: *mut u64, n_val_bytes: *mut u64) -> i32;
    pub fn vb_shuffle_export_bytes_buffers(s: *mut vb_shuf, keys: *mut *mut c_void, val_lens: *mut *mut u32,
                                           val_bytes: *mut *mut c_void) -> i32;
    pub fn vb_shuffle_import_bytes(s: *mut vb_shuf, keys: *const c_void, val_lens: *const u32, val_bytes: *const c_void,
                                   counts: *const u64, n_val_bytes: *const u64) -> i32;
    pub fn vb_shuffle_export_str_bytes_prepare(s: *mut vb_shuf, n_keys: *mut u64, n_key_bytes: *mut u64, n_vals: *mut u64,
                                               n_val_bytes: *mut u64) -> i32;
    pub fn vb_shuffle_export_str_bytes_buffers(s: *mut vb_shuf, key_lens: *mut *mut u32, key_bytes: *mut *mut c_void,
                                               val_counts: *mut *mut u32, val_lens: *mut *mut u32, val_bytes: *mut *mut c_void) -> i32;
    pub fn vb_shuffle_import_str_bytes(s: *mut vb_shuf, key_lens: *const u32, key_bytes: *const c_void, val_counts: *const u32,
                                       val_lens: *const u32, val_bytes: *const c_void, n_keys: *const u64, n_key_bytes: *const u64,
                                       n_vals: *const u64, n_val_bytes: *const u64) -> i32;
    // sort_by_key over String keys (one process): map with vb_shuffle_map_str, read with vb_shuffle_reduce_str (rows in
    // key order, each with its key; the payload in out_combined); val_dtype -1 is key-only
    pub fn vb_shuffle_create_str_sort(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, val_dtype: i32,
                                      out: *mut *mut vb_shuf) -> i32;
    // the same for rank `rank` of `world`: rows cross ranks through vb_shuffle_exchange (vb_ctx_comm_init), and rank r
    // holds output partitions p with p % world == r
    pub fn vb_shuffle_create_str_sort_dist(ctx: *mut vb_ctx, shuffle_id: u64, n_map: u32, n_reduce: u32, val_dtype: i32,
                                           rank: u32, world: u32, out: *mut *mut vb_shuf) -> i32;
    pub fn vb_hash_str(bytes: *const c_void, len: u64) -> u64;
    pub fn vb_get_partition_str(bytes: *const c_void, len: u64, n_reduce: u32) -> u32;
    // Vec<u8> / &[u8] / [u8; N] keys: MetroHash64_1(le64(len) ‖ bytes), and the kind of a string-key shuffle
    pub fn vb_hash_bytes(bytes: *const c_void, len: u64) -> u64;
    pub fn vb_get_partition_bytes(bytes: *const c_void, len: u64, n_reduce: u32) -> u32;
    pub fn vb_shuffle_set_str_key(s: *mut vb_shuf, kind: i32) -> i32;
    // each key's list of a GROUP / COGROUP shuffle in map order, or ascending (sorted on the device); before the first map call
    pub fn vb_shuffle_set_value_order(s: *mut vb_shuf, order: i32) -> i32;
    pub fn vb_shuffle_free(s: *mut vb_shuf) -> i32;
    pub fn vb_last_error() -> *const c_char;
    pub fn vb_get_partition(key: u64, key_width: u32, n_reduce: u32) -> u32;
}
