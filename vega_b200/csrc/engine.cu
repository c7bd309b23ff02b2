// engine.cu — C ABI of libvega_b200.so (see include/vega_b200.h) and the host orchestration of
// the shuffle + aggregation kernels in kernels.cuh.  sm_90a only; no CPU fallback: every
// compute entry needs a CUDA device and fails with VB_ERR_CUDA otherwise.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <chrono>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/vega_b200.h"
#include "kernels.cuh"
#include "sweep.cuh"
#include "gsweep.cuh"
#include "strkeys.cuh"
#include "bytevals.cuh"
#include "segsort.cuh"
#include "semijoin.cuh"
#include <type_traits>

using namespace vb;

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static int set_err(int code, const char *fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CU(expr)                                                                                        \
    do {                                                                                                \
        cudaError_t e_ = (expr);                                                                        \
        if (e_ != cudaSuccess) {                                                                        \
            cudaGetLastError();                                                                         \
            return set_err(e_ == cudaErrorMemoryAllocation ? VB_ERR_OOM : VB_ERR_CUDA, "%s:%d %s: %s", \
                           __FILE__, __LINE__, #expr, cudaGetErrorString(e_));                          \
        }                                                                                               \
    } while (0)

#define TRY(expr)                  \
    do {                           \
        int rc_ = (expr);          \
        if (rc_ != VB_OK) return rc_; \
    } while (0)

extern "C" const char *vb_last_error(void) { return g_err.c_str(); }
extern "C" const char *vb_version(void) { return "vega_b200 0.1 sm_90a"; }

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
enum { K_HASH_AGG = 0, K_DICT = 1, K_MERGE = 2, K_RP_HIST = 3, K_RP_SCAN = 4, K_RP_SCATTER = 5, K_MISC = 6, K_JOIN = 7, K_STR_ORDER = 8, K_N = 9 };

struct vb_ctx {
    int device = 0;
    int sm_count = 132;
    u64 l2_bytes = 50ull << 20;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;          // H2D staging copies (overlap the kernels on `stream`)
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_kernel[2] = {nullptr, nullptr}, ev_ready = nullptr;
    std::vector<void *> pinned_slots;            // 64-byte pinned cells for per-call D2H status words (free list)
    cudaMemPool_t pool = nullptr;
    std::mutex mu;                 // serialises device work of this context
    bool profile = false;
    void *h_scratch = nullptr;     // pinned, 1 MiB
    size_t h_scratch_bytes = 1 << 20;
    double *zipf_cdf = nullptr;    // cached device CDF for vb_gen_pairs
    u64 zipf_n = 0;
    double zipf_s = 0;
    std::map<const void *, int> occ_cache;
    // P2P exchange: this rank's receive arena (cudaMalloc'ed, exported with CUDA IPC) and the peers' arenas
    void *arena = nullptr;
    size_t arena_bytes = 0;
    u64 arena_gen = 0;
    struct Peer { void *base = nullptr; u64 gen = 0; bool self = false; };
    std::map<u32, Peer> peers;
    std::vector<void *> retired_arenas;   // outgrown arenas some peer may still have mapped: freed by vb_ctx_arena_release_retired
    struct Comm *comm = nullptr;          // NCCL communicator + exchange scratch (vb_ctx_comm_init)
};
static void comm_teardown(vb_ctx *c);

struct DevBuf {   // stream-ordered device allocation, freed on scope exit unless released
    vb_ctx *c = nullptr;
    void *p = nullptr;
    DevBuf() {}
    explicit DevBuf(vb_ctx *c_) : c(c_) {}
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { reset(); }
    void reset()
    {
        if (p) cudaFreeAsync(p, c->stream);
        p = nullptr;
    }
    int alloc(size_t bytes)
    {
        reset();
        if (bytes == 0) bytes = 16;
        CU(cudaMallocAsync(&p, bytes, c->pool, c->stream));
        return VB_OK;
    }
    template <typename T> T *as() const { return (T *)p; }
    void *release()
    {
        void *q = p;
        p = nullptr;
        return q;
    }
};

static void dev_free(vb_ctx *c, const void *p)
{
    if (p) cudaFreeAsync((void *)p, c->stream);
}

template <typename K>
static int occupancy(vb_ctx *c, K kernel, int threads, size_t smem)
{
    auto it = c->occ_cache.find((const void *)kernel);
    if (it != c->occ_cache.end()) return it->second;
    int nb = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, threads, smem) != cudaSuccess || nb < 1) {
        cudaGetLastError();
        nb = 1;
    }
    c->occ_cache[(const void *)kernel] = nb;
    return nb;
}

extern "C" int32_t vb_ctx_create(int32_t device_id, vb_ctx **out)
{
    if (!out) return set_err(VB_ERR_INVALID, "vb_ctx_create: out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return set_err(VB_ERR_CUDA, "vb_ctx_create: no CUDA device (%s); libvega_b200 has no CPU fallback",
                       e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    }
    if (device_id < 0 || device_id >= ndev) return set_err(VB_ERR_INVALID, "vb_ctx_create: device %d of %d", device_id, ndev);
    CU(cudaSetDevice(device_id));
    vb_ctx *c = new vb_ctx();
    c->device = device_id;
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device_id));
    c->sm_count = prop.multiProcessorCount;
    c->l2_bytes = (u64)prop.l2CacheSize;
    CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    // a private stream-ordered pool: the process-wide default pool (shared with any other cudaMallocAsync
    // user) is left untouched; ours keeps its memory between shuffles (steady-state steps never call
    // cudaMalloc) until vb_ctx_trim / vb_ctx_destroy
    cudaMemPoolProps pp;
    memset(&pp, 0, sizeof(pp));
    pp.allocType = cudaMemAllocationTypePinned;
    pp.handleTypes = cudaMemHandleTypeNone;
    pp.location.type = cudaMemLocationTypeDevice;
    pp.location.id = device_id;
    CU(cudaMemPoolCreate(&c->pool, &pp));
    uint64_t thr = ~0ull;
    CU(cudaMemPoolSetAttribute(c->pool, cudaMemPoolAttrReleaseThreshold, &thr));
    CU(cudaMallocHost(&c->h_scratch, c->h_scratch_bytes));
    CU(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        CU(cudaEventCreateWithFlags(&c->ev_copied[i], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&c->ev_kernel[i], cudaEventDisableTiming));
    }
    CU(cudaEventCreateWithFlags(&c->ev_ready, cudaEventDisableTiming));
    {   // the last 4 KiB of the pinned scratch page hold 64 status cells
        char *base = (char *)c->h_scratch + c->h_scratch_bytes - 4096;
        for (int i = 0; i < 64; ++i) c->pinned_slots.push_back(base + 64 * i);
    }
    *out = c;
    return VB_OK;
}

extern "C" int32_t vb_ctx_destroy(vb_ctx *c)
{
    if (!c) return VB_OK;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (c->zipf_cdf) cudaFreeAsync(c->zipf_cdf, c->stream);
    cudaStreamSynchronize(c->stream);
    for (auto &kv : c->peers) if (kv.second.base && !kv.second.self) cudaIpcCloseMemHandle(kv.second.base);
    // An exported arena must outlive every importer's mapping (cudaFree of a region a peer still has open is
    // undefined): with a communicator, all ranks close their mappings above, meet at a barrier, then free.
    comm_teardown(c);
    for (void *p : c->retired_arenas) cudaFree(p);
    if (c->arena) cudaFree(c->arena);
    cudaFreeHost(c->h_scratch);
    cudaStreamSynchronize(c->copy_stream);
    cudaStreamDestroy(c->copy_stream);
    for (int i = 0; i < 2; ++i) { cudaEventDestroy(c->ev_copied[i]); cudaEventDestroy(c->ev_kernel[i]); }
    cudaEventDestroy(c->ev_ready);
    cudaStreamDestroy(c->stream);
    if (c->pool) cudaMemPoolDestroy(c->pool);
    delete c;
    return VB_OK;
}

extern "C" int32_t vb_ctx_trim(vb_ctx *c, uint64_t keep_bytes)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemPoolTrimTo(c->pool, (size_t)keep_bytes));
    return VB_OK;
}

extern "C" int32_t vb_ctx_synchronize(vb_ctx *c)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_ctx_set_profile(vb_ctx *c, int32_t on)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    c->profile = on != 0;
    return VB_OK;
}

extern "C" int32_t vb_ctx_device(vb_ctx *c) { return c ? c->device : -1; }
extern "C" void *vb_ctx_stream(vb_ctx *c) { return c ? (void *)c->stream : nullptr; }

extern "C" int32_t vb_ctx_mem_info(vb_ctx *c, uint64_t *reserved, uint64_t *high_water)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    uint64_t r = 0, h = 0;
    CU(cudaMemPoolGetAttribute(c->pool, cudaMemPoolAttrReservedMemCurrent, &r));
    CU(cudaMemPoolGetAttribute(c->pool, cudaMemPoolAttrUsedMemHigh, &h));
    if (reserved) *reserved = r;
    if (high_water) *high_water = h;
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// shuffle state
// ---------------------------------------------------------------------------------------------
struct MapOut {
    bool present = false;
    u64 n_rows = 0;
    // reduce ops: the combined table of this map task (== SHUFFLE_CACHE[(sid, map, *)])
    void *table = nullptr;      // table_at(table, log_cap)
    u32 log_cap = 0;
    u64 n_inserted = 0;
    // group/sort ops: the rows (device), AoS or SoA
    const u64 *rows = nullptr;
    const u64 *keys = nullptr;
    const u64 *vals = nullptr;
    const u64 *cols[MA_MAX_COLS] = {};   // multi-aggregate shuffles: borrowed value columns (shared-table rebuilds)
    bool owned = false;
    bool vals_owned = false;  // byte-string values: the reference column is the shuffle's even when the keys are borrowed
    bool in_shared = false;   // reduce ops, borrowed device input: combined straight into the shuffle's shared table
};

struct Timer {
    cudaEvent_t a, b;
    int klass;   // K_* or -1 (map call) / -2 (seal call)
    u64 rows;
};

// vb_join_outer_size's result for one (right side's uid, partition, outer kind), kept for vb_join_outer
struct JoinPlan {
    u64 total = 0;
    u32 nl = 0;
    u64 *pos = nullptr;            // [nl + nr] exclusive: the left keys' rows first, then the right-only keys' rows
    u32 *match = nullptr;
    u32 nr = 0;                    // RIGHT / FULL: right keys of the partition
    u64 total_left = 0;            // rows of the left keys (pos[nl])
};

// vb_cogroup_n_size / vb_join_n_size / vb_join_n_outer_size's result for one (sides, partition, kind), kept for the
// write call.  Cogroup output keys: side 0's keys in its CSR order, then each later side's new keys (those no earlier
// side has) in that side's CSR order.  A join whose side 0 is required (every inner join) reads side 0's keys only.
struct CogroupNPlan {
    u64 n_keys = 0;                // output keys: every key, or side 0's keys of the partition
    u64 *new_keys = nullptr;       // [n_keys - side 0's keys] the keys after side 0's
    u32 *match = nullptr;          // [n_keys][n_sides] the key's index on every side, 0xFFFFFFFF where a side lacks it
    u64 *pos = nullptr;            // join: [n_keys] each key's first output row
    u64 total = 0;                 // join: rows of the partition
    // string sides (str_plan_keys): the keys the call writes (a join's: those with rows) as Arrow-style offsets
    bool str_done = false;
    u64 str_nk = 0, str_nkb = 0;   // keys written, and their bytes
    u64 *str_sel = nullptr;        // join: [str_nk] the plan keys with rows
    u64 *str_koff = nullptr;       // [str_nk + 1] key byte offsets from 0
    u64 *str_roff = nullptr;       // join: [str_nk + 1] each key's first row, then the total
};
// n_plans kinds: the cogroup, the inner join, (>= 0) an outer join by its mask of required sides, or (<= NP_SEMI) a
// semi join by its two masks (semi_kind)
constexpr i64 NP_COGROUP = -2, NP_INNER = -1, NP_SEMI = -3;

// vb_semi_join_n's filter for one (sides, required, excluded), built by the first call and kept on side 0 until
// vb_shuffle_free: the presence dictionary of the filter sides' keys, or, when side 0 was lazy, its kept rows grouped
struct SemiFilter {
    void *tab = nullptr;           // presence dictionary (NULL: the filter sides have no keys)
    u32 log_cap = 0;
    u32 *mask = nullptr;           // [slots] bit j: side j has the slot's key
    struct vb_shuf *kept = nullptr;   // side 0 lazy: an internal GROUP-like shuffle of its kept rows (tab, mask freed)
};

struct vb_shuf {
    vb_ctx *ctx = nullptr;
    u64 id = 0;
    u32 n_map = 0, n_reduce = 0;
    int kdt = 0, vdt = 0, agg = 0, part = 0;
    // multi-aggregate shuffle (vb_shuffle_create_multi, _str_multi): agg is VB_AGG_SUM for the reduce-op plumbing, the
    // accumulators are described by the specs below and the results live in res_cols.  A string-key reduce op has
    // the specs and res_cols too (one value column, one aggregate), with multi false: multi selects the _multi calls.
    bool multi = false;
    u32 n_cols = 0;
    AccSpec acc_map{}, acc_merge{};   // map-side combine / table merge (COUNT merges as ADD, no order transform)
    AccSpec acc_imp{};                // merge of partials received from other ranks: merge ops, the map spec's transforms
    OutSpec outs{};                   // one output column per vb_agg_col
    int out_dt[VB_MAX_AGGS] = {};     // each output column's dtype (a narrow view's value dtype)
    u64 *res_cols = nullptr;          // [outs.n][n_keys], partition-major like res_keys
    u32 key_width = 8;
    u64 hint = 0;
    u64 learned_distinct = 0;      // distinct keys seen by the previous table build of this shuffle
    // Shared table of the map tasks whose input is VB_DEVICE_BORROWED (valid until seal): the named ops are
    // associative and commutative, so those tasks combine into ONE table, launched back to back without a
    // host round trip per task and without a merge at seal.  If it overflows, or a map id is resubmitted,
    // seal rebuilds it from the still-borrowed inputs (same restart logic as build_table).
    void *sh_tab = nullptr;
    u32 sh_log_cap = 0;
    TableCtl *sh_ctl = nullptr;
    u64 sh_max_inserts = 0;
    bool sh_dirty = false;
    u32 rank = 0, world = 1;
    std::vector<MapOut> maps;
    std::mutex mu;
    std::condition_variable cv;
    bool sealed = false, failed = false, freed = false;
    bool sealing = false;          // a vb_shuffle_seal is running: a second caller waits for it instead of re-running
    u32 waiters = 0;               // threads blocked in wait_sealed: vb_shuffle_free drains them before deleting
    // export / import (world > 1)
    bool exported = false, imported = false;
    u64 *exp_keys = nullptr, *exp_vals = nullptr;     // multi-aggregate shuffles: exp_vals = the accumulators [n_acc][rows]
    // fused export (P2P): plan + scanned histogram + gathered input kept between export_counts and export_direct
    u32 *exp_hist = nullptr;
    u32 exp_parts = 0;
    u64 exp_rows_per_part = 0, exp_n = 0;
    const u64 *exp_rows = nullptr, *exp_k = nullptr, *exp_v = nullptr;
    std::vector<u64> exp_digit_start;
    bool exp_counted = false;
    const u64 *imp_keys = nullptr, *imp_vals = nullptr;   // multi-aggregate shuffles: imp_vals = the partials [n_acc][imp_n]
    u64 imp_n = 0;
    u64 *imp_own_k = nullptr, *imp_own_v = nullptr;   // receive buffers of vb_shuffle_exchange (freed with the inputs)
    std::vector<u64> sort_part_rows;                  // multi-rank sort: exact rows of every output partition this rank owns (0 elsewhere)
    vb_xstats xst{};
    // gathered input kept alive for the reduce side of group ops
    u64 *gath_keys = nullptr, *gath_vals = nullptr;
    // results
    u64 n_keys = 0, n_vals = 0;
    u64 *res_keys = nullptr, *res_comb = nullptr, *res_offs = nullptr, *res_vals = nullptr;
    std::vector<u64> bucket_off;   // n_reduce + 1 (key index)
    std::vector<u64> val_off;      // n_reduce + 1 (value index; group ops)
    void *dict = nullptr;          // group ops: key → slot table, kept for joins
    u32 dict_log_cap = 0;
    u32 *dense_of_slot = nullptr;
    std::map<std::tuple<u64, u32, int>, JoinPlan> join_plans;   // by (right side's uid, partition, outer kind)
    // on side 0 of a cogroup or a join, of two sides or N: by (every side's uid, partition, NP_* kind or outer mask)
    std::map<std::tuple<std::vector<u64>, u32, i64>, CogroupNPlan> n_plans;
    // on side 0 of a semi join: by (every side's uid, required, excluded)
    std::map<std::tuple<std::vector<u64>, u32, u32>, SemiFilter> semi;
    // COGROUP shuffles are grouped lazily: seal keeps the (owned) rows; the CSR is built by the first reduce call
    // (cogroup materialisation), or — if a join comes first — only for the rows the join kind needs: the keys on BOTH
    // sides (inner), every row of the preserved side plus the matching rows of the other (LEFT / RIGHT), or all (FULL).
    u64 uid = 0;                                   // process-unique id (cache key that survives pointer reuse)
    int vorder = VB_VALORDER_INPUT;                // vb_shuffle_set_value_order: each list of a GROUP CSR in map order or ascending
    bool internal = false;                         // made by make_internal_like: a narrow view or a filtered join's side
    bool lazy = false;                             // sealed, rows in lz_*, not grouped yet
    u64 *lz_keys = nullptr, *lz_vals = nullptr;
    u64 lz_n = 0;
    std::vector<vb_shuf *> trash;                  // internal shuffles of a failed filtered join
    struct StrState *str = nullptr;                // string-key shuffle (vb_shuffle_create_str): dictionary, rows, results
    struct RepState *rep = nullptr;                // repartition shuffle (vb_shuffle_create_repartition): items and results
    // byte-string values (val dtype VB_BYTES): per map id the store of its values, kept until vb_shuffle_free; the
    // device copy of the table is made by the first gather.  Internal shuffles of a filtered join have no store.
    std::vector<ByteSrc> bvals;
    ByteSrc *bvals_dev = nullptr;
    // ... across ranks (vb_shuffle_create_*bytes_dist): the packed values of the export (u32 lengths and the bytes, in
    // the exported rows' order), owned until seal; what a rank receives is one more store, bvals[n_map]
    bool bdist = false;
    u32 *bx_lens = nullptr;
    unsigned char *bx_bytes = nullptr;
    // by (the right side's uid, join kind): internal (left, right) shuffles over the rows that join kind keeps
    std::map<std::pair<u64, int>, std::pair<vb_shuf *, vb_shuf *>> filtered;
    // stats
    vb_stats st{};
    std::vector<Timer> timers;
    int kclass_as = -1;            // >= 0: every kernel launched meanwhile is counted in this class (a string sort's ordering)
    double kms[K_N] = {0};
    u64 klaunch[K_N] = {0};
};

static int seal_str(vb_shuf *s);
static int seal_str_import(vb_shuf *s);
static int export_str_locked(vb_shuf *s, u64 *n_keys, u64 *n_key_bytes, u64 *n_vals, u64 *n_val_bytes = nullptr);
static int bytes_pack(vb_shuf *s, const u64 *refs, u64 n, const std::vector<u64> &cut, std::vector<u64> &at);
static int bytes_adopt(vb_shuf *s, const u32 *lens, u64 n, DevBuf &bytes, u64 n_bytes, DevBuf &refs);
static int str_import_limits(const vb_shuf *s, u64 nk, u64 nv);
static int exchange_str_locked(vb_shuf *s);
static int exchange_str_accs_locked(vb_shuf *s);
static int exchange_str_sort_locked(vb_shuf *s);
static void free_str(vb_shuf *s);
static void free_rep(vb_shuf *s);
static int seal_rep(vb_shuf *s);
static int exchange_rep(vb_shuf *s, int mode);
static int reject_rep(const vb_shuf *s, const char *what);

static bool is_reduce_op(int agg) { return agg == VB_AGG_SUM || agg == VB_AGG_MIN || agg == VB_AGG_MAX || agg == VB_AGG_COUNT; }
static bool is_group_op(int agg) { return agg == VB_AGG_GROUP || agg == VB_AGG_COGROUP; }

static int val_tx(const vb_shuf *s)
{
    if (s->agg != VB_AGG_MIN && s->agg != VB_AGG_MAX) return TX_NONE;
    return s->vdt == VB_I64 ? TX_I64 : s->vdt == VB_F64 ? TX_F64 : TX_NONE;
}
static int map_opk(const vb_shuf *s)
{
    switch (s->agg) {
    case VB_AGG_SUM: return s->vdt == VB_F64 ? OPK_ADD_F64 : OPK_ADD_U64;
    case VB_AGG_MIN: return OPK_MIN_U64;
    case VB_AGG_MAX: return OPK_MAX_U64;
    case VB_AGG_COUNT: return OPK_COUNT;
    default: return OPK_DICT;
    }
}
static int merge_opk(const vb_shuf *s) { return s->agg == VB_AGG_COUNT ? OPK_ADD_U64 : map_opk(s); }

// kernel launch bookkeeping (+ CUDA-event timing on the launching stream when profiling)
struct KLaunch {
    vb_shuf *s;
    int klass;
    u64 rows;
    cudaEvent_t a = nullptr, b = nullptr;
    bool pushed = false;
    ~KLaunch()
    {
        if (a && !pushed) { cudaEventDestroy(a); cudaEventDestroy(b); }
    }
    KLaunch(vb_shuf *s_, int klass_, u64 rows_ = 0) : s(s_), klass(s_ && s_->kclass_as >= 0 && klass_ >= 0 ? s_->kclass_as : klass_), rows(rows_)
    {
        if (s && s->ctx->profile) {
            cudaEventCreate(&a);
            cudaEventCreate(&b);
            cudaEventRecord(a, s->ctx->stream);
        }
    }
    int done(const char *what)
    {
        cudaError_t e = cudaGetLastError();
        if (a) {
            cudaEventRecord(b, s->ctx->stream);
            s->timers.push_back(Timer{a, b, klass, rows});
            pushed = true;
        }
        if (s && klass >= 0) {
            s->klaunch[klass]++;
            s->st.kernel_launches++;
        }
        if (e != cudaSuccess) return set_err(VB_ERR_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
        return VB_OK;
    }
};

static void resolve_timers(vb_shuf *s)
{
    if (s->timers.empty()) return;
    cudaStreamSynchronize(s->ctx->stream);
    for (auto &t : s->timers) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) {
            if (t.klass >= 0) s->kms[t.klass] += ms;
            else if (t.klass == -1) s->st.map_ms += ms;
            else if (t.klass == -3) s->xst.exchange_ms += ms;
            else s->st.seal_ms += ms;
            int hot = is_reduce_op(s->agg) ? K_HASH_AGG : K_RP_SCATTER;
            if (t.klass == hot) {
                s->st.hot_kernel_ms += ms;
                s->st.hot_kernel_launches++;
                s->st.hot_kernel_rows += t.rows;
            }
        } else cudaGetLastError();
        cudaEventDestroy(t.a);
        cudaEventDestroy(t.b);
    }
    s->timers.clear();
}

static u32 ceil_log2_u64(u64 x)
{
    u32 l = 0;
    while ((1ull << l) < x && l < 63) ++l;
    return l;
}

// ---------------------------------------------------------------------------------------------
// hash table build (map-side combine / reduce-side merge / dictionary)
// ---------------------------------------------------------------------------------------------
struct AggInput {
    int in;          // IN_AOS / IN_SOA / IN_TABLE
    const u64 *a;
    const u64 *b;
    u64 n;           // rows (IN_TABLE: slots incl. the special one)
    int loc;         // VB_HOST or device
    u64 items = 0;   // IN_TABLE: upper bound on the occupied slots (n_inserted + 1); 0 = n
    const u64 *cols[MA_MAX_COLS] = {};   // multi-aggregate IN_SOA: value columns (b unused); IN_TABLE: b = first accumulator column
};

template <int IN, int OPK, int TX>
static int launch_hash_agg_t(vb_shuf *s, int klass, const u64 *a, const u64 *b, u64 n, void *tab, u32 log_cap,
                             TableCtl *ctl, u64 max_inserts, u32 *slot_out)
{
    vb_ctx *c = s->ctx;
    Table t = table_at(tab, log_cap);
    t.keep_l2 = table_bytes(log_cap) <= c->l2_bytes / 3 * 2;     // choose_log_cap's L2 budget
    t.max_probe = chain_limit(max_inserts != ~0ull);              // no insert limit: the table is at its final size
    if constexpr (IN != IN_TABLE) {
        // bulk-staged (copy engine) variant: 16-byte aligned inputs of at least a few tiles per CTA
        const bool aligned = (((uintptr_t)a | (uintptr_t)(b ? b : a)) & 15u) == 0;
        if (aligned && n >= (u64)HB_TILE * 64) {
            auto kb = hash_agg_bulk_kernel<IN, OPK, TX>;
            constexpr bool has_v = (IN == IN_AOS) || (OPK != OPK_COUNT && OPK != OPK_DICT);
            const size_t smem = hb_smem_bytes(has_v);
            if (c->occ_cache.find((const void *)kb) == c->occ_cache.end())
                CU(cudaFuncSetAttribute(kb, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int occ = occupancy(c, kb, HB_THREADS, smem);
            u64 grid = std::min<u64>(n / HB_TILE, (u64)c->sm_count * occ);
            KLaunch kl(s, klass, n);
            if (klass == K_HASH_AGG) s->st.hot_kernel_variant = 1;
            kb<<<(unsigned)grid, HB_THREADS, smem, c->stream>>>(a, b, n, t, ctl, max_inserts, slot_out);
            return kl.done("hash_agg_bulk_kernel");
        }
    }
    auto kern = hash_agg_kernel<IN, OPK, TX>;
    int occ = occupancy(c, kern, HA_THREADS, 0);
    u64 tiles = (n + HA_TILE - 1) / HA_TILE;
    u64 grid = std::min<u64>(tiles, (u64)c->sm_count * occ);
    if (grid == 0) return VB_OK;
    KLaunch kl(s, klass, n);
    kern<<<(unsigned)grid, HA_THREADS, 0, c->stream>>>(a, b, n, t, ctl, max_inserts, slot_out);
    return kl.done("hash_agg_kernel");
}

template <int IN>
static int launch_hash_agg_in(vb_shuf *s, int klass, int opk, int tx, const u64 *a, const u64 *b, u64 n, void *tab,
                              u32 log_cap, TableCtl *ctl, u64 mi, u32 *so)
{
#define HA(O, T) return launch_hash_agg_t<IN, O, T>(s, klass, a, b, n, tab, log_cap, ctl, mi, so)
    switch (opk) {
    case OPK_ADD_U64: HA(OPK_ADD_U64, TX_NONE);
    case OPK_ADD_F64: HA(OPK_ADD_F64, TX_NONE);
    case OPK_COUNT: if constexpr (IN != IN_TABLE) { HA(OPK_COUNT, TX_NONE); } break;
    case OPK_DICT: if constexpr (IN != IN_TABLE) { HA(OPK_DICT, TX_NONE); } break;
    case OPK_MIN_U64:
        if (IN == IN_TABLE || tx == TX_NONE) HA(OPK_MIN_U64, TX_NONE);
        if (tx == TX_I64) HA(OPK_MIN_U64, (IN == IN_TABLE ? TX_NONE : TX_I64));
        HA(OPK_MIN_U64, (IN == IN_TABLE ? TX_NONE : TX_F64));
    case OPK_MAX_U64:
        if (IN == IN_TABLE || tx == TX_NONE) HA(OPK_MAX_U64, TX_NONE);
        if (tx == TX_I64) HA(OPK_MAX_U64, (IN == IN_TABLE ? TX_NONE : TX_I64));
        HA(OPK_MAX_U64, (IN == IN_TABLE ? TX_NONE : TX_F64));
    }
#undef HA
    return set_err(VB_ERR_UNSUPPORTED, "hash_agg: unsupported op %d for input mode %d", opk, IN);
}

static int launch_hash_agg(vb_shuf *s, int klass, int in, int opk, int tx, const u64 *a, const u64 *b, u64 n, void *tab,
                           u32 log_cap, TableCtl *ctl, u64 mi, u32 *so)
{
    switch (in) {
    case IN_AOS: return launch_hash_agg_in<IN_AOS>(s, klass, opk, tx, a, b, n, tab, log_cap, ctl, mi, so);
    case IN_SOA: return launch_hash_agg_in<IN_SOA>(s, klass, opk, tx, a, b, n, tab, log_cap, ctl, mi, so);
    case IN_TABLE: return launch_hash_agg_in<IN_TABLE>(s, klass, opk, tx, a, b, n, tab, log_cap, ctl, mi, so);
    }
    return set_err(VB_ERR_INVALID, "hash_agg: bad input mode %d", in);
}

// Multi-aggregate combine: keys + NV value columns (IN_SOA), or a source table of the same spec (IN_TABLE).
template <int IN, int NV>
static int launch_hash_agg_multi_t(vb_shuf *s, int klass, const AccSpec &sp, const u64 *keys, const MaCols &cols, u64 n, void *tab,
                                   u32 log_cap, TableCtl *ctl, u64 max_inserts)
{
    vb_ctx *c = s->ctx;
    Table t = table_at(tab, log_cap);
    t.max_probe = chain_limit(max_inserts != ~0ull);              // no insert limit: the table is at its final size
    if constexpr (IN == IN_SOA) {
        uintptr_t addr = (uintptr_t)keys;
        for (int i = 0; i < NV; ++i) addr |= (uintptr_t)cols.c[i];
        constexpr u64 tile = (u64)HA_THREADS * ma_rows<NV>();
        if ((addr & 15u) == 0 && n >= tile * 64) {
            auto kb = hash_agg_multi_bulk_kernel<NV>;
            const size_t smem = ma_bulk_smem<NV>(MA_MAX_ACCS);     // sized for the widest spec: one occupancy for every spec
            if (c->occ_cache.find((const void *)kb) == c->occ_cache.end())
                CU(cudaFuncSetAttribute(kb, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const int occ = occupancy(c, kb, HB_THREADS, smem);
            const u64 grid = std::min<u64>(n / tile, (u64)c->sm_count * occ);
            KLaunch kl(s, klass, n);
            if (klass == K_HASH_AGG) s->st.hot_kernel_variant = 1;
            kb<<<(unsigned)grid, HB_THREADS, smem, c->stream>>>(keys, cols, n, t, sp, ctl, max_inserts);
            return kl.done("hash_agg_multi_bulk_kernel");
        }
    }
    auto kern = hash_agg_multi_kernel<IN, NV>;
    const size_t smem = IN == IN_SOA ? ma_cache_bytes(MA_MAX_ACCS) : 0;
    const int occ = occupancy(c, kern, HA_THREADS, smem);
    const u64 tile = (u64)HA_THREADS * ma_rows<NV>();
    const u64 grid = std::min<u64>((n + tile - 1) / tile, (u64)c->sm_count * occ);
    if (grid == 0) return VB_OK;
    KLaunch kl(s, klass, n);
    kern<<<(unsigned)grid, HA_THREADS, smem, c->stream>>>(keys, cols, n, t, sp, ctl, max_inserts);
    return kl.done("hash_agg_multi_kernel");
}

static int launch_hash_agg_multi(vb_shuf *s, int klass, const AccSpec &sp, const AggInput &in, const u64 *keys, const u64 *const *vcols,
                                 u64 n, void *tab, u32 log_cap, TableCtl *ctl, u64 mi)
{
    MaCols mc{};
    if (in.in == IN_TABLE) {
        mc.c[0] = in.b;
        mc.stride = (in.n - 1) + BUCKET;                    // the source has in.n - 1 regular slots
        return launch_hash_agg_multi_t<IN_TABLE, 1>(s, klass, sp, keys, mc, n, tab, log_cap, ctl, mi);
    }
    if (in.in == IN_ACCS) {
        mc.c[0] = in.b;
        mc.stride = in.n;                                   // received partials: [n_acc][in.n]
        return launch_hash_agg_multi_t<IN_ACCS, 1>(s, klass, sp, keys, mc, n, tab, log_cap, ctl, mi);
    }
    for (u32 i = 0; i < s->n_cols; ++i) mc.c[i] = vcols[i];
    switch (s->n_cols) {
    case 1: return launch_hash_agg_multi_t<IN_SOA, 1>(s, klass, sp, keys, mc, n, tab, log_cap, ctl, mi);
    case 2: return launch_hash_agg_multi_t<IN_SOA, 2>(s, klass, sp, keys, mc, n, tab, log_cap, ctl, mi);
    case 3: return launch_hash_agg_multi_t<IN_SOA, 3>(s, klass, sp, keys, mc, n, tab, log_cap, ctl, mi);
    case 4: return launch_hash_agg_multi_t<IN_SOA, 4>(s, klass, sp, keys, mc, n, tab, log_cap, ctl, mi);
    }
    return set_err(VB_ERR_INVALID, "hash_agg_multi: %u value columns", s->n_cols);
}

static int init_table(vb_shuf *s, void *tab, u32 log_cap, int opk, const AccSpec *ms)
{
    vb_ctx *c = s->ctx;
    KLaunch kl(s, K_MISC);
    const u64 blocks = std::min<u64>((acc_stride(log_cap) + 255) / 256, (u64)c->sm_count * 8);
    if (ms) table_init_multi_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(table_at(tab, log_cap), *ms);
    else table_init_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(table_at(tab, log_cap), op_identity(opk));
    return kl.done(ms ? "table_init_multi_kernel" : "table_init_kernel");
}

constexpr u64 HOST_CHUNK_ROWS = 8ull << 20;    // host inputs stream through two 128 MiB staging halves (double-buffered)

// vega issues its map tasks concurrently from a tokio blocking pool (local_scheduler.rs:336-352).  A map call holds
// the context lock while it ENQUEUES copies and kernels, but waits for its own completion (table overflow flag,
// insert count) with the lock released, so the next task's H2D copies queue up behind this one's without a gap.
static thread_local std::unique_lock<std::mutex> *tl_ctx_lock = nullptr;

// D2H of `bytes` (<= 64) from `dev` at the current end of c->stream, waited for with the context unlocked.
static int fetch_status_unlocked(vb_ctx *c, const void *dev, void *out, size_t bytes)
{
    if (!tl_ctx_lock || c->pinned_slots.empty()) {          // not inside a map call: plain synchronous fetch
        CU(cudaMemcpyAsync(c->h_scratch, dev, bytes, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        memcpy(out, c->h_scratch, bytes);
        return VB_OK;
    }
    void *slot = c->pinned_slots.back();
    c->pinned_slots.pop_back();
    cudaEvent_t ev;
    CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    cudaError_t e = cudaMemcpyAsync(slot, dev, bytes, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaEventRecord(ev, c->stream);
    tl_ctx_lock->unlock();
    if (e == cudaSuccess) e = cudaEventSynchronize(ev);
    tl_ctx_lock->lock();
    cudaSetDevice(c->device);
    memcpy(out, slot, bytes);
    c->pinned_slots.push_back(slot);
    cudaEventDestroy(ev);
    if (e != cudaSuccess) { cudaGetLastError(); return set_err(VB_ERR_CUDA, "status fetch: %s", cudaGetErrorString(e)); }
    return VB_OK;
}
constexpr u32 MAX_LOG_CAP = 31;

static int launch_hash_agg(vb_shuf *s, int klass, int in, int opk, int tx, const u64 *a, const u64 *b, u64 n, void *tab,
                           u32 log_cap, TableCtl *ctl, u64 mi, u32 *so);

// Distinct-count estimate from a strided sample of up to 2^20 keys of the first device-resident
// input: insert the sample into a scratch dictionary, read the number of distinct keys d_s, and
// solve d_s = D (1 - exp(-s / D)) for D (keys assumed roughly equally frequent).  Returns 0 when
// there is nothing to sample; a sample that is ~all distinct only proves D >~ 25 s.
static int estimate_distinct(vb_shuf *s, const std::vector<AggInput> &inputs, u64 total, u64 *out)
{
    vb_ctx *c = s->ctx;
    *out = 0;
    const AggInput *src = nullptr;
    for (auto &in : inputs)
        if (in.loc != VB_HOST && in.n && (in.in == IN_AOS || in.in == IN_SOA)) { src = &in; break; }
    if (!src) return VB_OK;
    const u32 m = (u32)std::min<u64>(src->n, 1u << 20);
    const u64 stride = std::max<u64>(1, src->n / m);
    const u32 log_cap = 21;
    DevBuf keys(c), tab(c), ctl(c), slots(c);
    TRY(keys.alloc((size_t)m * 8));
    TRY(slots.alloc((size_t)m * 4));
    TRY(tab.alloc(table_bytes(log_cap)));
    TRY(ctl.alloc(sizeof(TableCtl)));
    CU(cudaMemsetAsync(ctl.p, 0, sizeof(TableCtl), c->stream));
    {
        KLaunch kl(s, K_MISC);
        table_init_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(table_at(tab.p, log_cap), 0);
        TRY(kl.done("table_init_kernel"));
    }
    {
        KLaunch kl(s, K_MISC);
        if (src->in == IN_AOS) sample_keys_kernel<IN_AOS><<<(m + 255) / 256, 256, 0, c->stream>>>(src->a, src->n, stride, keys.as<u64>(), m);
        else sample_keys_kernel<IN_SOA><<<(m + 255) / 256, 256, 0, c->stream>>>(src->a, src->n, stride, keys.as<u64>(), m);
        TRY(kl.done("sample_keys_kernel"));
    }
    TRY(launch_hash_agg(s, K_MISC, IN_SOA, OPK_DICT, TX_NONE, keys.as<u64>(), nullptr, m, tab.p, log_cap, ctl.as<TableCtl>(), ~0ull,
                        slots.as<u32>()));
    TableCtl *h = (TableCtl *)c->h_scratch;
    CU(cudaMemcpyAsync(h, ctl.p, sizeof(TableCtl), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    const double ds = (double)h->n_inserted + 1.0, sm = (double)m;
    double D;
    if (ds >= 0.98 * sm) {
        D = std::min<double>((double)total, 32.0 * sm);     // unresolved: at least ~25 s distinct keys
        if (src->n <= m) D = ds;                             // the sample was the whole input
    } else {
        double lo = ds, hi = 64.0 * sm;                      // d(D) = D (1 - exp(-s/D)) is increasing in D
        for (int it = 0; it < 60; ++it) {
            double mid = 0.5 * (lo + hi);
            if (mid * (1.0 - exp(-sm / mid)) < ds) lo = mid; else hi = mid;
        }
        D = hi;
    }
    *out = (u64)std::min<double>((double)total, D * 1.25 + 16.0);
    return VB_OK;
}

// First table size.  Load factor <= 0.4 while the table (16 B/slot) still fits comfortably in L2, where a fuller
// 4-key bucket costs a second dependent probe; <= 0.5 for bigger tables, which pay DRAM traffic instead.
// When the load-0.4 table would spill out of L2 (2/3 of it is the budget: the input stream passes through the rest)
// but a table at load <= 0.5 of an *estimated* key count fits, the fuller L2-resident table is taken (the estimate
// already carries a 1.25x margin, so the real load stays under the 0.6 restart threshold).
// slot_bytes: 16 for a single accumulator, 8 * (1 + n_acc) for a multi-aggregate table.
static u32 choose_log_cap(u64 total, u64 hint_distinct, bool estimated, u32 max_log, u64 l2_bytes, u32 slot_bytes = 16)
{
    u64 target = hint_distinct ? (hint_distinct * 5) / 2 : std::min<u64>(2 * std::max<u64>(total, 1), 1ull << 21);
    if (hint_distinct && target > (1ull << 22)) target = 2 * hint_distinct;
    const u64 budget = l2_bytes / 3 * 2;
    auto bytes = [&](u32 lc) { return (((u64)1 << lc) + BUCKET) * slot_bytes; };
    if (estimated && bytes(ceil_log2_u64(target)) > budget &&
        bytes(ceil_log2_u64(hint_distinct * 8 / 5)) <= budget)
        target = hint_distinct * 8 / 5;
    // an estimate from a sample is a lower bound under skew: never start a large input below 2^21 slots (32 MB)
    if (estimated) target = std::max<u64>(target, 1ull << 21);
    return std::min(max_log, std::max<u32>(4, ceil_log2_u64(target)));
}

// Tables of 2^23 slots (128 MB) and more are far larger than the 50 MB L2: every probe and every RED becomes a
// random DRAM access.  Such inputs are first radix-partitioned by the top bits of the slot hash (one stable pass),
// so that consecutive tiles of hash_agg_kernel all probe the same <= 32 MB region of the table, which then
// stays L2-resident while it is being filled.  Reduce ops on device-resident rows only (the dictionary of group ops
// must keep row order, host inputs are PCIe-bound anyway).
struct PassPlan;
template <typename KeyT, bool HAS_VAL> static PassPlan plan_pass(vb_ctx *c, u64 n);
template <typename KeyT, bool HAS_VAL>
static int radix_pass(vb_shuf *s, const Loader &ld, const Digit &dg, u64 n, KeyT *out_keys, u64 *out_vals, u32 *d_hist, const PassPlan &plan,
                      u64 *csr = nullptr, bool *csr_done = nullptr);

constexpr u32 PARTITION_MIN_LOG_CAP = 23;

static bool want_partition(int in, int opk, u32 log_cap, u64 n)
{
    return opk != OPK_DICT && (in == IN_AOS || in == IN_SOA) && log_cap >= PARTITION_MIN_LOG_CAP && n >= (1ull << 22);
}

static int launch_hash_agg_partitioned(vb_shuf *s, int klass, int in, int opk, int tx, const u64 *a, const u64 *b, u64 n, void *tab,
                                       u32 log_cap, TableCtl *ctl, u64 mi);

// Feed every input into one fresh table; on overflow (abort flag) start again 4x larger.
// slot_out (OPK_DICT): one u32 per row over the concatenation of the inputs.
// ms != nullptr: a multi-aggregate table with these accumulators (opk / tx unused); inputs carry value columns.
static int build_table(vb_shuf *s, int klass, const std::vector<AggInput> &inputs, int opk, int tx, u64 hint_distinct,
                       void **out_tab, u32 *out_log_cap, u64 *out_inserted, u32 *slot_out, const AccSpec *ms = nullptr)
{
    vb_ctx *c = s->ctx;
    u64 total = 0;          // items that can each bring a new key (table inputs: occupied slots, not capacity)
    bool any_host = false;
    u64 max_host = 0;
    for (auto &in : inputs) {
        total += in.items ? std::min(in.items, in.n) : in.n;
        if (in.loc == VB_HOST) { any_host = true; max_host = std::max(max_host, in.n); }
    }
    if (slot_out && any_host) return set_err(VB_ERR_INVALID, "build_table: dictionary inputs must be on the device");
    // capacity never needs to exceed 2x the items; slot indices are 32-bit, so 2^31 slots is the ceiling — an input
    // with more than ~1.3e9 distinct keys fails with "overflow at maximum capacity", fewer distinct keys fit whatever the row
    // count and wherever they hash: a table of max_log slots holds at most half as many keys, so it runs without an insert
    // limit and no probe-round limit (chain_limit).  Only above 2^30 items, where the 2^31-slot ceiling can be over half
    // full, does the table keep the 0.6 insert limit and the HA_MAX_PROBE round limit.
    const u32 max_log = std::min<u32>(MAX_LOG_CAP, std::max<u32>(4, ceil_log2_u64(2 * std::max<u64>(total, 1))));
    bool estimated = false;
    if (!hint_distinct && total > (1ull << 20)) { TRY(estimate_distinct(s, inputs, total, &hint_distinct)); estimated = true; }
    const u32 slot_bytes = ms ? 8 * (1 + ms->n) : 16;
    u32 log_cap = choose_log_cap(total, hint_distinct, estimated, max_log, c->l2_bytes, slot_bytes);

    DevBuf ctl(c), stage_a(c), stage_b(c);
    TRY(ctl.alloc(sizeof(TableCtl)));
    const u64 stage_rows = std::min(max_host, HOST_CHUNK_ROWS);
    const u64 row_bytes = ms ? 8 * (1 + s->n_cols) : 16;
    bool half_used[2] = {false, false};
    if (any_host) {
        // per half: AoS rows, or SoA keys in the first 8 B/row / vals (multi: each value column) in the next
        TRY(stage_a.alloc(stage_rows * row_bytes));
        TRY(stage_b.alloc(stage_rows * row_bytes));
        CU(cudaEventRecord(c->ev_ready, c->stream));               // the pool hands the halves out in stream order
        CU(cudaStreamWaitEvent(c->copy_stream, c->ev_ready, 0));
    }
    TableCtl h_ctl_v;
    TableCtl *h_ctl = &h_ctl_v;
    for (;;) {
        const u64 cap = 1ull << log_cap;
        DevBuf tab(c);
        TRY(tab.alloc(ms ? table_bytes_multi(log_cap, ms->n) : table_bytes(log_cap)));
        TRY(init_table(s, tab.p, log_cap, opk, ms));
        CU(cudaMemsetAsync(ctl.p, 0, sizeof(TableCtl), c->stream));
        const u64 max_inserts = (log_cap == max_log && cap >= 2 * total) ? ~0ull : (cap / 10) * 6;
        u64 row_base = 0;
        for (auto &in : inputs) {
            if (in.n == 0) continue;
            if (ms && in.loc != VB_HOST) {             // partition-first building moves one value column: not for multi tables
                TRY(launch_hash_agg_multi(s, klass, *ms, in, in.a, in.cols, in.n, tab.p, log_cap, ctl.as<TableCtl>(), max_inserts));
            } else if (in.loc != VB_HOST && !slot_out && want_partition(in.in, opk, log_cap, in.n)) {
                TRY(launch_hash_agg_partitioned(s, klass, in.in, opk, tx, in.a, in.b, in.n, tab.p, log_cap, ctl.as<TableCtl>(), max_inserts));
            } else if (in.loc != VB_HOST) {
                TRY(launch_hash_agg(s, klass, in.in, opk, tx, in.a, in.b, in.n, tab.p, log_cap, ctl.as<TableCtl>(),
                                    max_inserts, slot_out ? slot_out + row_base : nullptr));
            } else {
                // double-buffered: the copy engine fills one half on the copy stream while hash_agg consumes the other
                const u64 chunk = std::min(in.n, stage_rows);
                u32 it = 0;
                for (u64 off = 0; off < in.n; off += chunk, ++it) {
                    const u64 m = std::min(chunk, in.n - off);
                    const u32 hb = it & 1u;
                    u64 *half = hb ? stage_b.as<u64>() : stage_a.as<u64>();
                    const u64 *da = half, *db = nullptr;
                    if (half_used[hb]) CU(cudaStreamWaitEvent(c->copy_stream, c->ev_kernel[hb], 0));   // its last reader is done
                    const u64 *vc[MA_MAX_COLS] = {};
                    if (ms) {
                        CU(cudaMemcpyAsync(half, in.a + off, m * 8, cudaMemcpyHostToDevice, c->copy_stream));
                        s->st.h2d_bytes += m * 8;
                        for (u32 col = 0; col < s->n_cols; ++col) {
                            if (!in.cols[col]) continue;
                            vc[col] = half + (u64)(1 + col) * chunk;
                            CU(cudaMemcpyAsync((void *)vc[col], in.cols[col] + off, m * 8, cudaMemcpyHostToDevice, c->copy_stream));
                            s->st.h2d_bytes += m * 8;
                        }
                    } else if (in.in == IN_AOS) {
                        CU(cudaMemcpyAsync(half, in.a + 2 * off, m * 16, cudaMemcpyHostToDevice, c->copy_stream));
                        s->st.h2d_bytes += m * 16;
                    } else {
                        CU(cudaMemcpyAsync(half, in.a + off, m * 8, cudaMemcpyHostToDevice, c->copy_stream));
                        s->st.h2d_bytes += m * 8;
                        if (in.b) {
                            db = half + chunk;
                            CU(cudaMemcpyAsync((void *)db, in.b + off, m * 8, cudaMemcpyHostToDevice, c->copy_stream));
                            s->st.h2d_bytes += m * 8;
                        }
                    }
                    CU(cudaEventRecord(c->ev_copied[hb], c->copy_stream));
                    CU(cudaStreamWaitEvent(c->stream, c->ev_copied[hb], 0));
                    if (ms) TRY(launch_hash_agg_multi(s, klass, *ms, in, da, vc, m, tab.p, log_cap, ctl.as<TableCtl>(), max_inserts));
                    else TRY(launch_hash_agg(s, klass, in.in, opk, tx, da, db, m, tab.p, log_cap, ctl.as<TableCtl>(), max_inserts, nullptr));
                    CU(cudaEventRecord(c->ev_kernel[hb], c->stream));
                    half_used[hb] = true;
                }
            }
            row_base += in.n;
        }
        TRY(fetch_status_unlocked(c, ctl.p, h_ctl, sizeof(TableCtl)));     // waits with the context unlocked inside a map call
        if (!h_ctl->abort) {
            *out_tab = tab.release();
            *out_log_cap = log_cap;
            *out_inserted = h_ctl->n_inserted;
            s->st.table_slots = std::max<u64>(s->st.table_slots, cap);
            return VB_OK;
        }
        if (log_cap >= max_log) return set_err(VB_ERR_CUDA, "hash table overflow at maximum capacity 2^%u (internal error)", log_cap);
        log_cap = std::min(max_log, log_cap + 2);
        s->st.table_restarts++;
    }
}

// ---------------------------------------------------------------------------------------------
// radix pass host side
// ---------------------------------------------------------------------------------------------
struct PassPlan {
    u32 num_parts = 0;
    u64 rows_per_part = 0;
    size_t hist_bytes() const { return ((size_t)RP_NB * num_parts + 1) * sizeof(u32); }
};

// (LDM, DGM) combinations the engine passes per row type; anything else is a programming error.
//   (u64, u64): seal_sort, the multisplits (a repartition's with the position loader) and the partition-first hash aggregate;
//   u64 key only: seal_sort;  (u32 id, u64): sort_id_pairs.
#define RP_COMBOS_U64V(X)                                                                            \
    X(LD_SOA64, DG_BITS) X(LD_AOS64, DG_BITS) X(LD_SOA64, DG_BUCKET) X(LD_TABLE_KV, DG_BUCKET)         \
    X(LD_TABLE_KI, DG_BUCKET) X(LD_SOA64, DG_DEST) X(LD_AOS64, DG_DEST) X(LD_SOA64, DG_HASHTOP)        \
    X(LD_AOS64, DG_HASHTOP) X(LD_POS, DG_BUCKET)
#define RP_COMBOS_U64K(X) X(LD_SOA64, DG_BITS)
#define RP_COMBOS_U32V(X) X(LD_KEY32_VAL_SOA, DG_BITS) X(LD_KEY32_VAL_AOS, DG_BITS)

template <typename KeyT, int LDM> constexpr bool rp_key_ok()
{
    return (LDM == LD_KEY32_VAL_SOA || LDM == LD_KEY32_VAL_AOS) ? sizeof(KeyT) == 4 : sizeof(KeyT) == 8;
}

template <typename KeyT, bool HAS_VAL>
static const void *scatter_fn(int ldm, int dgm)
{
#define X(L, D) if (ldm == L && dgm == D) return (const void *)rp_scatter_kernel<KeyT, HAS_VAL, L, D>;
    if constexpr (sizeof(KeyT) == 8 && HAS_VAL) { RP_COMBOS_U64V(X) }
    if constexpr (sizeof(KeyT) == 8 && !HAS_VAL) { RP_COMBOS_U64K(X) }
    if constexpr (sizeof(KeyT) == 4 && HAS_VAL) { RP_COMBOS_U32V(X) }
#undef X
    return nullptr;
}

template <typename KeyT>
static const void *hist_fn(int ldm, int dgm)
{
#define X(L, D) if (ldm == L && dgm == D) return (const void *)rp_hist_kernel<KeyT, L, D>;
    if constexpr (sizeof(KeyT) == 8) { RP_COMBOS_U64V(X) }     // covers the key-only pairs
    if constexpr (sizeof(KeyT) == 4) { RP_COMBOS_U32V(X) }
#undef X
    return nullptr;
}

// The gather sweep (gsweep.cuh) is the scatter of the DG_BITS passes.
template <typename KeyT, bool HAS_VAL>
static bool gsweep_lookup(int ldm, const void **kern, size_t *smem, u32 *tile, u32 *threads)
{
#define X(L)                                                                 \
    if (ldm == L) {                                                          \
        if constexpr (rp_key_ok<KeyT, L>() && (HAS_VAL || L == LD_SOA64)) { \
            *kern = (const void *)rp_gsweep_kernel<KeyT, HAS_VAL, L>;        \
            *smem = GsPlan<KeyT, HAS_VAL, L>::total;                         \
            *tile = (u32)GsPlan<KeyT, HAS_VAL, L>::T;                        \
            *threads = (u32)GsPlan<KeyT, HAS_VAL, L>::THREADS;               \
            return true;                                                     \
        }                                                                    \
    }
    X(LD_SOA64) X(LD_AOS64) X(LD_KEY32_VAL_SOA) X(LD_KEY32_VAL_AOS)
#undef X
    return false;
}

template <typename KeyT, bool HAS_VAL>
static PassPlan plan_pass(vb_ctx *c, u64 n)
{
    PassPlan p;
    if (n == 0) return p;
    // one part per resident CTA of the gather sweep
    const int occ = GsPlan<KeyT, HAS_VAL, (sizeof(KeyT) == 4 ? LD_KEY32_VAL_SOA : LD_SOA64)>::CTAS;
    u64 tiles = (n + RP_TILE - 1) / RP_TILE;
    u64 parts = std::min<u64>(tiles, (u64)c->sm_count * occ);
    u64 tiles_per_part = (tiles + parts - 1) / parts;
    if (tiles_per_part > 6) tiles_per_part = (tiles_per_part + 5) / 6 * 6;   // 24576-row units: a multiple of the sweep tile (6144 rows)
    p.rows_per_part = tiles_per_part * RP_TILE;
    p.num_parts = (u32)((n + p.rows_per_part - 1) / p.rows_per_part);
    return p;
}

// One stable pass: rows of `ld` (n of them) are written to out_keys/out_vals grouped by digit.
// d_hist (device, plan.hist_bytes()) afterwards holds the scanned histogram: d_hist[d*num_parts]
// is the output offset of digit d, d_hist[nb*num_parts] the number of valid rows.
template <typename KeyT>
static int radix_hist_scan(vb_shuf *s, const Loader &ld, const Digit &dg, u64 n, u32 *d_hist, const PassPlan &plan)
{
    vb_ctx *c = s->ctx;
    if (n == 0 || plan.num_parts == 0) return VB_OK;
    const void *hk = hist_fn<KeyT>(ld.mode, dg.mode);
    if (!hk) return set_err(VB_ERR_UNSUPPORTED, "radix pass: loader %d / digit %d not instantiated", ld.mode, dg.mode);
    const u64 tiles_per_part = plan.rows_per_part / RP_TILE;
    u32 split = (u32)std::max<u64>(1, std::min<u64>(tiles_per_part, ((u64)c->sm_count * 6 + plan.num_parts - 1) / plan.num_parts));
    CU(cudaMemsetAsync(d_hist, 0, plan.hist_bytes(), c->stream));
    u64 rows_per_part = plan.rows_per_part;
    u32 num_parts = plan.num_parts;
    Loader ldc = ld;
    Digit dgc = dg;
    {
        KLaunch kl(s, K_RP_HIST, n);
        void *args[] = {&ldc, &dgc, &n, &rows_per_part, &d_hist, &num_parts, &split};
        const size_t hsmem = rp_hist_smem();
        CU(cudaFuncSetAttribute(hk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hsmem));
        CU(cudaLaunchKernel(hk, dim3(plan.num_parts * split), dim3(RP_THREADS), args, hsmem, c->stream));
        TRY(kl.done("rp_hist_kernel"));
    }
    {
        KLaunch kl(s, K_RP_SCAN);
        rp_scan_kernel<<<1, 1024, 0, c->stream>>>(d_hist, RP_NB * plan.num_parts);
        TRY(kl.done("rp_scan_kernel"));
    }
    return VB_OK;
}

// Row-stream loader / digit pairs of the (u64, u64) multisplits rp_sweep_kernel is instantiated for (sweep.cuh).
// The DG_BITS passes never reach it: where the gather sweep's n >= 4 x its tile fails and the sweep's would hold,
// plan_pass gives 4096-row parts, which the sweep tile does not divide.
#define SW_COMBOS(X) X(LD_SOA64, DG_DEST) X(LD_AOS64, DG_DEST) X(LD_SOA64, DG_HASHTOP) X(LD_AOS64, DG_HASHTOP) X(LD_SOA64, DG_BUCKET)

template <typename KeyT, bool HAS_VAL>
static int radix_pass(vb_shuf *s, const Loader &ld, const Digit &dg, u64 n, KeyT *out_keys, u64 *out_vals, u32 *d_hist,
                      const PassPlan &plan, u64 *csr, bool *csr_done)
{
    vb_ctx *c = s->ctx;
    if (n == 0 || plan.num_parts == 0) return VB_OK;
    const void *sk = scatter_fn<KeyT, HAS_VAL>(ld.mode, dg.mode);
    if (!sk) return set_err(VB_ERR_UNSUPPORTED, "radix pass: loader %d / digit %d not instantiated", ld.mode, dg.mode);
    TRY((radix_hist_scan<KeyT>(s, ld, dg, n, d_hist, plan)));
    {   // LSD digit passes over row streams: the gather sweep (two 512-thread CTAs per SM, rows stay where the copy engine put them)
        const void *gk = nullptr;
        size_t gsm = 0;
        u32 GT = 0, gthreads = 0;
        if (dg.mode == DG_BITS && n < SW_ROW_LIMIT && plan.rows_per_part % 4096 == 0 &&
            gsweep_lookup<KeyT, HAS_VAL>(ld.mode, &gk, &gsm, &GT, &gthreads) && n >= 4ull * GT &&
            !(((uintptr_t)ld.keys & 15u) || (ld.vals && ((uintptr_t)ld.vals & 15u))) && !(HAS_VAL && ld.mode != LD_AOS64 && !ld.vals)) {
            if (c->occ_cache.find(gk) == c->occ_cache.end()) CU(cudaFuncSetAttribute(gk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm));
            (void)occupancy(c, gk, (int)gthreads, gsm);
            SweepArgs a{};
            a.keys = ld.keys; a.vals = ld.vals; a.n = n; a.n_tiles = 0;
            a.out_keys = out_keys; a.out_vals = out_vals;
            a.part_off = d_hist; a.num_parts = plan.num_parts; a.rows_per_part = plan.rows_per_part;
            if constexpr (sizeof(KeyT) == 4 && HAS_VAL) {
                // last pass of group_by_key's sort: value-run starts recorded by the scatter itself, ids not written (rp_gsweep_kernel<CSR>)
                if (csr && ld.mode == LD_KEY32_VAL_SOA) {
                    const void *ck = (const void *)rp_gsweep_kernel<u32, true, LD_KEY32_VAL_SOA, true>;
                    if (c->occ_cache.find(ck) == c->occ_cache.end()) CU(cudaFuncSetAttribute(ck, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm));
                    (void)occupancy(c, ck, (int)gthreads, gsm);
                    gk = ck;
                    a.csr = csr;
                    if (csr_done) *csr_done = true;
                }
            }
            Digit dgs = dg;
            KLaunch kl(s, K_RP_SCATTER, n);
            void *args[] = {&a, &dgs};
            CU(cudaLaunchKernel(gk, dim3(plan.num_parts), dim3(gthreads), args, gsm, c->stream));
            return kl.done("rp_gsweep_kernel");
        }
    }
    if constexpr (sizeof(KeyT) == 8 && HAS_VAL) {   // multisplits of row streams: the sweep tile pipeline fed by the per-part offsets
        const void *sw = nullptr;
        size_t swsm = 0;
#define X(L, D) if (ld.mode == L && dg.mode == D) { sw = (const void *)rp_sweep_kernel<L, D>; swsm = SwSmem<L>::total; }
        SW_COMBOS(X)
#undef X
        const u32 T = SW_TILE;
        if (sw && n < SW_ROW_LIMIT && plan.rows_per_part % T == 0 && n >= 4ull * T &&
            !(((uintptr_t)ld.keys & 15u) || (ld.vals && ((uintptr_t)ld.vals & 15u))) && !(ld.mode != LD_AOS64 && !ld.vals)) {
            if (c->occ_cache.find(sw) == c->occ_cache.end()) CU(cudaFuncSetAttribute(sw, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)swsm));
            (void)occupancy(c, sw, SW_THREADS, swsm);
            SweepArgs a{};
            a.keys = ld.keys; a.vals = ld.vals; a.n = n; a.n_tiles = (u32)((n + T - 1) / T);
            a.out_keys = out_keys; a.out_vals = out_vals;
            a.part_off = d_hist; a.num_parts = plan.num_parts; a.rows_per_part = plan.rows_per_part;
            Digit dgs = dg;
            KLaunch kl(s, K_RP_SCATTER, n);
            void *args[] = {&a, &dgs};
            CU(cudaLaunchKernel(sw, dim3(plan.num_parts), dim3(SW_THREADS), args, swsm, c->stream));
            return kl.done("rp_sweep_kernel");
        }
    }
    const size_t smem = rp_scatter_smem<KeyT, HAS_VAL>();
    CU(cudaFuncSetAttribute(sk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    u64 rows_per_part = plan.rows_per_part;
    u32 num_parts = plan.num_parts;
    Loader ldc = ld;
    Digit dgc = dg;
    {
        KLaunch kl(s, K_RP_SCATTER, n);
        const u32 *ch = d_hist;
        RemoteDst rd{nullptr, nullptr, nullptr, 0};
        void *args[] = {&ldc, &dgc, &n, &rows_per_part, &ch, &num_parts, &out_keys, &out_vals, &rd};
        CU(cudaLaunchKernel(sk, dim3(plan.num_parts), dim3(RPS_THREADS), args, smem, c->stream));
        TRY(kl.done("rp_scatter_kernel"));
    }
    return VB_OK;
}

static int launch_hash_agg_partitioned(vb_shuf *s, int klass, int in, int opk, int tx, const u64 *a, const u64 *b, u64 n, void *tab,
                                       u32 log_cap, TableCtl *ctl, u64 mi)
{
    vb_ctx *c = s->ctx;
    const u32 pbits = std::min<u32>(8, log_cap - 21);          // regions of <= 2^21 slots (32 MB) while 256 bins suffice
    DevBuf tk(c), tv(c), hist(c);
    TRY(tk.alloc(n * 8));
    TRY(tv.alloc(n * 8));
    PassPlan plan = plan_pass<u64, true>(c, n);
    TRY(hist.alloc(plan.hist_bytes()));
    Loader ld = (in == IN_AOS) ? Loader{LD_AOS64, a, nullptr, 0} : Loader{LD_SOA64, a, b, 0};
    Digit dg{};
    dg.mode = DG_HASHTOP;
    dg.shift = 64 - pbits;
    dg.mask = (1u << pbits) - 1;
    TRY((radix_pass<u64, true>(s, ld, dg, n, tk.as<u64>(), tv.as<u64>(), hist.as<u32>(), plan)));
    // stream-ordered frees: the buffers outlive the kernels queued on c->stream
    return launch_hash_agg(s, klass, IN_SOA, opk, tx, tk.as<u64>(), tv.as<u64>(), n, tab, log_cap, ctl, mi, nullptr);
}

// Copy the start offset of each of the first nb digits plus the total to the host: out[nb+1].
static int fetch_offsets(vb_ctx *c, const u32 *d_hist, const PassPlan &plan, u32 nb, u64 *out)
{
    u32 *h = (u32 *)c->h_scratch;
    CU(cudaMemcpy2DAsync(h, sizeof(u32), d_hist, (size_t)plan.num_parts * sizeof(u32), sizeof(u32), RP_NB,
                         cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(h + RP_NB, d_hist + (size_t)RP_NB * plan.num_parts, sizeof(u32), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (u32 d = 0; d < nb; ++d) out[d] = h[d];
    out[nb] = h[RP_NB];
    return VB_OK;
}

static Digit make_bucket_digit(const vb_shuf *s, int mode, u32 shift, u32 mask)
{
    Digit dg{};
    dg.mode = mode;
    dg.shift = shift;
    dg.mask = mask;
    dg.tx = TX_NONE;
    dg.key_width = s->key_width;
    dg.fm = make_fastmod(s->n_reduce);
    dg.fm_world = make_fastmod(s->world);
    return dg;
}

__global__ void bucket_hist_kernel(const u64 *__restrict__ keys, u64 n, Digit dg, u32 *__restrict__ cnt)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&cnt[get_partition(keys[i], dg.key_width, dg.fm)], 1u);
}

// Unordered multisplit of a combined table's occupied slots (reduce ops only; <= 256 bins): see kernels.cuh.
static int multisplit_table_unordered(vb_shuf *s, const Table &t, int mode, u32 nbins, u64 *out_keys, u64 *out_vals, std::vector<u64> &bin_off)
{
    vb_ctx *c = s->ctx;
    bin_off.assign((size_t)nbins + 1, 0);
    const u64 cap = 1ull << t.log_cap;
    DevBuf cc(c);
    TRY(cc.alloc(2 * TS_MAX_BINS * 4));
    CU(cudaMemsetAsync(cc.p, 0, 2 * TS_MAX_BINS * 4, c->stream));
    u32 *counts = cc.as<u32>(), *cursors = cc.as<u32>() + TS_MAX_BINS;
    Digit dg = make_bucket_digit(s, mode, 0, 0xFFFFFFFFu);
    const unsigned grid = (unsigned)std::min<u64>((cap + TS_TILE) / TS_TILE, (u64)c->sm_count * 4);
    {
        KLaunch kl(s, K_RP_HIST, cap + 1);
        if (mode == DG_DEST) table_bin_count_kernel<DG_DEST><<<grid, TS_THREADS, 0, c->stream>>>(t.keys, cap, dg, counts);
        else table_bin_count_kernel<DG_BUCKET><<<grid, TS_THREADS, 0, c->stream>>>(t.keys, cap, dg, counts);
        TRY(kl.done("table_bin_count_kernel"));
    }
    {
        KLaunch kl(s, K_RP_SCATTER, cap + 1);
        if (mode == DG_DEST) table_bin_scatter_kernel<DG_DEST><<<grid, TS_THREADS, 0, c->stream>>>(t.keys, t.accs, cap, dg, counts, cursors, out_keys, out_vals);
        else table_bin_scatter_kernel<DG_BUCKET><<<grid, TS_THREADS, 0, c->stream>>>(t.keys, t.accs, cap, dg, counts, cursors, out_keys, out_vals);
        TRY(kl.done("table_bin_scatter_kernel"));
    }
    u32 *h = (u32 *)c->h_scratch;
    CU(cudaMemcpyAsync(h, counts, TS_MAX_BINS * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    u64 run = 0;
    for (u32 d = 0; d < nbins; ++d) { bin_off[d] = run; run += h[d]; }
    bin_off[nbins] = run;
    return VB_OK;
}

// Stable multisplit of `n` loader rows by reduce partition (DG_BUCKET, nbins = n_reduce) or by
// owning rank (DG_DEST, nbins = world).  Invalid rows (empty table slots) are dropped.
// out_keys/out_vals must hold `max_valid` rows.  bin_off[nbins+1] (host) gets the offsets.
static int multisplit(vb_shuf *s, const Loader &ld, u64 n, int mode, u32 nbins, u64 max_valid, u64 *out_keys, u64 *out_vals,
                      std::vector<u64> &bin_off)
{
    vb_ctx *c = s->ctx;
    bin_off.assign((size_t)nbins + 1, 0);
    if (n == 0) return VB_OK;
    PassPlan plan = plan_pass<u64, true>(c, n);
    DevBuf hist(c);
    TRY(hist.alloc(plan.hist_bytes()));
    if (nbins <= RP_NB) {
        Digit dg = make_bucket_digit(s, mode, 0, 0xFFFFFFFFu);
        TRY((radix_pass<u64, true>(s, ld, dg, n, out_keys, out_vals, hist.as<u32>(), plan)));
        TRY(fetch_offsets(c, hist.as<u32>(), plan, nbins, bin_off.data()));
        return VB_OK;
    }
    if (mode != DG_BUCKET || nbins > 65536) return set_err(VB_ERR_UNSUPPORTED, "more than 65536 reduce partitions / 256 ranks");
    // two LSD passes over the 16-bit bucket id
    DevBuf tk(c), tv(c);
    TRY(tk.alloc(max_valid * 8));
    TRY(tv.alloc(max_valid * 8));
    Digit d0 = make_bucket_digit(s, DG_BUCKET, 0, 0xFF);
    TRY((radix_pass<u64, true>(s, ld, d0, n, tk.as<u64>(), tv.as<u64>(), hist.as<u32>(), plan)));
    std::vector<u64> tmp(RP_NB + 1);
    TRY(fetch_offsets(c, hist.as<u32>(), plan, RP_NB, tmp.data()));
    const u64 nv = tmp[RP_NB];
    if (nv == 0) return VB_OK;
    PassPlan plan2 = plan_pass<u64, true>(c, nv);
    DevBuf hist2(c);
    TRY(hist2.alloc(plan2.hist_bytes()));
    Loader l2{LD_SOA64, tk.p, tv.p, 0};
    Digit d1 = make_bucket_digit(s, DG_BUCKET, 8, 0xFF);
    TRY((radix_pass<u64, true>(s, l2, d1, nv, out_keys, out_vals, hist2.as<u32>(), plan2)));
    DevBuf cnt(c);
    TRY(cnt.alloc((size_t)nbins * 4));
    CU(cudaMemsetAsync(cnt.p, 0, (size_t)nbins * 4, c->stream));
    {
        KLaunch kl(s, K_MISC);
        bucket_hist_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, c->stream>>>(out_keys, nv, d0, cnt.as<u32>());
        TRY(kl.done("bucket_hist_kernel"));
    }
    std::vector<u32> hc(nbins);
    CU(cudaMemcpyAsync(hc.data(), cnt.p, (size_t)nbins * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    u64 run = 0;
    for (u32 b = 0; b < nbins; ++b) { bin_off[b] = run; run += hc[b]; }
    bin_off[nbins] = run;
    return VB_OK;
}

// LSD radix sort of (u32 id, u64 val) pairs over `bits` low bits.  ids_a is overwritten.
// The first pass reads values through `first` (ids come from ids_a).  Results: *out_ids, *out_vals
// (owned by the caller afterwards).
static int sort_id_pairs(vb_shuf *s, u32 *ids_a, const Loader &first, u64 n, u32 bits, u32 **out_ids, u64 **out_vals, const u32 *xlat = nullptr,
                         u64 *csr = nullptr, bool *csr_done = nullptr)
{
    vb_ctx *c = s->ctx;
    const u32 passes = std::max<u32>(1, (bits + 7) / 8);
    if (xlat) {                               // slot ids -> dense ids, in place
        KLaunch kl(s, K_MISC);
        u64 blocks = std::min<u64>((n + 255) / 256, (u64)c->sm_count * 8);
        translate_ids_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(ids_a, n, xlat);
        TRY(kl.done("translate_ids_kernel"));
    }
    PassPlan plan = plan_pass<u32, true>(c, n);
    DevBuf hist(c), ids_b(c), vals_a(c), vals_b(c);
    TRY(hist.alloc(plan.hist_bytes()));
    TRY(ids_b.alloc(n * 4));
    TRY(vals_b.alloc(n * 8));
    if (passes >= 2) TRY(vals_a.alloc(n * 8));
    u32 *src_ids = ids_a, *dst_ids = ids_b.as<u32>();
    u64 *src_vals = nullptr, *dst_vals = vals_b.as<u64>();
    for (u32 p = 0; p < passes; ++p) {
        Loader ld = first;
        if (p == 0) ld.keys = src_ids;
        else ld = Loader{LD_KEY32_VAL_SOA, src_ids, src_vals, 0};
        Digit dg{};
        dg.mode = DG_BITS;
        dg.shift = 8 * p;
        dg.mask = 0xFF;
        dg.tx = TX_NONE;
        const bool last = (p + 1 == passes);
        TRY((radix_pass<u32, true>(s, ld, dg, n, dst_ids, dst_vals, hist.as<u32>(), plan, last ? csr : nullptr, last ? csr_done : nullptr)));
        std::swap(src_ids, dst_ids);
        u64 *nv = (src_vals == nullptr) ? vals_a.as<u64>() : src_vals;
        src_vals = dst_vals;
        dst_vals = nv;
    }
    // results are in src_ids / src_vals
    *out_ids = src_ids;
    *out_vals = src_vals;
    if (src_ids == ids_b.as<u32>()) ids_b.release();          // ids_a stays with the caller either way
    if (src_vals == vals_b.as<u64>()) vals_b.release(); else vals_a.release();
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// shuffle lifecycle
// ---------------------------------------------------------------------------------------------
static std::atomic<u64> next_uid{1};   // vb_shuf::uid of every shuffle, the internal ones of a filtered join included

extern "C" int32_t vb_shuffle_create(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t kdt,
                                     int32_t vdt, int32_t agg, int32_t part, vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create: NULL argument");
    *out = nullptr;
    if (n_reduce < 1) return set_err(VB_ERR_INVALID, "vb_shuffle_create: n_reduce must be >= 1");
    if (kdt < VB_U64 || kdt > VB_F64 || vdt < VB_U64 || vdt > VB_BYTES) return set_err(VB_ERR_INVALID, "bad dtype");
    if (agg < VB_AGG_GROUP || agg > VB_AGG_SORT) return set_err(VB_ERR_INVALID, "bad agg %d", agg);
    if (vdt == VB_BYTES && !is_group_op(agg) && agg != VB_AGG_SORT)
        return set_err(VB_ERR_UNSUPPORTED, "byte-string values go with GROUP, COGROUP and SORT only (agg %d computes on values)", agg);
    if (agg != VB_AGG_SORT && kdt == VB_F64) return set_err(VB_ERR_UNSUPPORTED, "f64 keys are not hashable (Rust f64 is not Hash)");
    if ((agg == VB_AGG_SORT) != (part == VB_PART_RANGE)) return set_err(VB_ERR_INVALID, "VB_PART_RANGE goes with VB_AGG_SORT only");
    if (n_reduce > 65536) return set_err(VB_ERR_UNSUPPORTED, "more than 65536 reduce partitions");
    vb_shuf *s = new vb_shuf();
    s->uid = next_uid.fetch_add(1);
    s->ctx = c;
    s->id = shuffle_id;
    s->n_map = n_map;
    s->n_reduce = n_reduce;
    s->kdt = kdt;
    s->vdt = vdt;
    s->agg = agg;
    s->part = part;
    s->maps.resize(n_map);
    if (vdt == VB_BYTES) s->bvals.assign(n_map, ByteSrc{nullptr, nullptr, 0});
    *out = s;
    return VB_OK;
}

// Accumulators of a multi-aggregate shuffle: aggregate a owns accumulator a; a MEAN's is its SUM, and every MEAN
// divides by the spec's first COUNT accumulator, or by one appended after the aggregates when the spec has none.
// The specs of the map-side combine, the table merge and the import merge, and the output columns: filled in by
// multi_spec, shared by the integer-key and the string-key combine.
struct MultiSpec {
    u32 n_cols = 0;
    AccSpec map{}, merge{}, imp{};
    OutSpec outs{};
    int out_dt[VB_MAX_AGGS] = {};
};

static int multi_spec(uint32_t n_val_cols, const int32_t *val_dtypes, uint32_t n_aggs, const vb_agg_col *aggs, MultiSpec *ms)
{
    if (n_val_cols < 1 || n_val_cols > VB_MAX_VAL_COLS) return set_err(VB_ERR_INVALID, "%u value columns (1..%d)", n_val_cols, VB_MAX_VAL_COLS);
    if (n_aggs < 1 || n_aggs > VB_MAX_AGGS) return set_err(VB_ERR_INVALID, "%u aggregates (1..%d)", n_aggs, VB_MAX_AGGS);
    for (u32 i = 0; i < n_val_cols; ++i)
        if (val_dtypes[i] < VB_U64 || val_dtypes[i] > VB_F64) return set_err(VB_ERR_INVALID, "bad dtype %d of value column %u", val_dtypes[i], i);
    int count_acc = -1;
    bool any_mean = false;
    for (u32 a = 0; a < n_aggs; ++a) {
        const int op = aggs[a].agg;
        if (op != VB_AGG_SUM && op != VB_AGG_MIN && op != VB_AGG_MAX && op != VB_AGG_COUNT && op != VB_AGG_MEAN)
            return set_err(VB_ERR_INVALID, "aggregate %u: op %d is not SUM / MIN / MAX / COUNT / MEAN", a, op);
        if (op != VB_AGG_COUNT && (aggs[a].src < 0 || (u32)aggs[a].src >= n_val_cols))
            return set_err(VB_ERR_INVALID, "aggregate %u reads column %d of %u", a, aggs[a].src, n_val_cols);
        if (op == VB_AGG_COUNT && count_acc < 0) count_acc = (int)a;
        any_mean |= op == VB_AGG_MEAN;
    }
    const u32 n_acc = n_aggs + ((any_mean && count_acc < 0) ? 1 : 0);
    if (n_acc > VB_MAX_AGGS) return set_err(VB_ERR_INVALID, "%u aggregates plus the COUNT a MEAN needs exceed %d", n_aggs, VB_MAX_AGGS);
    if (count_acc < 0) count_acc = (int)n_aggs;
    ms->n_cols = n_val_cols;
    AccSpec &mp = ms->map, &mg = ms->merge;
    OutSpec &os = ms->outs;
    mp.n = mg.n = ms->imp.n = n_acc;
    os.n = n_aggs;
    for (u32 a = 0; a < n_acc; ++a) {
        const int op = a < n_aggs ? aggs[a].agg : VB_AGG_COUNT;
        const int src = op == VB_AGG_COUNT ? 0 : aggs[a].src;
        const int dt = val_dtypes[src];
        int opk = OPK_COUNT, tx = TX_NONE;
        if (op == VB_AGG_SUM || op == VB_AGG_MEAN) opk = dt == VB_F64 ? OPK_ADD_F64 : OPK_ADD_U64;
        else if (op == VB_AGG_MIN || op == VB_AGG_MAX) {
            opk = op == VB_AGG_MIN ? OPK_MIN_U64 : OPK_MAX_U64;
            tx = dt == VB_I64 ? TX_I64 : dt == VB_F64 ? TX_F64 : TX_NONE;
        }
        spec_set(mp.op, a, opk); spec_set(mp.tx, a, tx); spec_set(mp.src, a, src);
        spec_set(mg.op, a, merge_op(opk)); spec_set(mg.src, a, a);
        spec_set(ms->imp.op, a, merge_op(opk)); spec_set(ms->imp.tx, a, tx);
        if (a >= n_aggs) continue;
        ms->out_dt[a] = op == VB_AGG_COUNT ? VB_U64 : op == VB_AGG_MEAN ? VB_F64 : dt;
        os.acc[a] = (unsigned char)a;
        os.cnt[a] = (unsigned char)count_acc;
        os.tx[a] = (unsigned char)tx;
        os.kind[a] = op != VB_AGG_MEAN ? MO_COPY : dt == VB_U64 ? MO_MEAN_U64 : dt == VB_I64 ? MO_MEAN_I64 : MO_MEAN_F64;
    }
    return VB_OK;
}

// The accumulator spec only: s->multi (the _multi ABI) is set by the callers that create such a shuffle.
static void set_spec(vb_shuf *s, const MultiSpec &ms)
{
    s->n_cols = ms.n_cols;
    s->acc_map = ms.map;
    s->acc_merge = ms.merge;
    s->acc_imp = ms.imp;
    s->outs = ms.outs;
    std::copy(ms.out_dt, ms.out_dt + VB_MAX_AGGS, s->out_dt);
}

extern "C" int32_t vb_shuffle_create_multi(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t kdt,
                                           uint32_t n_val_cols, const int32_t *val_dtypes, uint32_t n_aggs, const vb_agg_col *aggs,
                                           vb_shuf **out)
{
    if (!c || !out || !val_dtypes || !aggs) return set_err(VB_ERR_INVALID, "vb_shuffle_create_multi: NULL argument");
    *out = nullptr;
    MultiSpec ms;
    TRY(multi_spec(n_val_cols, val_dtypes, n_aggs, aggs, &ms));
    TRY(vb_shuffle_create(c, shuffle_id, n_map, n_reduce, kdt, VB_U64, VB_AGG_SUM, VB_PART_HASH_METRO64, out));
    set_spec(*out, ms);
    (*out)->multi = true;
    return VB_OK;
}

static_assert(MA_MAX_COLS == VB_MAX_VAL_COLS && MA_MAX_ACCS == VB_MAX_AGGS, "kernel limits = ABI limits");

static int reject_multi(const vb_shuf *s, const char *what)
{
    return set_err(VB_ERR_UNSUPPORTED, "shuffle %llu has several aggregates per key: %s is not supported for it yet", (unsigned long long)s->id, what);
}

// string-key shuffles: calls that do not apply (VB_ERR_INVALID) and calls not supported for them yet (VB_ERR_UNSUPPORTED)
static int invalid_str(const vb_shuf *s, const char *what)
{
    return set_err(VB_ERR_INVALID, "shuffle %llu has string keys: %s does not apply to it", (unsigned long long)s->id, what);
}
static int reject_str(const vb_shuf *s, const char *what)
{
    return set_err(VB_ERR_UNSUPPORTED, "shuffle %llu has string keys: %s is not supported for it yet", (unsigned long long)s->id, what);
}
// byte-string values stay on one device for now: every call that moves rows between ranks or serialises them
static int reject_bytes(const vb_shuf *s, const char *what)
{
    return set_err(VB_ERR_UNSUPPORTED, "shuffle %llu has byte-string values: %s is not supported for them yet", (unsigned long long)s->id, what);
}

extern "C" int32_t vb_shuffle_set_key_width(vb_shuf *s, uint32_t bytes)
{
    if (!s || (bytes != 4 && bytes != 8)) return set_err(VB_ERR_INVALID, "key width must be 4 or 8");
    if (s->rep) return reject_rep(s, "vb_shuffle_set_key_width (positions hash as 8 bytes)");
    if (s->str) return invalid_str(s, "vb_shuffle_set_key_width");
    s->key_width = bytes;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_set_hint(vb_shuf *s, uint64_t d)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    s->hint = d;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_set_dist(vb_shuf *s, uint32_t rank, uint32_t world)
{
    if (!s || world < 1 || rank >= world || world > 256) return set_err(VB_ERR_INVALID, "bad rank/world");
    if (s->rep) return reject_rep(s, "vb_shuffle_set_dist");
    if (s->multi && (world > 1 || s->world > 1)) return reject_multi(s, "multi-rank use through vb_shuffle_set_dist (vb_shuffle_create_multi_dist is)");
    if (s->vdt == VB_BYTES && world > 1) return set_err(VB_ERR_UNSUPPORTED, "shuffle %llu has byte-string values: they do not cross ranks yet", (unsigned long long)s->id);
    if (s->str && (world > 1 || s->world > 1)) return reject_str(s, "multi-rank use through vb_shuffle_set_dist (vb_shuffle_create_str_dist is)");
    s->rank = rank;
    s->world = world;
    return VB_OK;
}

static void free_map(vb_shuf *s, MapOut &m)
{
    vb_ctx *c = s->ctx;
    if (m.table) dev_free(c, m.table);
    if (m.owned) { dev_free(c, m.rows); dev_free(c, m.keys); dev_free(c, m.vals); }
    else if (m.vals_owned) dev_free(c, m.vals);
    m = MapOut();
}

static const AccSpec *map_spec(const vb_shuf *s) { return s->multi ? &s->acc_map : nullptr; }

// cols: the value columns of a multi-aggregate shuffle (keys + cols, vals unused)
// own_vals: a device value column the shuffle takes over (byte-string values: the references), read in place of vals
static int shuffle_map(vb_shuf *s, u32 map_id, const u64 *rows, const u64 *keys, const u64 *vals, u64 n, int loc, bool combined = false,
                       const u64 *const *cols = nullptr, DevBuf *own_vals = nullptr)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (s->rep) return reject_rep(s, "vb_shuffle_map_aos / vb_shuffle_map_soa");
    if (s->str) return invalid_str(s, "an integer-key map call");
    if (map_id >= s->n_map) return set_err(VB_ERR_INVALID, "map_id %u >= n_map %u", map_id, s->n_map);
    if (loc < VB_HOST || loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc %d", loc);
    if (n && !rows && !keys) return set_err(VB_ERR_INVALID, "NULL input with n_rows > 0");
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "map partition of %llu rows", (unsigned long long)n);
    vb_ctx *c = s->ctx;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->exported || s->freed) return set_err(VB_ERR_STATE, "shuffle %llu: map after seal/export", (unsigned long long)s->id);
    }
    std::unique_lock<std::mutex> lk(c->mu);
    struct TlGuard { TlGuard(std::unique_lock<std::mutex> *l) { tl_ctx_lock = l; } ~TlGuard() { tl_ctx_lock = nullptr; } } tlg(&lk);
    CU(cudaSetDevice(c->device));
    KLaunch call(s, -1);
    MapOut &m = s->maps[map_id];
    if (m.present) {                                                // stage resubmission: overwrite
        if (m.in_shared) s->sh_dirty = true;                        // its rows are already in the shared table: rebuild at seal
        s->st.rows_in -= m.n_rows;
        free_map(s, m);
    }
    m.n_rows = n;
    const AccSpec *ms = map_spec(s);
    if (is_reduce_op(s->agg) && loc == VB_DEVICE_BORROWED && !combined) {
        if (!ms && !rows && !vals && s->agg != VB_AGG_COUNT && n) return set_err(VB_ERR_INVALID, "values required for this aggregator");
        std::vector<AggInput> in(1);
        in[0] = AggInput{rows ? IN_AOS : IN_SOA, rows ? rows : keys, vals, n, VB_DEVICE};
        if (ms) for (u32 i = 0; i < s->n_cols; ++i) in[0].cols[i] = m.cols[i] = cols[i];
        if (!s->sh_tab && !s->sh_dirty && n) {       // first borrowed map task: size and create the shared table
            u64 hint = s->hint;
            bool estimated = false;
            const u64 total_guess = n * std::max<u64>(1, s->n_map / std::max<u32>(1, s->world));
            if (!hint && n > (1ull << 20)) { TRY(estimate_distinct(s, in, total_guess, &hint)); estimated = true; }
            const u32 max_log = std::min<u32>(MAX_LOG_CAP, std::max<u32>(4, ceil_log2_u64(2 * std::max<u64>(total_guess, 1))));
            s->sh_log_cap = choose_log_cap(total_guess, hint, estimated, max_log, c->l2_bytes, ms ? 8 * (1 + ms->n) : 16);
            DevBuf tab(c), ctl(c);
            TRY(tab.alloc(ms ? table_bytes_multi(s->sh_log_cap, ms->n) : table_bytes(s->sh_log_cap)));
            TRY(ctl.alloc(sizeof(TableCtl)));
            CU(cudaMemsetAsync(ctl.p, 0, sizeof(TableCtl), c->stream));
            TRY(init_table(s, tab.p, s->sh_log_cap, map_opk(s), ms));
            // the total is a guess from the first map task, so even a table at max_log keeps the insert limit (and the
            // HA_MAX_PROBE chain limit): a wrong guess or a long chain rebuilds it at seal through build_table
            s->sh_max_inserts = ((1ull << s->sh_log_cap) / 10) * 6;
            s->sh_tab = tab.release();
            s->sh_ctl = (TableCtl *)ctl.release();
            s->st.table_slots = std::max<u64>(s->st.table_slots, 1ull << s->sh_log_cap);
        }
        if (s->sh_tab && !s->sh_dirty && n) {         // asynchronous: checked at seal
            if (ms)
                TRY(launch_hash_agg_multi(s, K_HASH_AGG, *ms, in[0], keys, cols, n, s->sh_tab, s->sh_log_cap, s->sh_ctl, s->sh_max_inserts));
            else if (want_partition(in[0].in, map_opk(s), s->sh_log_cap, n))
                TRY(launch_hash_agg_partitioned(s, K_HASH_AGG, in[0].in, map_opk(s), val_tx(s), in[0].a, in[0].b, n, s->sh_tab, s->sh_log_cap,
                                                s->sh_ctl, s->sh_max_inserts));
            else
                TRY(launch_hash_agg(s, K_HASH_AGG, in[0].in, map_opk(s), val_tx(s), in[0].a, in[0].b, n, s->sh_tab, s->sh_log_cap, s->sh_ctl,
                                    s->sh_max_inserts, nullptr));
        }
        m.rows = rows; m.keys = keys; m.vals = vals; m.owned = false; m.in_shared = true;
    } else if (is_reduce_op(s->agg)) {
        if (!ms && !rows && !vals && s->agg != VB_AGG_COUNT && n) return set_err(VB_ERR_INVALID, "values required for this aggregator");
        std::vector<AggInput> in(1);
        in[0] = AggInput{rows ? IN_AOS : IN_SOA, rows ? rows : keys, vals, n, loc == VB_HOST ? VB_HOST : VB_DEVICE};
        if (ms) for (u32 i = 0; i < s->n_cols; ++i) in[0].cols[i] = cols[i];
        const u64 hint = s->hint ? s->hint : (s->learned_distinct ? s->learned_distinct + s->learned_distinct / 4 : 0);
        // a map-side-combined bucket carries combiners, merged with merge_combiners (partial counts are summed)
        TRY(build_table(s, K_HASH_AGG, in, combined ? merge_opk(s) : map_opk(s), val_tx(s), hint, &m.table, &m.log_cap, &m.n_inserted, nullptr,
                        ms));
        s->learned_distinct = std::max<u64>(m.n_inserted, 1);
    } else if (n) {
        if (loc == VB_DEVICE_BORROWED) {
            m.rows = rows; m.keys = keys; m.vals = vals; m.owned = false;
        } else {
            const cudaMemcpyKind kind = loc == VB_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
            DevBuf a(c), b(c);
            // the copies run on the copy stream (ordered after the pool's hand-out), so a concurrent map task's kernels
            // on c->stream are not held up by this task's PCIe transfer
            if (rows) TRY(a.alloc(n * 16));
            else { TRY(a.alloc(n * 8)); if (vals) TRY(b.alloc(n * 8)); }
            cudaEvent_t ev_in, ev_done;
            CU(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
            CU(cudaEventCreateWithFlags(&ev_done, cudaEventDisableTiming));
            CU(cudaEventRecord(ev_in, c->stream));
            CU(cudaStreamWaitEvent(c->copy_stream, ev_in, 0));
            if (rows) {
                CU(cudaMemcpyAsync(a.p, rows, n * 16, kind, c->copy_stream));
                if (loc == VB_HOST) s->st.h2d_bytes += n * 16;
            } else {
                CU(cudaMemcpyAsync(a.p, keys, n * 8, kind, c->copy_stream));
                if (loc == VB_HOST) s->st.h2d_bytes += n * 8;
                if (vals) {
                    CU(cudaMemcpyAsync(b.p, vals, n * 8, kind, c->copy_stream));
                    if (loc == VB_HOST) s->st.h2d_bytes += n * 8;
                }
            }
            CU(cudaEventRecord(ev_done, c->copy_stream));
            CU(cudaStreamWaitEvent(c->stream, ev_done, 0));      // later work on c->stream sees the rows
            lk.unlock();                                         // the caller may reuse its buffer on return: wait, unlocked
            cudaError_t ce = cudaEventSynchronize(ev_done);
            lk.lock();
            cudaSetDevice(c->device);
            cudaEventDestroy(ev_in); cudaEventDestroy(ev_done);
            if (ce != cudaSuccess) { cudaGetLastError(); return set_err(VB_ERR_CUDA, "input copy: %s", cudaGetErrorString(ce)); }
            if (rows) m.rows = (const u64 *)a.release();
            else { m.keys = (const u64 *)a.release(); m.vals = vals ? (const u64 *)b.release() : nullptr; }
            m.owned = true;
        }
        if (own_vals) { m.vals = (const u64 *)own_vals->release(); m.vals_owned = !m.owned; }
    }
    m.present = true;
    s->st.rows_in += n;
    TRY(call.done("map"));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_map_aos(vb_shuf *s, uint32_t map_id, const void *rows, uint64_t n, int32_t loc)
{
    if (s && s->multi && !s->str) return reject_multi(s, "AoS rows");
    if (s && s->vdt == VB_BYTES) return set_err(VB_ERR_INVALID, "shuffle %llu has byte-string values: map it with vb_shuffle_map_bytes", (unsigned long long)s->id);
    // every AoS loader reads a row as one 16-byte vector load; host rows are copied into aligned buffers first
    if (n && loc != VB_HOST && ((uintptr_t)rows & 15u))
        return set_err(VB_ERR_INVALID, "device AoS rows at %p: 16-byte rows must start on a 16-byte boundary", rows);
    return shuffle_map(s, map_id, (const u64 *)rows, nullptr, nullptr, n, loc);
}
extern "C" int32_t vb_shuffle_map_soa(vb_shuf *s, uint32_t map_id, const void *keys, const void *vals, uint64_t n, int32_t loc)
{
    if (s && s->multi) return set_err(VB_ERR_INVALID, "shuffle %llu has several aggregates per key: map it with vb_shuffle_map_cols", (unsigned long long)s->id);
    if (s && s->vdt == VB_BYTES) return set_err(VB_ERR_INVALID, "shuffle %llu has byte-string values: map it with vb_shuffle_map_bytes", (unsigned long long)s->id);
    return shuffle_map(s, map_id, nullptr, (const u64 *)keys, (const u64 *)vals, n, loc);
}
extern "C" int32_t vb_shuffle_map_cols(vb_shuf *s, uint32_t map_id, const void *keys, const void *const *vals, uint64_t n, int32_t loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->multi) return set_err(VB_ERR_INVALID, "vb_shuffle_map_cols needs a shuffle from vb_shuffle_create_multi");
    const u64 *cols[MA_MAX_COLS] = {};
    for (u32 i = 0; vals && i < s->n_cols; ++i) cols[i] = (const u64 *)vals[i];
    for (u32 a = 0; a < s->acc_map.n; ++a)
        if (n && spec_at(s->acc_map.op, a) != OPK_COUNT && !cols[spec_at(s->acc_map.src, a)])
            return set_err(VB_ERR_INVALID, "value column %d is read by an aggregate but NULL", spec_at(s->acc_map.src, a));
    if (n && !keys) return set_err(VB_ERR_INVALID, "NULL keys with n_rows > 0");
    return shuffle_map(s, map_id, nullptr, (const u64 *)keys, nullptr, n, loc, false, cols);
}

// ---------------------------------------------------------------------------------------------
// reduce side
// ---------------------------------------------------------------------------------------------
// Concatenate the rows of all present map partitions in map-id order.  Zero-copy when they are
// one AoS run (adjacent in memory) or a single partition; otherwise SoA copies owned by s.
struct Gathered {
    const u64 *rows = nullptr, *keys = nullptr, *vals = nullptr;
    u64 n = 0;
};

static int gather_maps(vb_shuf *s, Gathered *g)
{
    vb_ctx *c = s->ctx;
    u64 n = 0;
    std::vector<MapOut *> segs;
    for (auto &m : s->maps)
        if (m.present && m.n_rows) { segs.push_back(&m); n += m.n_rows; }
    g->n = n;
    if (n == 0) return VB_OK;
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "shuffle of %llu rows on one device", (unsigned long long)n);
    bool contiguous = true;
    for (size_t i = 0; i < segs.size(); ++i) {
        if (!segs[i]->rows) { contiguous = false; break; }
        if (i && segs[i - 1]->rows + 2 * segs[i - 1]->n_rows != segs[i]->rows) { contiguous = false; break; }
    }
    if (contiguous) { g->rows = segs[0]->rows; return VB_OK; }
    if (segs.size() == 1) { g->keys = segs[0]->keys; g->vals = segs[0]->vals; return VB_OK; }
    bool any_vals = false;
    for (auto *m : segs) any_vals |= (m->rows != nullptr) || (m->vals != nullptr);
    DevBuf k(c), v(c);
    TRY(k.alloc(n * 8));
    if (any_vals) TRY(v.alloc(n * 8));
    u64 off = 0;
    for (auto *m : segs) {
        if (m->rows) {
            KLaunch kl(s, K_MISC);
            u64 blocks = std::min<u64>((m->n_rows + 255) / 256, (u64)c->sm_count * 8);
            aos_to_soa_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(m->rows, m->n_rows, k.as<u64>() + off, v.as<u64>() + off);
            TRY(kl.done("aos_to_soa_kernel"));
        } else {
            CU(cudaMemcpyAsync(k.as<u64>() + off, m->keys, m->n_rows * 8, cudaMemcpyDeviceToDevice, c->stream));
            if (any_vals) {
                if (m->vals) CU(cudaMemcpyAsync(v.as<u64>() + off, m->vals, m->n_rows * 8, cudaMemcpyDeviceToDevice, c->stream));
                else CU(cudaMemsetAsync(v.as<u64>() + off, 0, m->n_rows * 8, c->stream));
            }
        }
        off += m->n_rows;
    }
    s->gath_keys = (u64 *)k.release();
    s->gath_vals = any_vals ? (u64 *)v.release() : nullptr;
    g->keys = s->gath_keys;
    g->vals = s->gath_vals;
    for (auto &m : s->maps) if (m.present && m.owned) { dev_free(c, m.rows); dev_free(c, m.keys); dev_free(c, m.vals); m.rows = m.keys = m.vals = nullptr; m.owned = false; }
    return VB_OK;
}

__global__ void gather_u64_kernel(const u64 *__restrict__ src, const u64 *__restrict__ idx, u32 n, u64 *__restrict__ out)
{
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = src[idx[i]];
}

__global__ void rebase_kernel(const u64 *__restrict__ src, u64 n, u64 base, u64 *__restrict__ out)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = src[i] - base;
}

static int sort_segments(vb_shuf *s, const u64 *offs, u64 D, u64 *vals, u64 n);

// group_by_key / cogroup reduce side over n rows (AoS `rows`, or SoA keys/vals).
static int seal_group(vb_shuf *s, const Gathered &g)
{
    vb_ctx *c = s->ctx;
    const u32 R = s->n_reduce;
    s->bucket_off.assign((size_t)R + 1, 0);
    s->val_off.assign((size_t)R + 1, 0);
    const u64 n = g.n;
    if (n == 0) return VB_OK;
    // 1. dictionary: key → slot, slot per row
    DevBuf ids(c);
    TRY(ids.alloc(n * 4));
    std::vector<AggInput> in(1);
    in[0] = AggInput{g.rows ? IN_AOS : IN_SOA, g.rows ? g.rows : g.keys, nullptr, n, VB_DEVICE};
    u64 n_ins = 0;
    TRY(build_table(s, K_DICT, in, OPK_DICT, TX_NONE, s->hint, &s->dict, &s->dict_log_cap, &n_ins, ids.as<u32>()));
    const u64 cap = 1ull << s->dict_log_cap;
    // 2. distinct keys grouped by reduce partition (stable by slot)
    const u64 max_d = n_ins + 1;
    DevBuf ckeys(c), cslot(c);
    TRY(ckeys.alloc(max_d * 8));
    TRY(cslot.alloc(max_d * 8));
    const Table dt = table_at(s->dict, s->dict_log_cap);
    Loader lt{LD_TABLE_KI, dt.keys, nullptr, cap};
    TRY(multisplit(s, lt, cap + 1, DG_BUCKET, R, max_d, ckeys.as<u64>(), cslot.as<u64>(), s->bucket_off));
    const u64 D = s->bucket_off[R];
    // 3. slot → dense id (bucket-major)
    DevBuf dense(c);
    TRY(dense.alloc((cap + 1) * 4));
    {
        KLaunch kl(s, K_MISC);
        scatter_dense_kernel<<<(unsigned)((D + 255) / 256), 256, 0, c->stream>>>(cslot.as<u64>(), (u32)D, dense.as<u32>());
        TRY(kl.done("scatter_dense_kernel"));
    }
    cslot.reset();
    // 4. ids[i] = dense_of_slot[slot_of_row[i]]: first thing sort_id_pairs does (translate_ids_kernel)
    // 5. stable LSD sort of (id, value) — the reduce partition is the high part of the dense id
    Loader first = g.rows ? Loader{LD_KEY32_VAL_AOS, nullptr, g.rows, 0} : Loader{LD_KEY32_VAL_SOA, nullptr, g.vals, 0};
    u32 *sorted_ids = nullptr;
    u64 *sorted_vals = nullptr;
    // 6. CSR offsets: recorded by the last sort pass itself when it runs as rp_gsweep_kernel<CSR> (offsets pre-set to all ones,
    //    offsets[D] = n), otherwise from the sorted ids
    DevBuf offs(c);
    TRY(offs.alloc((D + 1) * 8));
    CU(cudaMemsetAsync(offs.p, 0xFF, (D + 1) * 8, c->stream));
    bool csr_done = false;
    TRY(sort_id_pairs(s, ids.as<u32>(), first, n, ceil_log2_u64(std::max<u64>(D, 2)), &sorted_ids, &sorted_vals, dense.as<u32>(), offs.as<u64>(), &csr_done));
    DevBuf sid_guard(c);
    if (sorted_ids != ids.as<u32>()) sid_guard.p = sorted_ids;
    if (csr_done) {
        const u64 total = n;
        CU(cudaMemcpyAsync(offs.as<u64>() + D, &total, 8, cudaMemcpyHostToDevice, c->stream));   // pageable 8-byte source: copied before the call returns
    } else {
        KLaunch kl(s, K_MISC);
        u64 blocks = std::min<u64>((n + 255) / 256, (u64)c->sm_count * 8);
        csr_bounds_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(sorted_ids, n, offs.as<u64>(), D);
        TRY(kl.done("csr_bounds_kernel"));
    }
    DevBuf sv_guard(c);
    sv_guard.p = sorted_vals;
    // 7. each list ascending where the shuffle asks for it (vb_shuffle_set_value_order)
    TRY(sort_segments(s, offs.as<u64>(), D, sorted_vals, n));
    sv_guard.release();
    // 8. value offsets at the partition boundaries
    {
        DevBuf idx(c), out(c);
        TRY(idx.alloc(((size_t)R + 1) * 8));
        TRY(out.alloc(((size_t)R + 1) * 8));
        CU(cudaMemcpyAsync(idx.p, s->bucket_off.data(), ((size_t)R + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        KLaunch kl(s, K_MISC);
        gather_u64_kernel<<<(R + 1 + 255) / 256, 256, 0, c->stream>>>(offs.as<u64>(), idx.as<u64>(), R + 1, out.as<u64>());
        TRY(kl.done("gather_u64_kernel"));
        CU(cudaMemcpyAsync(s->val_off.data(), out.p, ((size_t)R + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    s->n_keys = D;
    s->n_vals = n;
    s->res_keys = (u64 *)ckeys.release();
    s->res_offs = (u64 *)offs.release();
    s->res_vals = sorted_vals;
    s->dense_of_slot = (u32 *)dense.release();
    s->st.rows_out = n;
    return VB_OK;
}

// Merge the per-map combined tables of this process into one (ShuffledRdd::compute's
// merge_combiners loop, shuffled_rdd.rs:154-164, for the partitions held locally).
// Settle the shared table of the borrowed-input map tasks: wait for the queued kernels, and if the table
// overflowed or a map id was resubmitted, rebuild it from the (still borrowed) inputs with build_table's
// restart logic.
static int settle_shared_table(vb_shuf *s, u64 *n_ins)
{
    vb_ctx *c = s->ctx;
    *n_ins = 0;
    bool any = false;
    for (auto &m : s->maps) any |= (m.present && m.in_shared && m.n_rows);
    bool rebuild = s->sh_dirty;
    if (s->sh_tab) {
        TableCtl *h = (TableCtl *)c->h_scratch;
        CU(cudaMemcpyAsync(h, s->sh_ctl, sizeof(TableCtl), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        if (h->abort) { rebuild = true; s->st.table_restarts++; }
        *n_ins = h->n_inserted;
    }
    if (rebuild) {
        dev_free(c, s->sh_tab); dev_free(c, s->sh_ctl);
        s->sh_tab = nullptr; s->sh_ctl = nullptr;
        s->sh_dirty = false;
        if (any) {
            std::vector<AggInput> in;
            for (auto &m : s->maps)
                if (m.present && m.in_shared && m.n_rows) {
                    in.push_back(AggInput{m.rows ? IN_AOS : IN_SOA, m.rows ? m.rows : m.keys, m.vals, m.n_rows, VB_DEVICE});
                    std::copy(m.cols, m.cols + MA_MAX_COLS, in.back().cols);
                }
            TRY(build_table(s, K_HASH_AGG, in, map_opk(s), val_tx(s), std::max<u64>(s->hint, 2 * (*n_ins)), &s->sh_tab, &s->sh_log_cap, n_ins, nullptr,
                            map_spec(s)));
        }
    }
    return VB_OK;
}

static int merge_map_tables(vb_shuf *s, void **tab, u32 *log_cap, u64 *n_ins)
{
    u64 sh_ins = 0;
    TRY(settle_shared_table(s, &sh_ins));
    struct T { void *tab; u32 log_cap; u64 ins; };
    std::vector<T> ts;
    if (s->sh_tab) ts.push_back(T{s->sh_tab, s->sh_log_cap, sh_ins});
    for (auto &m : s->maps) if (m.present && m.table) ts.push_back(T{m.table, m.log_cap, m.n_inserted});
    auto disown = [&]() {
        s->sh_tab = nullptr;
        dev_free(s->ctx, s->sh_ctl); s->sh_ctl = nullptr;
        for (auto &m : s->maps) m.table = nullptr;
    };
    if (ts.empty()) { *tab = nullptr; *log_cap = 0; *n_ins = 0; return VB_OK; }
    if (ts.size() == 1) {
        *tab = ts[0].tab; *log_cap = ts[0].log_cap; *n_ins = ts[0].ins;
        disown();
        return VB_OK;
    }
    std::vector<AggInput> in;
    u64 max_ins = 0;
    for (auto &t : ts) {
        const Table mt = table_at(t.tab, t.log_cap);
        in.push_back(AggInput{IN_TABLE, mt.keys, mt.accs, (1ull << t.log_cap) + 1, VB_DEVICE, t.ins + 1});
        max_ins = std::max(max_ins, t.ins);
    }
    TRY(build_table(s, K_MERGE, in, merge_opk(s), TX_NONE, std::max<u64>(max_ins, s->hint), tab, log_cap, n_ins, nullptr,
                    s->multi ? &s->acc_merge : nullptr));
    for (auto &t : ts) dev_free(s->ctx, t.tab);
    disown();
    return VB_OK;
}

// Final (K, C) rows of a combined table, grouped by reduce partition.
static int finalize_reduce(vb_shuf *s, void *tab, u32 log_cap, u64 n_ins)
{
    vb_ctx *c = s->ctx;
    const u32 R = s->n_reduce;
    s->bucket_off.assign((size_t)R + 1, 0);
    s->val_off.assign((size_t)R + 1, 0);
    if (!tab) return VB_OK;
    const u64 cap = 1ull << log_cap;
    const u64 max_d = n_ins + 1;
    if (s->multi) {
        // keys and slot indices grouped by reduce partition, then one gather per output column
        DevBuf k(c), sl(c), out(c);
        TRY(k.alloc(max_d * 8));
        TRY(sl.alloc(max_d * 8));
        const Table ft = table_at(tab, log_cap);
        TRY(multisplit(s, Loader{LD_TABLE_KI, ft.keys, nullptr, cap}, cap + 1, DG_BUCKET, R, max_d, k.as<u64>(), sl.as<u64>(), s->bucket_off));
        const u64 D = s->bucket_off[R];
        if (D) {
            TRY(out.alloc(D * 8 * s->outs.n));
            KLaunch kl(s, K_MISC);
            const u64 blocks = std::min<u64>((D + 255) / 256, (u64)c->sm_count * 8);
            multi_finalize_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(ft.accs, acc_stride(log_cap), sl.as<u64>(), D, s->outs, out.as<u64>());
            TRY(kl.done("multi_finalize_kernel"));
        }
        s->n_keys = D;
        s->res_keys = (u64 *)k.release();
        s->res_cols = (u64 *)out.release();
        s->st.rows_out = D;
        return VB_OK;
    }
    DevBuf k(c), v(c);
    TRY(k.alloc(max_d * 8));
    TRY(v.alloc(max_d * 8));
    const Table ft = table_at(tab, log_cap);
    Loader lt{LD_TABLE_KV, ft.keys, ft.accs, cap};
    if (R <= (u32)TS_MAX_BINS) TRY(multisplit_table_unordered(s, ft, DG_BUCKET, R, k.as<u64>(), v.as<u64>(), s->bucket_off));
    else TRY(multisplit(s, lt, cap + 1, DG_BUCKET, R, max_d, k.as<u64>(), v.as<u64>(), s->bucket_off));
    const u64 D = s->bucket_off[R];
    const int tx = val_tx(s);
    if (tx != TX_NONE && D) {
        KLaunch kl(s, K_MISC);
        tx_inv_kernel<<<(unsigned)((D + 255) / 256), 256, 0, c->stream>>>(v.as<u64>(), D, tx);
        TRY(kl.done("tx_inv_kernel"));
    }
    s->n_keys = D;
    s->res_keys = (u64 *)k.release();
    s->res_comb = (u64 *)v.release();
    s->st.rows_out = D;
    return VB_OK;
}

// Stable LSD sort of n (u64 key, u64 value) rows by tx_fwd(key); the first pass reads them through `first`, whose keys
// are also at kscan, kstride words apart.  The rows end in *out_k / *out_v, which lie in ka or kb and va or vbuf (the
// passes alternate between them, starting with ka / va).
static int lsd_sort_u64(vb_shuf *s, const Loader &first, const u64 *kscan, u32 kstride, u64 n, int tx, bool has_val, DevBuf &ka, DevBuf &kb,
                        DevBuf &va, DevBuf &vbuf, u64 **out_k, u64 **out_v)
{
    vb_ctx *c = s->ctx;
    DevBuf hist(c);
    TRY(ka.alloc(n * 8));
    TRY(kb.alloc(n * 8));
    if (has_val) { TRY(va.alloc(n * 8)); TRY(vbuf.alloc(n * 8)); }
    u64 *src_k = nullptr, *src_v = nullptr, *dst_k = ka.as<u64>(), *dst_v = va.as<u64>();
    PassPlan plan = has_val ? plan_pass<u64, true>(c, n) : plan_pass<u64, false>(c, n);
    TRY(hist.alloc(plan.hist_bytes()));
    // digits on which all keys agree are skipped (e.g. 32-bit-range keys take 4 passes, not 8)
    u64 varying;
    {
        DevBuf bits(c);
        TRY(bits.alloc(16));
        const unsigned long long init[2] = {0ull, ~0ull};
        CU(cudaMemcpyAsync(bits.p, init, 16, cudaMemcpyHostToDevice, c->stream));
        KLaunch kl(s, K_MISC);
        key_bits_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(kscan, kstride, n, tx, (unsigned long long *)bits.p);
        TRY(kl.done("key_bits_kernel"));
        u64 *h = (u64 *)c->h_scratch;
        CU(cudaMemcpyAsync(h, bits.p, 16, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        varying = h[0] ^ h[1];
    }
    bool at_first = true;
    u32 done = 0;
    for (u32 p = 0; p < 8; ++p) {
        const u64 dmask = 0xFFull << (8 * p);
        const bool last_chance = p == 7 && done == 0;      // at least one pass: it also copies the rows out
        if (!(varying & dmask) && !last_chance) continue;
        ++done;
        const Loader ld = at_first ? first : Loader{LD_SOA64, src_k, has_val ? src_v : nullptr, 0};
        at_first = false;
        Digit dg{};
        dg.mode = DG_BITS; dg.shift = 8 * p; dg.mask = 0xFF; dg.tx = tx;
        if (has_val) TRY((radix_pass<u64, true>(s, ld, dg, n, dst_k, dst_v, hist.as<u32>(), plan)));
        else TRY((radix_pass<u64, false>(s, ld, dg, n, dst_k, nullptr, hist.as<u32>(), plan)));
        u64 *nk = (src_k == nullptr) ? kb.as<u64>() : src_k;
        u64 *nv = (src_v == nullptr) ? vbuf.as<u64>() : src_v;
        src_k = dst_k; src_v = dst_v; dst_k = nk; dst_v = nv;
    }
    *out_k = src_k;
    *out_v = has_val ? src_v : nullptr;
    return VB_OK;
}

static int seal_sort(vb_shuf *s, const Gathered &g)
{
    vb_ctx *c = s->ctx;
    const u32 R = s->n_reduce;
    s->bucket_off.assign((size_t)R + 1, 0);
    s->val_off.assign((size_t)R + 1, 0);
    const u64 n = g.n;
    if (n == 0) return VB_OK;
    const bool has_val = g.rows != nullptr || g.vals != nullptr;
    const int tx = s->kdt == VB_I64 ? TX_I64 : s->kdt == VB_F64 ? TX_F64 : TX_NONE;
    DevBuf ka(c), kb(c), va(c), vbuf(c);
    u64 *src_k = nullptr, *src_v = nullptr;
    const Loader first = g.rows ? Loader{LD_AOS64, g.rows, nullptr, 0} : Loader{LD_SOA64, g.keys, g.vals, 0};
    TRY(lsd_sort_u64(s, first, g.rows ? g.rows : g.keys, g.rows ? 2 : 1, n, tx, has_val, ka, kb, va, vbuf, &src_k, &src_v));
    DevBuf starts(c);
    TRY(starts.alloc(((size_t)R + 1) * 8));
    {
        KLaunch kl(s, K_MISC);
        sort_cuts_kernel<<<(R + 1 + 255) / 256, 256, 0, c->stream>>>(src_k, n, R, starts.as<u64>());
        TRY(kl.done("sort_cuts_kernel"));
    }
    CU(cudaMemcpyAsync(s->bucket_off.data(), starts.p, ((size_t)R + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    s->n_keys = n;
    s->res_keys = src_k;
    s->res_comb = has_val ? src_v : nullptr;
    if (src_k == ka.as<u64>()) ka.release(); else kb.release();
    if (has_val) { if (src_v == va.as<u64>()) va.release(); else vbuf.release(); }
    s->st.rows_out = n;
    return VB_OK;
}

// Each CSR run vals[offs[i] .. offs[i+1]) of the D keys sorted ascending in the value dtype's order, in place, when the
// shuffle asks for it (vb_shuffle_set_value_order; segsort.cuh).  Runs of 2 to SS_T values are sorted in shared memory,
// one launch per size class; the longer ones are gathered into one buffer of their values and run ranks, sorted stably
// by value and then by rank with the radix passes, and scattered back (temporary memory ~ 60 B per value of those runs).
static int sort_segments(vb_shuf *s, const u64 *offs, u64 D, u64 *vals, u64 n)
{
    if (s->vorder != VB_VALORDER_ASC || n <= D) return VB_OK;     // n == D: every list holds one value
    vb_ctx *c = s->ctx;
    const int tx = s->vdt == VB_I64 ? TX_I64 : s->vdt == VB_F64 ? TX_F64 : TX_NONE;
    DevBuf ctr(c), list(c);
    TRY(ctr.alloc(SS_NCLS * 4));
    CU(cudaMemsetAsync(ctr.p, 0, SS_NCLS * 4, c->stream));
    const unsigned grid = (unsigned)std::min<u64>((D + 255) / 256, (u64)c->sm_count * 8);
    {
        KLaunch kl(s, K_MISC, D);
        seg_classify_kernel<<<grid, 256, 0, c->stream>>>(offs, D, ctr.as<u32>(), nullptr, 0);
        TRY(kl.done("seg_classify_kernel"));
    }
    u32 *h = (u32 *)c->h_scratch;
    CU(cudaMemcpyAsync(h, ctr.p, SS_NCLS * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    std::vector<u32> cnt(h, h + SS_NCLS), start(SS_NCLS + 1, 0);
    for (int k = 0; k < SS_NCLS; ++k) start[k + 1] = start[k] + cnt[k];
    if (start[SS_NCLS] == 0) return VB_OK;
    TRY(list.alloc((u64)start[SS_NCLS] * 4));
    CU(cudaMemcpyAsync(ctr.p, start.data(), SS_NCLS * 4, cudaMemcpyHostToDevice, c->stream));   // pageable: copied before the call returns
    {
        KLaunch kl(s, K_MISC, D);
        seg_classify_kernel<<<grid, 256, 0, c->stream>>>(offs, D, ctr.as<u32>(), list.as<u32>(), 1);
        TRY(kl.done("seg_classify_kernel"));
    }
    const size_t smem = (size_t)SS_T * 8;
    CU(cudaFuncSetAttribute((const void *)seg_sort_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (u32 k = 0; k < (u32)SS_LOG_T; ++k) {
        if (!cnt[k]) continue;
        const u32 log_c = k + 1, per_cta = (u32)SS_T >> log_c;
        KLaunch kl(s, K_MISC, cnt[k]);
        seg_sort_cta_kernel<<<(cnt[k] + per_cta - 1) / per_cta, SS_THREADS, smem, c->stream>>>(vals, offs, list.as<u32>() + start[k], cnt[k],
                                                                                               log_c, tx);
        TRY(kl.done("seg_sort_cta_kernel"));
    }
    const u32 nl = cnt[SS_LOG_T];
    if (!nl) return VB_OK;
    // the large runs: bounds, and their values' buffer positions in list order
    DevBuf starts(c), lens(c), pref(c);
    TRY(starts.alloc((u64)nl * 8));
    TRY(lens.alloc((u64)nl * 8));
    TRY(pref.alloc(((u64)nl + 1) * 8));
    {
        KLaunch kl(s, K_MISC, nl);
        seg_bounds_kernel<<<(nl + 255) / 256, 256, 0, c->stream>>>(offs, list.as<u32>() + start[SS_LOG_T], nl, starts.as<u64>(), lens.as<u64>());
        TRY(kl.done("seg_bounds_kernel"));
    }
    std::vector<u64> hp((size_t)nl + 1, 0);
    CU(cudaMemcpyAsync(hp.data() + 1, lens.p, (u64)nl * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (u32 r = 0; r < nl; ++r) hp[r + 1] += hp[r];
    const u64 NL = hp[nl];
    CU(cudaMemcpyAsync(pref.p, hp.data(), ((u64)nl + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    lens.reset();
    const unsigned mgrid = (unsigned)std::min<u64>((NL + 255) / 256, (u64)c->sm_count * 8);
    DevBuf buf(c), rank(c);
    TRY(buf.alloc(NL * 8));
    TRY(rank.alloc(NL * 8));
    {
        KLaunch kl(s, K_MISC, NL);
        seg_move_kernel<<<mgrid, 256, 0, c->stream>>>(vals, starts.as<u64>(), pref.as<u64>(), nl, NL, buf.as<u64>(), rank.as<u64>(), 1);
        TRY(kl.done("seg_move_kernel"));
    }
    // stable by value (rank carried along), then stable by rank: each run's values together, ascending
    DevBuf ka(c), kb(c), va(c), vbuf(c), ids(c);
    u64 *sk = nullptr, *sr = nullptr;
    TRY(lsd_sort_u64(s, Loader{LD_SOA64, buf.as<u64>(), rank.as<u64>(), 0}, buf.as<u64>(), 1, NL, tx, true, ka, kb, va, vbuf, &sk, &sr));
    buf.reset();
    rank.reset();
    TRY(ids.alloc(NL * 4));
    {
        KLaunch kl(s, K_MISC, NL);
        narrow_u32_kernel<<<mgrid, 256, 0, c->stream>>>(sr, NL, ids.as<u32>());
        TRY(kl.done("narrow_u32_kernel"));
    }
    u32 *sorted_ids = nullptr;
    u64 *sorted_vals = nullptr;
    TRY(sort_id_pairs(s, ids.as<u32>(), Loader{LD_KEY32_VAL_SOA, nullptr, sk, 0}, NL, ceil_log2_u64(std::max<u64>(nl, 2)), &sorted_ids, &sorted_vals));
    DevBuf sid_guard(c), sv_guard(c);
    if (sorted_ids != ids.as<u32>()) sid_guard.p = sorted_ids;
    sv_guard.p = sorted_vals;
    KLaunch kl(s, K_MISC, NL);
    seg_move_kernel<<<mgrid, 256, 0, c->stream>>>(vals, starts.as<u64>(), pref.as<u64>(), nl, NL, sorted_vals, nullptr, 0);
    return kl.done("seg_move_kernel");
}

static void release_inputs(vb_shuf *s)
{
    dev_free(s->ctx, s->sh_tab); dev_free(s->ctx, s->sh_ctl);
    s->sh_tab = nullptr; s->sh_ctl = nullptr;
    for (auto &m : s->maps) if (m.present) { u64 n = m.n_rows; free_map(s, m); m.present = true; m.n_rows = n; }
    dev_free(s->ctx, s->gath_keys);
    dev_free(s->ctx, s->gath_vals);
    s->gath_keys = s->gath_vals = nullptr;
    dev_free(s->ctx, s->exp_keys);
    dev_free(s->ctx, s->exp_vals);
    dev_free(s->ctx, s->exp_hist);
    s->exp_keys = s->exp_vals = nullptr;
    s->exp_hist = nullptr;
    dev_free(s->ctx, s->imp_own_k);
    dev_free(s->ctx, s->imp_own_v);
    s->imp_own_k = s->imp_own_v = nullptr;
    dev_free(s->ctx, s->bx_lens);
    dev_free(s->ctx, s->bx_bytes);
    s->bx_lens = nullptr;
    s->bx_bytes = nullptr;
}

// Finish the local map side and pack rows by destination rank (caller holds c->mu).
static int export_prepare_locked(vb_shuf *s, uint64_t *counts)
{
    vb_ctx *c = s->ctx;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->exported || s->freed) return set_err(VB_ERR_STATE, "export after seal/export");
    }
    std::vector<u64> off;
    if (is_reduce_op(s->agg)) {
        void *tab = nullptr; u32 log_cap = 0; u64 n_ins = 0;
        TRY(merge_map_tables(s, &tab, &log_cap, &n_ins));
        off.assign((size_t)s->world + 1, 0);
        if (tab) {
            DevBuf guard(c); guard.p = tab;
            DevBuf k(c), v(c);
            TRY(k.alloc((n_ins + 1) * 8));
            TRY(v.alloc((n_ins + 1) * 8));
            const Table et = table_at(tab, log_cap);
            // vb_shuffle_set_dist caps world at TS_MAX_BINS (256): the unordered table split always applies
            TRY(multisplit_table_unordered(s, et, DG_DEST, s->world, k.as<u64>(), v.as<u64>(), off));
            s->exp_keys = (u64 *)k.release();
            s->exp_vals = (u64 *)v.release();
        }
    } else {
        Gathered g;
        TRY(gather_maps(s, &g));
        off.assign((size_t)s->world + 1, 0);
        if (g.n) {
            DevBuf k(c), v(c);
            TRY(k.alloc(g.n * 8));
            TRY(v.alloc(g.n * 8));
            Loader ld = g.rows ? Loader{LD_AOS64, g.rows, nullptr, 0} : Loader{LD_SOA64, g.keys, g.vals, 0};
            TRY(multisplit(s, ld, g.n, DG_DEST, s->world, g.n, k.as<u64>(), v.as<u64>(), off));
            s->exp_keys = (u64 *)k.release();
            s->exp_vals = (u64 *)v.release();
        }
    }
    for (u32 r = 0; r < s->world; ++r) counts[r] = off[r + 1] - off[r];
    std::lock_guard<std::mutex> g(s->mu);
    s->exported = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_prepare(vb_shuf *s, uint64_t *counts)
{
    if (s && s->rep) return reject_rep(s, "vb_shuffle_export_prepare");
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_export_prepare");
    if (!s || !counts) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "multi-rank exchange");
    if (s->str) return reject_str(s, "multi-rank exchange");
    // the packing below splits by hash destination; a sort shuffle is range-partitioned by cuts agreed across ranks
    if (s->agg == VB_AGG_SORT) return set_err(VB_ERR_UNSUPPORTED, "multi-rank sort_by_key goes through vb_shuffle_exchange");
    if (s->world < 2) return set_err(VB_ERR_STATE, "vb_shuffle_export_prepare needs vb_shuffle_set_dist(world > 1)");
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    TRY(export_prepare_locked(s, counts));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

// export_prepare_locked of a byte-string-value shuffle across ranks: the rows packed by destination, then their values'
// bytes packed in that order (bytes_pack); n_val_bytes[d] = the value bytes that go to rank d.  Caller holds c->mu.
static int export_bytes_locked(vb_shuf *s, u64 *counts, u64 *n_val_bytes)
{
    const u32 W = s->world;
    TRY(export_prepare_locked(s, counts));
    std::vector<u64> cut((size_t)W + 1, 0), at;
    for (u32 d = 0; d < W; ++d) cut[d + 1] = cut[d] + counts[d];
    TRY(bytes_pack(s, s->exp_vals, cut[W], cut, at));
    for (u32 d = 0; d < W; ++d) n_val_bytes[d] = at[d + 1] - at[d];
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// P2P exchange: rows go straight from the partition kernel into the peers' HBM over NVLink
// ---------------------------------------------------------------------------------------------
static int arena_reserve_locked(vb_ctx *c, uint64_t bytes, void *handle_out, uint64_t *generation)
{
    if (bytes > c->arena_bytes || !c->arena) {
        CU(cudaStreamSynchronize(c->stream));
        // peers may still have the old allocation mapped (they close it in vb_ctx_peer_open when they see the new
        // generation): keep it until vb_ctx_arena_release_retired, which the caller invokes after a barrier
        if (c->arena) c->retired_arenas.push_back(c->arena);
        c->arena = nullptr;
        size_t want = std::max<size_t>((size_t)bytes + bytes / 4, (size_t)64 << 20);
        want = (want + ((size_t)2 << 20) - 1) & ~(((size_t)2 << 20) - 1);
        CU(cudaMalloc(&c->arena, want));     // cudaMalloc, not the async pool: legacy IPC handles need it
        c->arena_bytes = want;
        c->arena_gen++;
    }
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, c->arena));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle_out, &h, sizeof(h));
    *generation = c->arena_gen;
    return VB_OK;
}

extern "C" int32_t vb_ctx_arena_reserve(vb_ctx *c, uint64_t bytes, void *handle_out, uint64_t *generation)
{
    if (!c || !handle_out || !generation) return set_err(VB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    return arena_reserve_locked(c, bytes, handle_out, generation);
}

// Free the arenas outgrown by vb_ctx_arena_reserve.  Contract: every peer has called vb_ctx_peer_open with this
// rank's current generation (which closes its mapping of the old one) — i.e. call it after the barrier that
// follows the exchange.
extern "C" int32_t vb_ctx_arena_release_retired(vb_ctx *c)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (void *p : c->retired_arenas) CU(cudaFree(p));
    c->retired_arenas.clear();
    return VB_OK;
}

static int peer_open_locked(vb_ctx *c, uint32_t peer_rank, const void *handle, uint64_t generation, int32_t is_self)
{
    auto &p = c->peers[peer_rank];
    if (is_self) { p.base = c->arena; p.gen = c->arena_gen; p.self = true; return VB_OK; }
    if (p.base && p.gen == generation && !p.self) return VB_OK;
    if (p.base && !p.self) { CU(cudaStreamSynchronize(c->stream)); cudaIpcCloseMemHandle(p.base); p.base = nullptr; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    void *base = nullptr;
    CU(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    p.base = base; p.gen = generation; p.self = false;
    return VB_OK;
}

extern "C" int32_t vb_ctx_peer_open(vb_ctx *c, uint32_t peer_rank, const void *handle, uint64_t generation, int32_t is_self)
{
    if (!c || (!handle && !is_self)) return set_err(VB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    return peer_open_locked(c, peer_rank, handle, generation, is_self);
}

// Histogram of this rank's rows by destination rank (no data movement yet); keeps the scanned
// per-part histogram for vb_shuffle_export_direct.  group ops only (reduce ops exchange a few MB of
// combined rows: vb_shuffle_export_prepare + one all-to-all-v is the right tool there).
static int export_counts_locked(vb_shuf *s, uint64_t *counts)
{
    if (!is_group_op(s->agg)) return set_err(VB_ERR_UNSUPPORTED, "the fused P2P export is for GROUP/COGROUP shuffles");
    vb_ctx *c = s->ctx;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->exported || s->exp_counted || s->freed) return set_err(VB_ERR_STATE, "export after seal/export");
    }
    Gathered g;
    TRY(gather_maps(s, &g));
    s->exp_rows = g.rows; s->exp_k = g.keys; s->exp_v = g.vals; s->exp_n = g.n;
    s->exp_digit_start.assign((size_t)s->world + 1, 0);
    if (g.n) {
        PassPlan plan = plan_pass<u64, true>(c, g.n);
        DevBuf hist(c);
        TRY(hist.alloc(plan.hist_bytes()));
        Loader ld = g.rows ? Loader{LD_AOS64, g.rows, nullptr, 0} : Loader{LD_SOA64, g.keys, g.vals, 0};
        Digit dg = make_bucket_digit(s, DG_DEST, 0, 0xFFFFFFFFu);
        TRY((radix_hist_scan<u64>(s, ld, dg, g.n, hist.as<u32>(), plan)));
        TRY(fetch_offsets(c, hist.as<u32>(), plan, s->world, s->exp_digit_start.data()));
        s->exp_hist = (u32 *)hist.release();
        s->exp_parts = plan.num_parts;
        s->exp_rows_per_part = plan.rows_per_part;
    }
    for (u32 r = 0; r < s->world; ++r) counts[r] = s->exp_digit_start[r + 1] - s->exp_digit_start[r];
    std::lock_guard<std::mutex> gg(s->mu);
    s->exp_counted = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_counts(vb_shuf *s, uint64_t *counts)
{
    if (s && s->rep) return reject_rep(s, "vb_shuffle_export_counts");
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_export_counts");
    if (!s || !counts) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "multi-rank exchange");
    if (s->str) return reject_str(s, "multi-rank exchange");
    if (s->world < 2) return set_err(VB_ERR_STATE, "vb_shuffle_export_counts needs vb_shuffle_set_dist(world > 1)");
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    return export_counts_locked(s, counts);
}

// The scatter: every row is stored into the arena of the rank that owns its reduce partition.
// dst_row_offset[d]: first row of my block inside rank d's arena; dst_total_rows[d]: rows rank d receives in total
// (its arena holds keys[total] then vals[total]).  Returns after the stores are complete on this GPU; the
// host then barriers the ranks before anyone reads its arena.
static int export_direct_locked(vb_shuf *s, const uint64_t *dst_row_offset, const uint64_t *dst_total_rows, bool sync)
{
    if (!s->exp_counted || s->exported) return set_err(VB_ERR_STATE, "vb_shuffle_export_direct needs vb_shuffle_export_counts first");
    vb_ctx *c = s->ctx;
    const u32 W = s->world;
    if (s->exp_n) {
        std::vector<u64 *> hk(W), hv(W);
        std::vector<u32> hadj(W);
        for (u32 d = 0; d < W; ++d) {
            auto it = c->peers.find(d);
            const u64 cnt = s->exp_digit_start[d + 1] - s->exp_digit_start[d];
            if (it == c->peers.end() || !it->second.base) {
                if (cnt) return set_err(VB_ERR_STATE, "peer %u arena not opened (vb_ctx_peer_open)", d);
                hk[d] = hv[d] = nullptr; hadj[d] = 0;
                continue;
            }
            if (dst_row_offset[d] + cnt > dst_total_rows[d] || dst_total_rows[d] >= 0xFFFFFFFFull)
                return set_err(VB_ERR_INVALID, "bad arena layout for destination %u", d);
            hk[d] = (u64 *)it->second.base;
            hv[d] = hk[d] + dst_total_rows[d];
            hadj[d] = (u32)(dst_row_offset[d] - s->exp_digit_start[d]);
        }
        DevBuf dk(c), dv(c), da(c);
        TRY(dk.alloc(W * 8)); TRY(dv.alloc(W * 8)); TRY(da.alloc(W * 4));
        CU(cudaMemcpyAsync(dk.p, hk.data(), W * 8, cudaMemcpyHostToDevice, c->stream));
        CU(cudaMemcpyAsync(dv.p, hv.data(), W * 8, cudaMemcpyHostToDevice, c->stream));
        CU(cudaMemcpyAsync(da.p, hadj.data(), W * 4, cudaMemcpyHostToDevice, c->stream));
        Loader ld = s->exp_rows ? Loader{LD_AOS64, s->exp_rows, nullptr, 0} : Loader{LD_SOA64, s->exp_k, s->exp_v, 0};
        Digit dg = make_bucket_digit(s, DG_DEST, 0, 0xFFFFFFFFu);
        const void *sk = s->exp_rows ? (const void *)rp_scatter_kernel<u64, true, LD_AOS64, DG_DEST, true>
                                     : (const void *)rp_scatter_kernel<u64, true, LD_SOA64, DG_DEST, true>;
        const size_t smem = rp_scatter_smem<u64, true>();
        CU(cudaFuncSetAttribute(sk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        u64 n = s->exp_n, rpp = s->exp_rows_per_part;
        u32 np = s->exp_parts;
        const u32 *ch = s->exp_hist;
        u64 *nullk = nullptr, *nullv = nullptr;
        RemoteDst rd{dk.as<u64 *>(), dv.as<u64 *>(), da.as<u32>(), W};
        KLaunch kl(s, K_RP_SCATTER, n);
        void *args[] = {&ld, &dg, &n, &rpp, &ch, &np, &nullk, &nullv, &rd};
        CU(cudaLaunchKernel(sk, dim3(np), dim3(RPS_THREADS), args, smem, c->stream));
        TRY(kl.done("rp_scatter_kernel<REMOTE>"));
        if (sync) CU(cudaStreamSynchronize(c->stream));
    }
    dev_free(c, s->exp_hist);
    s->exp_hist = nullptr;
    std::lock_guard<std::mutex> g(s->mu);
    s->exported = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_direct(vb_shuf *s, const uint64_t *dst_row_offset, const uint64_t *dst_total_rows)
{
    if (s && s->rep) return reject_rep(s, "vb_shuffle_export_direct");
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_export_direct");
    if (!s || !dst_row_offset || !dst_total_rows) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "multi-rank exchange");
    if (s->str) return reject_str(s, "multi-rank exchange");
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    return export_direct_locked(s, dst_row_offset, dst_total_rows, true);
}

// The rows of every source rank are already in this context's arena (keys[total] then vals[total],
// source-rank major): hand them to the reduce side.  counts[world] as in vb_shuffle_import.
extern "C" int32_t vb_shuffle_import_arena(vb_shuf *s, const uint64_t *counts)
{
    if (s && s->rep) return reject_rep(s, "vb_shuffle_import_arena");
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_import_arena");
    if (!s || !counts) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "multi-rank exchange");
    if (s->str) return reject_str(s, "multi-rank exchange");
    if (!s->exported || s->sealed) return set_err(VB_ERR_STATE, "import needs the export first and no seal yet");
    u64 n = 0;
    for (u32 r = 0; r < s->world; ++r) n += counts[r];
    if (n * 16 > s->ctx->arena_bytes) return set_err(VB_ERR_INVALID, "arena holds %zu bytes, %llu rows announced", s->ctx->arena_bytes, (unsigned long long)n);
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "import of %llu rows", (unsigned long long)n);
    s->imp_keys = (const u64 *)s->ctx->arena;
    s->imp_vals = s->imp_keys + n;
    s->imp_n = n;
    s->imported = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_buffers(vb_shuf *s, void **keys_dev, void **vals_dev)
{
    if (s && s->rep) return reject_rep(s, "vb_shuffle_export_buffers");
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_export_buffers");
    if (!s || !keys_dev || !vals_dev) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "multi-rank exchange");
    if (s->str) return reject_str(s, "multi-rank exchange");
    if (!s->exported) return set_err(VB_ERR_STATE, "vb_shuffle_export_buffers before vb_shuffle_export_prepare");
    *keys_dev = s->exp_keys;
    *vals_dev = s->exp_vals;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_import(vb_shuf *s, const void *keys_dev, const void *vals_dev, const uint64_t *counts)
{
    if (s && s->rep) return reject_rep(s, "vb_shuffle_import");
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_import");
    if (!s || !counts) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "multi-rank exchange");
    if (s->str) return reject_str(s, "multi-rank exchange");
    if (!s->exported || s->sealed) return set_err(VB_ERR_STATE, "import needs export_prepare first and no seal yet");
    u64 n = 0;
    for (u32 r = 0; r < s->world; ++r) n += counts[r];
    if (n && (!keys_dev || !vals_dev)) return set_err(VB_ERR_INVALID, "NULL buffers with rows to import");
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "import of %llu rows", (unsigned long long)n);
    s->imp_keys = (const u64 *)keys_dev;
    s->imp_vals = (const u64 *)vals_dev;
    s->imp_n = n;
    s->imported = true;
    return VB_OK;
}


// ---------------------------------------------------------------------------------------------
// The exchange behind the C ABI (ShuffleFetcher::fetch, src/shuffle/shuffle_fetcher.rs:16-119):
// one NCCL communicator per context, counts + rows exchanged on the library's own stream.
// NCCL is loaded with dlopen on first use, so single-GPU users carry no dependency on it.
// ---------------------------------------------------------------------------------------------
#include <dlfcn.h>
#include <nccl.h>

struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int *) = nullptr;
};
static NcclApi g_nccl;
static std::mutex g_nccl_mu;

static int nccl_load()
{
    std::lock_guard<std::mutex> g(g_nccl_mu);
    if (g_nccl.h) return VB_OK;
    const char *names[] = {getenv("VEGA_B200_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    void *h = nullptr;
    for (const char *nm : names) {
        if (!nm) continue;
        h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
        if (h) break;
    }
    if (!h) return set_err(VB_ERR_UNSUPPORTED, "NCCL not found (dlopen libnccl.so.2): %s", dlerror());
#define LD(f)                                                                                      \
    do {                                                                                           \
        *(void **)(&g_nccl.f) = dlsym(h, "nccl" #f);                                               \
        if (!g_nccl.f) return set_err(VB_ERR_UNSUPPORTED, "libnccl lacks nccl" #f);                \
    } while (0)
    LD(GetUniqueId); LD(CommInitRank); LD(CommDestroy); LD(GroupStart); LD(GroupEnd); LD(Send); LD(Recv); LD(AllGather);
    LD(GetErrorString); LD(GetVersion);
#undef LD
    g_nccl.h = h;
    return VB_OK;
}

#define NC(expr)                                                                                             \
    do {                                                                                                     \
        ncclResult_t r_ = (expr);                                                                            \
        if (r_ != ncclSuccess) return set_err(VB_ERR_CUDA, "%s:%d %s: NCCL %s", __FILE__, __LINE__, #expr,    \
                                              g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "error");   \
    } while (0)

struct Comm {
    ncclComm_t comm = nullptr;
    u32 rank = 0, world = 1;
    u64 *d_send = nullptr;     // [comm_row(world)]: this rank's row of the count all-gather (comm_all_gather)
    u64 *d_recv = nullptr;     // [world][comm_row(world)]
    unsigned char *d_hs = nullptr, *d_hr = nullptr;   // IPC handle + generation: 80 bytes, [world] x 80
    std::vector<u64> peer_arena_bytes, peer_gen_seen;
    bool handles_valid = false;
};
constexpr u32 COMM_MAX_WORLD = 64;
constexpr size_t COMM_HOST_OFF = 256 << 10;   // staging region inside vb_ctx::h_scratch: the count matrix, then the IPC handles
constexpr size_t COMM_MAT_BYTES = 192 << 10;  // the count matrix and this rank's row: (world + 1) * comm_row(world) u64
static_assert(COMM_HOST_OFF + COMM_MAT_BYTES + 128 + 80 * 64 <= (1 << 20) - 4096, "staging inside h_scratch, before its status cells");
// u64 per rank of the count all-gather: world + 2 for integer rows (counts, arena bytes and generation), world + 3 for
// combine_by_key (counts and the spec's fingerprint), 3 * world for String keys, 2 * world + 3 for String-key
// combine_by_key (key and byte counts, and the spec's fingerprint), 2 * world for integer rows with byte-string values
// (counts and value bytes), 4 * world for String keys with them, 2 for sort, 3 for String sort
static size_t comm_row(u32 world) { return std::max<size_t>({(size_t)world + 2, 4 * (size_t)world, 2 * (size_t)world + 3}); }
static_assert((COMM_MAX_WORLD + 1) * 4 * COMM_MAX_WORLD * 8 <= COMM_MAT_BYTES, "the widest count matrix fits its staging");

static void comm_teardown(vb_ctx *c)
{
    Comm *m = c->comm;
    if (!m) return;
    // every rank has closed its peer mappings before this point; the all-gather is the barrier that lets the
    // owners free the exported arenas afterwards
    if (m->comm && g_nccl.AllGather && m->d_send && m->d_recv) {
        if (g_nccl.AllGather(m->d_send, m->d_recv, 1, ncclUint64, m->comm, c->stream) == ncclSuccess) cudaStreamSynchronize(c->stream);
    }
    if (m->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(m->comm);
    cudaFree(m->d_send); cudaFree(m->d_recv); cudaFree(m->d_hs); cudaFree(m->d_hr);
    cudaGetLastError();
    delete m;
    c->comm = nullptr;
}

extern "C" int32_t vb_comm_unique_id(void *id_out)
{
    if (!id_out) return set_err(VB_ERR_INVALID, "id_out is NULL");
    TRY(nccl_load());
    static_assert(sizeof(ncclUniqueId) == VB_UNIQUE_ID_BYTES, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    NC(g_nccl.GetUniqueId(&id));
    memcpy(id_out, &id, sizeof(id));
    return VB_OK;
}

extern "C" int32_t vb_ctx_comm_init(vb_ctx *c, const void *unique_id, uint32_t rank, uint32_t world)
{
    if (!c || !unique_id) return set_err(VB_ERR_INVALID, "NULL argument");
    if (world < 1 || rank >= world || world > COMM_MAX_WORLD) return set_err(VB_ERR_INVALID, "bad rank/world (world <= %u)", COMM_MAX_WORLD);
    TRY(nccl_load());
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    if (c->comm) return set_err(VB_ERR_STATE, "context already has a communicator");
    Comm *m = new Comm();
    m->rank = rank; m->world = world;
    ncclUniqueId id;
    memcpy(&id, unique_id, sizeof(id));
    ncclResult_t r = g_nccl.CommInitRank(&m->comm, (int)world, id, (int)rank);
    if (r != ncclSuccess) { delete m; return set_err(VB_ERR_CUDA, "ncclCommInitRank: %s", g_nccl.GetErrorString(r)); }
    c->comm = m;
    CU(cudaMalloc((void **)&m->d_send, comm_row(world) * 8));
    CU(cudaMalloc((void **)&m->d_recv, (size_t)world * comm_row(world) * 8));
    CU(cudaMalloc((void **)&m->d_hs, 80));
    CU(cudaMalloc((void **)&m->d_hr, (size_t)world * 80));
    CU(cudaMemset(m->d_send, 0, comm_row(world) * 8));
    m->peer_arena_bytes.assign(world, 0);
    m->peer_gen_seen.assign(world, 0);
    return VB_OK;
}

extern "C" int32_t vb_ctx_comm_destroy(vb_ctx *c)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    for (auto &kv : c->peers) if (kv.second.base && !kv.second.self) { cudaIpcCloseMemHandle(kv.second.base); kv.second.base = nullptr; }
    c->peers.clear();
    comm_teardown(c);
    return VB_OK;
}

extern "C" int32_t vb_ctx_comm_info(vb_ctx *c, uint32_t *rank, uint32_t *world, int32_t *nccl_version)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    if (!c->comm) return set_err(VB_ERR_STATE, "no communicator (vb_ctx_comm_init)");
    if (rank) *rank = c->comm->rank;
    if (world) *world = c->comm->world;
    if (nccl_version) { int v = 0; g_nccl.GetVersion(&v); *nccl_version = v; }
    return VB_OK;
}

// ---- the exchange, written once -------------------------------------------------------------------------------
// Every kind runs the same steps: export; ONE all-gather of a row of u64 counts per rank (comm_all_gather); limit
// checks taken from the gathered matrix for every rank, so all ranks return the same code and either every rank
// enters the send/recv group or none does; receive buffers; ONE grouped send/recv (post_group); bookkeeping
// (xchg_done).  The column kinds (integer rows, combine_by_key, String keys) describe their columns to xfers, which
// splits each by one count vector of the matrix; sort sends per output partition and builds its own transfer list.
// A failed local allocation after the checks can still leave one rank out of the group: that is not covered.

// All-gather of this rank's row of `len` u64 (at most comm_row(world)) through the pinned staging area: one small
// collective and one D2H.  Returns the host matrix [world][len].
static int comm_all_gather(vb_ctx *c, const u64 *row, size_t len, const u64 **matrix)
{
    Comm *m = c->comm;
    const u32 W = m->world;
    if (len > comm_row(W)) return set_err(VB_ERR_INVALID, "count row of %zu u64 exceeds the communicator's %zu", len, comm_row(W));
    u64 *h = (u64 *)((char *)c->h_scratch + COMM_HOST_OFF);
    u64 *hs = h + (size_t)W * len;
    memcpy(hs, row, len * 8);
    CU(cudaMemcpyAsync(m->d_send, hs, len * 8, cudaMemcpyHostToDevice, c->stream));
    NC(g_nccl.AllGather(m->d_send, m->d_recv, len, ncclUint64, m->comm, c->stream));
    CU(cudaMemcpyAsync(h, m->d_recv, (size_t)W * len * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    *matrix = h;
    return VB_OK;
}

struct Xfer {   // one transfer of a grouped send/recv: n elements of type dt to (send) or from peer at p
    bool send;
    u32 peer;
    const void *p;
    u64 n;
    ncclDataType_t dt;
};

// Device interval of the exchange, resolved later by vb_shuffle_exchange_stats / vb_shuffle_stats (no host wait here)
static cudaEvent_t xchg_mark(vb_ctx *c)
{
    cudaEvent_t e = nullptr;
    if (c->profile) { cudaEventCreate(&e); cudaEventRecord(e, c->stream); }
    return e;
}

static void xchg_timed(vb_shuf *s, cudaEvent_t e0)
{
    if (!e0) return;
    cudaEvent_t e1 = nullptr;
    cudaEventCreate(&e1);
    cudaEventRecord(e1, s->ctx->stream);
    s->timers.push_back(Timer{e0, e1, -3, 0});
}

// The one GroupStart ... GroupEnd: every transfer of `xs` with a non-zero count, timed as the exchange
static int post_group(vb_shuf *s, const std::vector<Xfer> &xs)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    const cudaEvent_t e0 = xchg_mark(c);
    NC(g_nccl.GroupStart());
    for (const Xfer &x : xs) {
        if (!x.n) continue;
        if (x.send) NC(g_nccl.Send(x.p, x.n, x.dt, (int)x.peer, m->comm, c->stream));
        else NC(g_nccl.Recv((void *)x.p, x.n, x.dt, (int)x.peer, m->comm, c->stream));
    }
    NC(g_nccl.GroupEnd());
    xchg_timed(s, e0);
    return VB_OK;
}

// What rank `me` sends to and receives from every peer by count vector `vec` (entries [vec * W, vec * W + W) of every
// row) of the gathered matrix, and where each peer's run starts on either side (source-rank major at the receiver)
struct XSplit { std::vector<u64> send, recv, soff, roff; };   // [W], [W], [W + 1], [W + 1]

static XSplit xsplit(const u64 *mat, size_t len, u32 W, u32 me, u32 vec)
{
    XSplit x{std::vector<u64>(W), std::vector<u64>(W), std::vector<u64>(W + 1, 0), std::vector<u64>(W + 1, 0)};
    for (u32 p = 0; p < W; ++p) {
        x.send[p] = mat[me * len + (size_t)vec * W + p];
        x.recv[p] = mat[p * len + (size_t)vec * W + me];
        x.soff[p + 1] = x.soff[p] + x.send[p];
        x.roff[p + 1] = x.roff[p] + x.recv[p];
    }
    return x;
}

// One column of a per-peer exchange: element type, send and receive base, and the count vector that splits it
struct XCol { ncclDataType_t dt; const void *send; void *recv; u32 vec; };

// The transfer list of the column kinds: to and from every peer, each column's run at its offset
static std::vector<Xfer> xfers(const std::vector<XSplit> &sp, const std::vector<XCol> &cols, u32 W)
{
    auto bytes = [](ncclDataType_t dt) -> u64 { return dt == ncclUint8 ? 1 : dt == ncclUint32 ? 4 : 8; };
    std::vector<Xfer> xs;
    for (u32 p = 0; p < W; ++p) {
        for (const XCol &k : cols)
            xs.push_back(Xfer{true, p, (const char *)k.send + sp[k.vec].soff[p] * bytes(k.dt), sp[k.vec].send[p], k.dt});
        for (const XCol &k : cols)
            xs.push_back(Xfer{false, p, (char *)k.recv + sp[k.vec].roff[p] * bytes(k.dt), sp[k.vec].recv[p], k.dt});
    }
    return xs;
}

// vb_shuffle_exchange_stats of one exchange.  Host wall clock of each of the three phases (export, count all-gather,
// the rest): lap() = ms since t, and t = now.  `sent` and `recv` count what crossed to or from other ranks, in the
// kind's unit of a row: values for String keys, keys for combine_by_key, rows otherwise.
static double lap(std::chrono::steady_clock::time_point &t)
{
    const auto t0 = t;
    t = std::chrono::steady_clock::now();
    return std::chrono::duration<double, std::milli>(t - t0).count();
}

static void xchg_done(vb_shuf *s, int kind, u64 sent, u64 recv)
{
    s->xst.sent_rows += sent;
    s->xst.recv_rows += recv;
    s->xst.exchanges += 1;
    s->xst.kind = kind;
}

// reduce ops and non-P2P group ops: pack by destination, then ONE grouped send/recv carrying both columns
static int exchange_nccl_locked(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    const u32 W = m->world, me = m->rank;
    // byte-string values: counts[W] and value bytes[W], and u32 value lengths plus the bytes in place of the values
    const bool bx = s->bdist;
    const size_t len = bx ? 2 * (size_t)W : (size_t)W + 2;   // counts[W], arena bytes, arena generation
    std::vector<u64> row(len, 0);
    auto clk = std::chrono::steady_clock::now();
    TRY(bx ? export_bytes_locked(s, row.data(), row.data() + W) : export_prepare_locked(s, row.data()));
    s->xst.prepare_wall_ms += lap(clk);
    if (!bx) {
        row[W] = c->arena_bytes;
        row[W + 1] = c->arena_gen;
    }
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, row.data(), len, &mat));
    s->xst.counts_wall_ms += lap(clk);
    for (u32 d = 0; d < W; ++d) {
        const u64 nd = xsplit(mat, len, W, d, 0).roff[W];
        if (nd >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "rank %u would receive %llu rows", d, (unsigned long long)nd);
    }
    std::vector<XSplit> sp{xsplit(mat, len, W, me, 0)};
    if (bx) sp.push_back(xsplit(mat, len, W, me, 1));
    const u64 n_recv = sp[0].roff[W];
    DevBuf rk(c), rv(c), rl(c), rb(c);
    TRY(rk.alloc(std::max<u64>(n_recv, 1) * 8));
    if (bx) {
        TRY(rl.alloc(n_recv * 4));
        TRY(rb.alloc(sp[1].roff[W]));
        TRY(post_group(s, xfers(sp, {{ncclUint64, s->exp_keys, rk.p, 0}, {ncclUint32, s->bx_lens, rl.p, 0}, {ncclUint8, s->bx_bytes, rb.p, 1}}, W)));
        TRY(bytes_adopt(s, rl.as<u32>(), n_recv, rb, sp[1].roff[W], rv));
    } else {
        TRY(rv.alloc(std::max<u64>(n_recv, 1) * 8));
        TRY(post_group(s, xfers(sp, {{ncclUint64, s->exp_keys, rk.p, 0}, {ncclUint64, s->exp_vals, rv.p, 0}}, W)));
    }
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_NCCL, sp[0].soff[W] - sp[0].send[me], n_recv - sp[0].recv[me]);
    s->imp_own_k = (u64 *)rk.release();
    s->imp_own_v = (u64 *)rv.release();
    std::lock_guard<std::mutex> g(s->mu);
    s->imp_keys = s->imp_own_k; s->imp_vals = s->imp_own_v; s->imp_n = n_recv;
    s->imported = true;
    return VB_OK;
}

// group ops: the destination-rank partition kernel stores straight into the owners' arenas (peer memory)
static int exchange_p2p_locked(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    const u32 W = m->world, me = m->rank;
    const size_t len = (size_t)W + 2;            // counts[W], arena bytes, arena generation
    std::vector<u64> row(len, 0);
    const cudaEvent_t e0 = xchg_mark(c);
    auto clk = std::chrono::steady_clock::now();
    TRY(export_counts_locked(s, row.data()));
    s->xst.prepare_wall_ms += lap(clk);
    row[W] = c->arena_bytes;
    row[W + 1] = c->arena_gen;
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, row.data(), len, &mat));
    s->xst.counts_wall_ms += lap(clk);
    // arena layout (source-rank major = map-id order) from the count matrix
    std::vector<u64> total(W, 0), my_off(W, 0);
    for (u32 dst = 0; dst < W; ++dst)
        for (u32 src = 0; src < W; ++src) {
            const u64 x = mat[src * len + dst];
            if (src < me) my_off[dst] += x;
            total[dst] += x;
        }
    // who must (re)grow its arena is a pure function of the gathered matrix: handles are re-exchanged only then
    bool any_regrow = !m->handles_valid;
    for (u32 p = 0; p < W; ++p) {
        const u64 need = 16 * std::max<u64>(total[p], 1), have = mat[p * len + W], gen = mat[p * len + W + 1];
        if (need > have || gen == 0 || gen != m->peer_gen_seen[p]) any_regrow = true;
    }
    unsigned char hbuf[80];
    u64 gen = 0;
    TRY(arena_reserve_locked(c, 16 * std::max<u64>(total[me], 1), hbuf, &gen));
    if (any_regrow) {
        memcpy(hbuf + 64, &gen, 8);
        memset(hbuf + 72, 0, 8);
        unsigned char *hh = (unsigned char *)c->h_scratch + COMM_HOST_OFF + COMM_MAT_BYTES;
        memcpy(hh, hbuf, 80);
        CU(cudaMemcpyAsync(m->d_hs, hh, 80, cudaMemcpyHostToDevice, c->stream));
        NC(g_nccl.AllGather(m->d_hs, m->d_hr, 80, ncclUint8, m->comm, c->stream));
        CU(cudaMemcpyAsync(hh + 128, m->d_hr, (size_t)W * 80, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        for (u32 p = 0; p < W; ++p) {
            u64 pg;
            memcpy(&pg, hh + 128 + (size_t)p * 80 + 64, 8);
            TRY(peer_open_locked(c, p, hh + 128 + (size_t)p * 80, pg, p == me));
            m->peer_gen_seen[p] = pg;
        }
        m->handles_valid = true;
    }
    TRY(export_direct_locked(s, my_off.data(), total.data(), false));
    // stream-ordered barrier: every rank's stores precede its part of this collective, which precedes my reads
    NC(g_nccl.AllGather(m->d_send, m->d_recv, 1, ncclUint64, m->comm, c->stream));
    if (any_regrow) {       // every peer has re-opened: outgrown arenas can go
        CU(cudaStreamSynchronize(c->stream));
        for (void *p : c->retired_arenas) CU(cudaFree(p));
        c->retired_arenas.clear();
    }
    const XSplit sp = xsplit(mat, len, W, me, 0);
    const u64 n = sp.roff[W];
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "import of %llu rows", (unsigned long long)n);
    xchg_timed(s, e0);
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_P2P, sp.soff[W] - sp.send[me], n - sp.recv[me]);
    std::lock_guard<std::mutex> g(s->mu);
    s->imp_keys = (const u64 *)c->arena;
    s->imp_vals = s->imp_keys + n;
    s->imp_n = n;
    s->imported = true;
    return VB_OK;
}


// ---------------------------------------------------------------------------------------------
// combine_by_key across ranks (vb_shuffle_create_multi_dist): each rank exports one row per distinct key it holds,
// the key plus the partial of every accumulator in plain value form, packed by destination rank; the owner merges the
// received partials into a fresh table (hash_agg_multi_kernel<IN_ACCS>) and finalizes it as the one-process seal does.
// ---------------------------------------------------------------------------------------------
extern "C" int32_t vb_shuffle_create_multi_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t kdt,
                                                uint32_t n_val_cols, const int32_t *val_dtypes, uint32_t n_aggs, const vb_agg_col *aggs,
                                                uint32_t rank, uint32_t world, vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_multi_dist: NULL argument");
    *out = nullptr;
    if (world < 1 || world > 256 || rank >= world) return set_err(VB_ERR_INVALID, "bad rank %u / world %u (1 <= world <= 256)", rank, world);
    TRY(vb_shuffle_create_multi(c, shuffle_id, n_map, n_reduce, kdt, n_val_cols, val_dtypes, n_aggs, aggs, out));
    (*out)->rank = rank;
    (*out)->world = world;
    return VB_OK;
}

// the checks every _cols export / import call makes first
static int multi_dist_check(const vb_shuf *s, const char *what)
{
    if (!s->multi || s->str) return set_err(VB_ERR_INVALID, "%s needs a shuffle from vb_shuffle_create_multi_dist", what);
    if (s->world < 2) return set_err(VB_ERR_STATE, "%s needs a multi-aggregate shuffle of world > 1 (vb_shuffle_create_multi_dist)", what);
    return VB_OK;
}

// Merge the local map tables and split the merged table's keys by owner rank: count, read the counts back, then one
// scatter of the key and every accumulator column with the exact exported total as column stride.  Caller holds c->mu.
static int export_cols_locked(vb_shuf *s, u64 *counts)
{
    vb_ctx *c = s->ctx;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->sealing || s->exported || s->freed) return set_err(VB_ERR_STATE, "export after seal/export");
    }
    const u32 W = s->world;
    for (u32 d = 0; d < W; ++d) counts[d] = 0;
    void *tab = nullptr; u32 log_cap = 0; u64 n_ins = 0;
    TRY(merge_map_tables(s, &tab, &log_cap, &n_ins));
    if (tab) {
        DevBuf guard(c); guard.p = tab;
        const Table et = table_at(tab, log_cap);
        const u64 cap = 1ull << log_cap;
        DevBuf cc(c);
        TRY(cc.alloc(2 * TS_MAX_BINS * 4));
        CU(cudaMemsetAsync(cc.p, 0, 2 * TS_MAX_BINS * 4, c->stream));
        u32 *cnt = cc.as<u32>(), *cursors = cc.as<u32>() + TS_MAX_BINS;
        const Digit dg = make_bucket_digit(s, DG_DEST, 0, 0xFFFFFFFFu);
        const unsigned grid = (unsigned)std::min<u64>((cap + TS_TILE) / TS_TILE, (u64)c->sm_count * 4);
        {
            KLaunch kl(s, K_RP_HIST, cap + 1);
            table_bin_count_kernel<DG_DEST><<<grid, TS_THREADS, 0, c->stream>>>(et.keys, cap, dg, cnt);
            TRY(kl.done("table_bin_count_kernel"));
        }
        u32 *h = (u32 *)c->h_scratch;
        CU(cudaMemcpyAsync(h, cnt, W * 4, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        u64 total = 0;
        for (u32 d = 0; d < W; ++d) { counts[d] = h[d]; total += h[d]; }
        if (total) {
            DevBuf k(c), a(c);
            TRY(k.alloc(total * 8));
            TRY(a.alloc(total * 8 * s->acc_map.n));
            KLaunch kl(s, K_RP_SCATTER, cap + 1);
            table_bin_scatter_multi_kernel<<<grid, TS_THREADS, 0, c->stream>>>(et.keys, et.accs, acc_stride(log_cap), cap, dg, s->acc_map, cnt,
                                                                               cursors, total, k.as<u64>(), a.as<u64>());
            TRY(kl.done("table_bin_scatter_multi_kernel"));
            s->exp_keys = (u64 *)k.release();
            s->exp_vals = (u64 *)a.release();
        }
        CU(cudaStreamSynchronize(c->stream));
    }
    std::lock_guard<std::mutex> g(s->mu);
    s->exported = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_cols_prepare(vb_shuf *s, uint64_t *counts)
{
    if (!s || !counts) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(multi_dist_check(s, "vb_shuffle_export_cols_prepare"));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    return export_cols_locked(s, counts);
}

extern "C" int32_t vb_shuffle_export_cols_buffers(vb_shuf *s, void **keys, void **accs, uint32_t *n_acc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    TRY(multi_dist_check(s, "vb_shuffle_export_cols_buffers"));
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (!s->exported || s->sealed || s->freed) return set_err(VB_ERR_STATE, "vb_shuffle_export_cols_buffers needs vb_shuffle_export_cols_prepare first and no seal yet");
    }
    if (keys) *keys = s->exp_keys;
    if (accs) *accs = s->exp_vals;
    if (n_acc) *n_acc = s->acc_map.n;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_import_cols(vb_shuf *s, const void *keys, const void *accs, uint32_t n_acc, const uint64_t *counts)
{
    if (!s || !counts) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(multi_dist_check(s, "vb_shuffle_import_cols"));
    if (n_acc != s->acc_map.n) return set_err(VB_ERR_INVALID, "%u accumulator columns imported, the shuffle has %u", n_acc, s->acc_map.n);
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (!s->exported || s->imported || s->sealed || s->sealing || s->freed)
            return set_err(VB_ERR_STATE, "vb_shuffle_import_cols needs vb_shuffle_export_cols_prepare first, once, and no seal yet");
    }
    u64 n = 0;
    for (u32 r = 0; r < s->world; ++r) n += counts[r];
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "import of %llu rows (fewer than 2^32 - 2 are supported)", (unsigned long long)n);
    if (n && (!keys || !accs)) return set_err(VB_ERR_INVALID, "NULL column with a non-zero count");
    std::lock_guard<std::mutex> g(s->mu);
    s->imp_keys = (const u64 *)keys;
    s->imp_vals = (const u64 *)accs;
    s->imp_n = n;
    s->imported = true;
    return VB_OK;
}

// vb_shuffle_exchange of a multi-aggregate shuffle: export, then the exchange of the key column and the n_acc
// accumulator columns, all split by the key counts.  The gathered row carries the spec's fingerprint after the counts,
// so a rank whose spec differs is refused on every rank.
static int exchange_multi_locked(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    const u32 W = m->world, me = m->rank, NA = s->acc_map.n;
    const size_t len = (size_t)W + 3;            // counts[W], then the fingerprint: <= comm_row(W) for W >= 2
    std::vector<u64> row(len, 0);
    auto clk = std::chrono::steady_clock::now();
    TRY(export_cols_locked(s, row.data()));
    s->xst.prepare_wall_ms += lap(clk);
    row[W] = s->acc_map.op;
    row[W + 1] = s->acc_map.tx;
    row[W + 2] = (u64)NA | (u64)s->key_width << 8 | (u64)s->n_reduce << 32;
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, row.data(), len, &mat));
    s->xst.counts_wall_ms += lap(clk);
    for (u32 p = 1; p < W; ++p)
        for (u32 i = 0; i < 3; ++i)
            if (mat[p * len + W + i] != mat[W + i])
                return set_err(VB_ERR_INVALID, "rank %u's combine spec differs from rank 0's (accumulators, ops, transforms, key width or n_reduce)", p);
    for (u32 d = 0; d < W; ++d) {
        const u64 nd = xsplit(mat, len, W, d, 0).roff[W];
        if (nd >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "rank %u would receive %llu rows", d, (unsigned long long)nd);
    }
    const std::vector<XSplit> sp{xsplit(mat, len, W, me, 0)};
    const u64 n_sent = sp[0].soff[W], n_recv = sp[0].roff[W];
    DevBuf rk(c), ra(c);
    TRY(rk.alloc(std::max<u64>(n_recv, 1) * 8));
    TRY(ra.alloc(std::max<u64>(n_recv, 1) * 8 * NA));
    std::vector<XCol> cols{{ncclUint64, s->exp_keys, rk.p, 0}};
    for (u32 a = 0; a < NA; ++a) cols.push_back({ncclUint64, s->exp_vals + (u64)a * n_sent, ra.as<u64>() + (u64)a * n_recv, 0});
    TRY(post_group(s, xfers(sp, cols, W)));
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_NCCL, n_sent - sp[0].send[me], n_recv - sp[0].recv[me]);
    s->imp_own_k = (u64 *)rk.release();
    s->imp_own_v = (u64 *)ra.release();
    std::lock_guard<std::mutex> g(s->mu);
    s->imp_keys = s->imp_own_k; s->imp_vals = s->imp_own_v; s->imp_n = n_recv;
    s->imported = true;
    return VB_OK;
}


// ---- multi-rank sort_by_key -----------------------------------------------------------------------------------
// (no reference code: sort_by_key is absent from vega, SURVEY.md F2 — semantics = the single-GPU ones: output
// partition p is the p-th contiguous key range, cut at floor(p*N/R) moved past equal keys, stable.)
// Every rank sorts its rows locally, the ranks find the EXACT global cut keys by bisection over the key space
// (64 rounds, each one tiny all-gather of R-1 counts obtained by binary search in the sorted local run), each
// rank's sorted run is then cut into contiguous segments that travel in ONE grouped send/recv to the owners
// (partition p lives on rank p % world), and the owner's seal re-sorts what it received (stable: source-rank-major
// arrival order = map-id order).
__global__ void count_le_kernel(const u64 *__restrict__ sorted, u64 n, int tx, const u64 *__restrict__ cand, u32 m, u64 *__restrict__ out)
{
    const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const u64 v = cand[p];
    u64 lo = 0, hi = n;                       // first index whose transformed key is > v
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (tx_fwd(sorted[mid], tx) <= v) lo = mid + 1; else hi = mid;
    }
    out[p] = lo;
}

static int exchange_sort_locked(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    const u32 W = m->world, me = m->rank, R = s->n_reduce;
    if (R > 4096) return set_err(VB_ERR_UNSUPPORTED, "multi-rank sort_by_key supports up to 4096 output partitions");
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->exported || s->freed) return set_err(VB_ERR_STATE, "export after seal/export");
    }
    const int tx = s->kdt == VB_I64 ? TX_I64 : s->kdt == VB_F64 ? TX_F64 : TX_NONE;
    auto clk = std::chrono::steady_clock::now();
    // 1. local sort
    Gathered g;
    TRY(gather_maps(s, &g));
    const bool has_val = g.rows != nullptr || g.vals != nullptr;
    TRY(seal_sort(s, g));
    const u64 n_local = g.n;
    u64 *lk = s->res_keys, *lv = s->res_comb;
    s->res_keys = s->res_comb = nullptr; s->n_keys = 0;
    DevBuf lk_guard(c), lv_guard(c);
    lk_guard.p = lk; lv_guard.p = lv;
    // every rank must agree on whether a payload travels (a rank with zero rows has no way to know locally)
    s->xst.prepare_wall_ms += lap(clk);
    const u64 c0[2] = {n_local, has_val ? 1ull : 0ull};
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, c0, 2, &mat));
    s->xst.counts_wall_ms += lap(clk);
    u64 N = 0; bool any_val = s->bdist;          // byte-string values: lengths and bytes always travel
    for (u32 r = 0; r < W; ++r) { N += mat[2 * r]; if (mat[2 * r] && mat[2 * r + 1]) any_val = true; }
    // 2. exact cut keys: s_p = the key of global rank c_p - 1, c_p = floor(p N / R); rows with key <= s_p go to partitions < p
    const u32 P = R - 1;
    std::vector<u64> need(P), lo(P, 0), hi(P, ~0ull), cut(R + 1, 0);
    std::vector<char> none(P, 0);
    for (u32 p = 1; p < R; ++p) {
        const u64 cp = (u64)(((unsigned __int128)p * N) / R);
        need[p - 1] = cp;                     // need count_le(v) >= c_p  (i.e. >= (c_p - 1) + 1)
        none[p - 1] = (cp == 0);
    }
    DevBuf d_cand(c), d_cnt(c), d_all(c);
    std::vector<u64> h_all((size_t)W * std::max<u32>(P, 1));
    if (P) {
        TRY(d_cand.alloc((size_t)P * 8)); TRY(d_cnt.alloc((size_t)P * 8)); TRY(d_all.alloc((size_t)W * P * 8));
        std::vector<u64> mid(P);
        for (int round = 0; round <= 64; ++round) {
            const bool final_round = (round == 64);
            for (u32 i = 0; i < P; ++i) mid[i] = final_round ? lo[i] : lo[i] + ((hi[i] - lo[i]) >> 1);
            CU(cudaMemcpyAsync(d_cand.p, mid.data(), (size_t)P * 8, cudaMemcpyHostToDevice, c->stream));
            {
                KLaunch kl(s, K_MISC);
                count_le_kernel<<<(P + 127) / 128, 128, 0, c->stream>>>(lk, n_local, tx, d_cand.as<u64>(), P, d_cnt.as<u64>());
                TRY(kl.done("count_le_kernel"));
            }
            if (final_round) {                 // local cut positions for the agreed cut keys
                CU(cudaMemcpyAsync(h_all.data(), d_cnt.p, (size_t)P * 8, cudaMemcpyDeviceToHost, c->stream));
                CU(cudaStreamSynchronize(c->stream));
                for (u32 i = 0; i < P; ++i) cut[i + 1] = none[i] ? 0 : h_all[i];
                break;
            }
            NC(g_nccl.AllGather(d_cnt.p, d_all.p, P, ncclUint64, m->comm, c->stream));
            CU(cudaMemcpyAsync(h_all.data(), d_all.p, (size_t)W * P * 8, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaStreamSynchronize(c->stream));
            bool open = false;
            for (u32 i = 0; i < P; ++i) {
                u64 tot = 0;
                for (u32 r = 0; r < W; ++r) tot += h_all[(size_t)r * P + i];
                if (tot >= need[i]) hi[i] = mid[i]; else lo[i] = mid[i] + 1;
                open |= lo[i] < hi[i];
            }
            if (!open) round = 63;             // converged everywhere: go to the final round
        }
    }
    cut[0] = 0; cut[R] = n_local;
    for (u32 p = 1; p <= R; ++p) cut[p] = std::max(cut[p], cut[p - 1]);
    // 3. segment sizes of every rank for every partition (byte-string values: then each segment's value bytes, from the
    // pack of the sorted payload)
    const bool bx = s->bdist;
    const u32 SR = bx ? 2 * R : R;
    std::vector<u64> seg(SR), bat;
    for (u32 p = 0; p < R; ++p) seg[p] = cut[p + 1] - cut[p];
    if (bx) {
        TRY(bytes_pack(s, lv, n_local, cut, bat));
        for (u32 p = 0; p < R; ++p) seg[R + p] = bat[p + 1] - bat[p];
    }
    DevBuf d_seg(c), d_segall(c);
    TRY(d_seg.alloc((size_t)SR * 8)); TRY(d_segall.alloc((size_t)W * SR * 8));
    std::vector<u64> segall((size_t)W * SR);
    CU(cudaMemcpyAsync(d_seg.p, seg.data(), (size_t)SR * 8, cudaMemcpyHostToDevice, c->stream));
    NC(g_nccl.AllGather(d_seg.p, d_segall.p, SR, ncclUint64, m->comm, c->stream));
    CU(cudaMemcpyAsync(segall.data(), d_segall.p, (size_t)W * SR * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    // every rank's receive total, so that all ranks refuse alike
    for (u32 d = 0; d < W; ++d) {
        u64 nd = 0;
        for (u32 p = d; p < R; p += W)
            for (u32 r = 0; r < W; ++r) nd += segall[(size_t)r * SR + p];
        if (nd >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "rank %u would receive %llu rows", d, (unsigned long long)nd);
    }
    s->sort_part_rows.assign(R, 0);
    u64 n_recv = 0, nb_recv = 0;
    for (u32 p = me; p < R; p += W)
        for (u32 r = 0; r < W; ++r) {
            s->sort_part_rows[p] += segall[(size_t)r * SR + p];
            n_recv += segall[(size_t)r * SR + p];
            if (bx) nb_recv += segall[(size_t)r * SR + R + p];
        }
    // 4. one grouped send/recv: partition-major, source-rank-major at the receiver
    DevBuf rk(c), rv(c), rl(c), rb(c);
    TRY(rk.alloc(std::max<u64>(n_recv, 1) * 8));
    if (bx) { TRY(rl.alloc(n_recv * 4)); TRY(rb.alloc(nb_recv)); }
    else if (any_val) TRY(rv.alloc(std::max<u64>(n_recv, 1) * 8));
    DevBuf zero_v(c);
    if (any_val && !bx && !lv && n_local) { TRY(zero_v.alloc(n_local * 8)); CU(cudaMemsetAsync(zero_v.p, 0, n_local * 8, c->stream)); lv = zero_v.as<u64>(); }
    std::vector<Xfer> xs;
    u64 sent = 0, own = 0;
    for (u32 p = 0; p < R; ++p) {
        xs.push_back(Xfer{true, p % W, lk + cut[p], seg[p], ncclUint64});
        if (bx) {
            xs.push_back(Xfer{true, p % W, s->bx_lens + cut[p], seg[p], ncclUint32});
            xs.push_back(Xfer{true, p % W, s->bx_bytes + bat[p], seg[R + p], ncclUint8});
        } else if (any_val) xs.push_back(Xfer{true, p % W, lv + cut[p], seg[p], ncclUint64});
        (p % W == me ? own : sent) += seg[p];
    }
    u64 off = 0, boff = 0;
    for (u32 p = me; p < R; p += W)
        for (u32 r = 0; r < W; ++r) {
            const u64 cnt = segall[(size_t)r * SR + p];
            xs.push_back(Xfer{false, r, rk.as<u64>() + off, cnt, ncclUint64});
            if (bx) {
                const u64 nb = segall[(size_t)r * SR + R + p];
                xs.push_back(Xfer{false, r, rl.as<u32>() + off, cnt, ncclUint32});
                xs.push_back(Xfer{false, r, rb.as<unsigned char>() + boff, nb, ncclUint8});
                boff += nb;
            } else if (any_val) xs.push_back(Xfer{false, r, rv.as<u64>() + off, cnt, ncclUint64});
            off += cnt;
        }
    TRY(post_group(s, xs));
    if (bx) TRY(bytes_adopt(s, rl.as<u32>(), n_recv, rb, nb_recv, rv));
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_NCCL, sent, n_recv - own);
    s->imp_own_k = (u64 *)rk.release();
    s->imp_own_v = any_val ? (u64 *)rv.release() : nullptr;
    std::lock_guard<std::mutex> gg(s->mu);
    s->imp_keys = s->imp_own_k; s->imp_vals = s->imp_own_v; s->imp_n = n_recv;
    s->imported = true;
    s->exported = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_exchange(vb_shuf *s, int32_t mode)
{
    if (s && s->rep) return exchange_rep(s, mode);
    if (s && s->vdt == VB_BYTES && !s->bdist) return reject_bytes(s, "vb_shuffle_exchange (the _bytes_dist creates make shuffles that cross ranks)");
    if (s && s->bdist && mode == VB_XCHG_P2P) return reject_bytes(s, "the fused P2P exchange (VB_XCHG_NCCL is supported)");
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (s->multi && s->world < 2) return reject_multi(s, "an exchange of a one-process shuffle (vb_shuffle_create_multi_dist has world > 1)");
    if (s->multi && mode == VB_XCHG_P2P) return reject_multi(s, "the fused P2P exchange (VB_XCHG_NCCL is supported)");
    if (s->str && s->world < 2) return reject_str(s, "an exchange of a one-process shuffle (vb_shuffle_create_str_dist has world > 1)");
    if (s->str && mode == VB_XCHG_P2P) return reject_str(s, "the fused P2P exchange (VB_XCHG_NCCL is supported)");
    vb_ctx *c = s->ctx;
    if (s->world < 2) return set_err(VB_ERR_STATE, "vb_shuffle_exchange needs vb_shuffle_set_dist(world > 1)");
    if (!c->comm) return set_err(VB_ERR_STATE, "vb_shuffle_exchange needs vb_ctx_comm_init");
    if (c->comm->world != s->world || c->comm->rank != s->rank) return set_err(VB_ERR_INVALID, "shuffle rank/world differ from the communicator's");
    if (mode < VB_XCHG_AUTO || mode > VB_XCHG_P2P) return set_err(VB_ERR_INVALID, "bad exchange mode");
    if (s->str || s->multi) {
        std::lock_guard<std::mutex> lk(c->mu);
        CU(cudaSetDevice(c->device));
        return s->str ? (is_reduce_op(s->agg) ? exchange_str_accs_locked(s) : exchange_str_locked(s)) : exchange_multi_locked(s);
    }
    if (mode == VB_XCHG_AUTO) mode = is_group_op(s->agg) && !s->bdist ? VB_XCHG_P2P : VB_XCHG_NCCL;
    if (mode == VB_XCHG_P2P && !is_group_op(s->agg)) return set_err(VB_ERR_UNSUPPORTED, "the fused P2P exchange is for GROUP/COGROUP shuffles");
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    if (s->agg == VB_AGG_SORT) return exchange_sort_locked(s);
    return mode == VB_XCHG_P2P ? exchange_p2p_locked(s) : exchange_nccl_locked(s);
}

extern "C" int32_t vb_shuffle_exchange_stats(vb_shuf *s, vb_xstats *out)
{
    if (!s || !out) return set_err(VB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    cudaSetDevice(s->ctx->device);
    resolve_timers(s);
    *out = s->xst;
    return VB_OK;
}


// ---------------------------------------------------------------------------------------------
// lazy COGROUP + semi-join filter (CoGroupedRdd::compute + join, co_grouped_rdd.rs:206-249 / pair_rdd.rs:104-121)
// The reference cogroups both parents completely and then keeps the keys with values on both sides.  Grouping is the
// expensive part (dictionary + stable sort of every row), and an inner join only needs it for the keys that match:
// for BASELINE configs[3] that is 2 % of the rows.  So seal of a COGROUP shuffle only takes ownership of the rows;
// vb_join* first finds the matching keys (dictionary of the right keys, one probe per left row), compacts both sides
// to the matching rows (stable) and groups just those.  vb_shuffle_reduce* (the cogroup itself) groups everything.
// ---------------------------------------------------------------------------------------------
// take ownership of the gathered rows as SoA (copy when they are borrowed, in the shared arena, or AoS)
static int seal_lazy(vb_shuf *s, const Gathered &g, bool rows_are_owned_imports)
{
    vb_ctx *c = s->ctx;
    const u32 R = s->n_reduce;
    s->bucket_off.assign((size_t)R + 1, 0);
    s->val_off.assign((size_t)R + 1, 0);
    s->lz_n = g.n;
    s->lazy = true;
    if (g.n == 0) return VB_OK;
    if (rows_are_owned_imports) {                      // NCCL receive buffers: just keep them
        s->lz_keys = s->imp_own_k; s->lz_vals = s->imp_own_v;
        s->imp_own_k = s->imp_own_v = nullptr;
        return VB_OK;
    }
    if (!g.rows && g.keys == s->gath_keys && s->gath_keys) {   // gather_maps already made owned SoA copies
        s->lz_keys = s->gath_keys; s->lz_vals = s->gath_vals;
        s->gath_keys = s->gath_vals = nullptr;
        return VB_OK;
    }
    DevBuf k(c), v(c);
    TRY(k.alloc(g.n * 8));
    if (g.rows) {
        TRY(v.alloc(g.n * 8));
        KLaunch kl(s, K_MISC);
        u64 blocks = std::min<u64>((g.n + 255) / 256, (u64)c->sm_count * 8);
        aos_to_soa_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(g.rows, g.n, k.as<u64>(), v.as<u64>());
        TRY(kl.done("aos_to_soa_kernel"));
    } else {
        CU(cudaMemcpyAsync(k.p, g.keys, g.n * 8, cudaMemcpyDeviceToDevice, c->stream));
        if (g.vals) { TRY(v.alloc(g.n * 8)); CU(cudaMemcpyAsync(v.p, g.vals, g.n * 8, cudaMemcpyDeviceToDevice, c->stream)); }
    }
    s->lz_keys = (u64 *)k.release();
    s->lz_vals = (u64 *)v.release();
    return VB_OK;
}

static void free_lazy_rows(vb_shuf *s)
{
    dev_free(s->ctx, s->lz_keys); dev_free(s->ctx, s->lz_vals);
    s->lz_keys = s->lz_vals = nullptr;
}

// group everything (caller holds c->mu)
static int ensure_grouped(vb_shuf *s)
{
    if (!s->lazy) return VB_OK;
    Gathered g;
    g.keys = s->lz_keys; g.vals = s->lz_vals; g.n = s->lz_n;
    TRY(seal_group(s, g));
    CU(cudaStreamSynchronize(s->ctx->stream));
    free_lazy_rows(s);
    s->lazy = false;
    return VB_OK;
}

// match[i] = 1 iff keys[i] is in the dictionary; its slot is marked in slot_flag
__global__ void semi_probe_kernel(const u64 *__restrict__ keys, u64 n, Table t, unsigned char *__restrict__ slot_flag, unsigned char *__restrict__ match)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 st = (u64)gridDim.x * blockDim.x;
    const u64 pol = policy_evict_first();
    for (; i < n; i += st) {
        const u32 sl = table_find(t, ld_stream_u64(keys + i, pol));
        const bool hit = sl != 0xFFFFFFFFu;
        match[i] = hit ? 1 : 0;
        if (hit) slot_flag[sl] = 1;
    }
}
__global__ void mark_rows_kernel(const u32 *__restrict__ slot_of_row, u64 n, const unsigned char *__restrict__ slot_flag, unsigned char *__restrict__ match)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 st = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += st) match[i] = slot_flag[slot_of_row[i]];
}

// stable compaction, 4096 rows per block: counts, scan, scatter
constexpr int CP_THREADS = 256, CP_ITEMS = 16, CP_TILE = CP_THREADS * CP_ITEMS;
__global__ void __launch_bounds__(CP_THREADS) compact_count_kernel(const unsigned char *__restrict__ match, u64 n, u64 *__restrict__ block_cnt)
{
    __shared__ u32 ws[CP_THREADS / 32];
    const u64 base = (u64)blockIdx.x * CP_TILE + (u64)threadIdx.x * CP_ITEMS;
    u32 c = 0;
#pragma unroll
    for (int i = 0; i < CP_ITEMS; ++i) c += (base + i < n) ? match[base + i] : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) { u32 t = 0; for (int w = 0; w < CP_THREADS / 32; ++w) t += ws[w]; block_cnt[blockIdx.x] = t; }
}
__global__ void __launch_bounds__(CP_THREADS)
compact_scatter_kernel(const unsigned char *__restrict__ match, u64 n, const u64 *__restrict__ block_off, const u64 *__restrict__ keys,
                       const u64 *__restrict__ vals, u64 *__restrict__ out_keys, u64 *__restrict__ out_vals)
{
    __shared__ u32 ws[CP_THREADS / 32];
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const u64 base = (u64)blockIdx.x * CP_TILE + (u64)tid * CP_ITEMS;
    unsigned char m[CP_ITEMS];
    u32 c = 0;
#pragma unroll
    for (int i = 0; i < CP_ITEMS; ++i) { m[i] = (base + i < n) ? match[base + i] : 0; c += m[i]; }
    u32 incl = c;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) { const u32 t = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= (u32)off) incl += t; }
    if (lane == 31) ws[warp] = incl;
    __syncthreads();
    u32 wbase = 0;
    for (u32 w = 0; w < warp; ++w) wbase += ws[w];
    u64 o = block_off[blockIdx.x] + wbase + incl - c;
#pragma unroll
    for (int i = 0; i < CP_ITEMS; ++i)
        if (m[i]) { out_keys[o] = keys[base + i]; if (out_vals) out_vals[o] = vals ? vals[base + i] : 0ull; ++o; }
}

static int exclusive_scan_u64(vb_shuf *s, const u64 *in, u64 *out, u64 n, u64 *d_total);

// keys_to: write the kept keys there (room for every kept key) instead of into ok
static int compact_rows(vb_shuf *s, const u64 *keys, const u64 *vals, u64 n, const unsigned char *match, DevBuf &ok, DevBuf &ov, u64 *m_out,
                        u64 *keys_to = nullptr)
{
    vb_ctx *c = s->ctx;
    *m_out = 0;
    if (n == 0) return VB_OK;
    const u64 blocks = (n + CP_TILE - 1) / CP_TILE;
    DevBuf cnt(c), off(c), tot(c);
    TRY(cnt.alloc(blocks * 8)); TRY(off.alloc(blocks * 8)); TRY(tot.alloc(8));
    {
        KLaunch kl(s, K_JOIN);
        compact_count_kernel<<<(unsigned)blocks, CP_THREADS, 0, c->stream>>>(match, n, cnt.as<u64>());
        TRY(kl.done("compact_count_kernel"));
    }
    TRY(exclusive_scan_u64(s, cnt.as<u64>(), off.as<u64>(), blocks, tot.as<u64>()));
    u64 m = 0;
    CU(cudaMemcpyAsync(c->h_scratch, tot.p, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    m = *(u64 *)c->h_scratch;
    *m_out = m;
    if (m == 0) return VB_OK;
    if (!keys_to) { TRY(ok.alloc(m * 8)); keys_to = ok.as<u64>(); }
    TRY(ov.alloc(m * 8));
    KLaunch kl(s, K_JOIN);
    compact_scatter_kernel<<<(unsigned)blocks, CP_THREADS, 0, c->stream>>>(match, n, off.as<u64>(), keys, vals, keys_to, ov.as<u64>());
    return kl.done("compact_scatter_kernel");
}

static vb_shuf *make_internal_like(const vb_shuf *s)
{
    vb_shuf *t = new vb_shuf();
    t->uid = next_uid.fetch_add(1);                 // N-way plans are cached by the sides' uids
    t->ctx = s->ctx; t->id = s->id; t->n_map = 0; t->n_reduce = s->n_reduce;
    t->kdt = s->kdt; t->vdt = s->vdt; t->agg = s->agg; t->part = s->part; t->key_width = s->key_width;
    t->vorder = s->vorder;                          // a filtered join's sides read their lists in the user shuffle's order
    t->internal = true;
    t->rank = 0; t->world = 1;                      // internal shuffles are device-local
    t->sealed = true;
    return t;
}

extern "C" int32_t vb_shuffle_free(vb_shuf *s);

// both sides lazy: internal (left, right) shuffles grouped over the rows the join kind needs.  A side the kind
// preserves (LEFT: the left, RIGHT: the right, FULL: both) keeps every row; any other side keeps the rows whose key
// occurs on both sides.
static int filtered_pair(vb_shuf *l, vb_shuf *r, int kind, vb_shuf **fl_out, vb_shuf **fr_out)
{
    const auto cache_key = std::make_pair(r->uid, kind);
    auto it = l->filtered.find(cache_key);
    if (it != l->filtered.end()) { *fl_out = it->second.first; *fr_out = it->second.second; return VB_OK; }
    vb_ctx *c = l->ctx;
    vb_shuf *fl = make_internal_like(l), *fr = make_internal_like(r);
    auto fail = [&](int rc) { delete fl; delete fr; return rc; };
    fl->bucket_off.assign((size_t)l->n_reduce + 1, 0); fl->val_off = fl->bucket_off;
    fr->bucket_off = fl->bucket_off; fr->val_off = fl->bucket_off;
    const bool all_l = kind == JK_LEFT || kind == JK_FULL, all_r = kind == JK_RIGHT || kind == JK_FULL;
    Gathered gl, gr;                                // the rows each internal shuffle groups
    DevBuf lk(c), lv(c), rk(c), rv(c);
    if (all_l) { gl.keys = l->lz_keys; gl.vals = l->lz_vals; gl.n = l->lz_n; }
    if (all_r) { gr.keys = r->lz_keys; gr.vals = r->lz_vals; gr.n = r->lz_n; }
    u64 cap = 0;
    int rc = VB_OK;
    if (l->lz_n && r->lz_n && !(all_l && all_r)) {
        // 1. dictionary of the right keys (slot per right row)
        DevBuf ids_r(c);
        if ((rc = ids_r.alloc(r->lz_n * 4))) return fail(rc);
        std::vector<AggInput> in(1);
        in[0] = AggInput{IN_SOA, r->lz_keys, nullptr, r->lz_n, VB_DEVICE};
        void *tab = nullptr; u32 log_cap = 0; u64 n_ins = 0;
        if ((rc = build_table(l, K_DICT, in, OPK_DICT, TX_NONE, r->hint, &tab, &log_cap, &n_ins, ids_r.as<u32>()))) return fail(rc);
        DevBuf tab_guard(c); tab_guard.p = tab;
        cap = 1ull << log_cap;
        // 2. probe with every left row; 3. mark the right rows whose key matched
        DevBuf slot_flag(c), ml(c), mr(c);
        if ((rc = slot_flag.alloc(cap + 1 + 16)) || (rc = ml.alloc(l->lz_n)) || (rc = mr.alloc(r->lz_n))) return fail(rc);
        cudaMemsetAsync(slot_flag.p, 0, cap + 1 + 16, c->stream);
        {
            KLaunch kl(l, K_JOIN);
            const unsigned g = (unsigned)std::min<u64>((l->lz_n + 255) / 256, (u64)c->sm_count * 16);
            semi_probe_kernel<<<g, 256, 0, c->stream>>>(l->lz_keys, l->lz_n, table_at(tab, log_cap), slot_flag.as<unsigned char>(), ml.as<unsigned char>());
            if ((rc = kl.done("semi_probe_kernel"))) return fail(rc);
        }
        if (!all_r) {
            KLaunch kl(l, K_JOIN);
            const unsigned g = (unsigned)std::min<u64>((r->lz_n + 255) / 256, (u64)c->sm_count * 16);
            mark_rows_kernel<<<g, 256, 0, c->stream>>>(ids_r.as<u32>(), r->lz_n, slot_flag.as<unsigned char>(), mr.as<unsigned char>());
            if ((rc = kl.done("mark_rows_kernel"))) return fail(rc);
        }
        // 4. stable compaction of the side(s) the kind does not preserve, then the ordinary cogroup of what is left
        if (!all_l) {
            if ((rc = compact_rows(l, l->lz_keys, l->lz_vals, l->lz_n, ml.as<unsigned char>(), lk, lv, &gl.n))) return fail(rc);
            gl.keys = lk.as<u64>(); gl.vals = lv.as<u64>();
        }
        if (!all_r) {
            if ((rc = compact_rows(l, r->lz_keys, r->lz_vals, r->lz_n, mr.as<unsigned char>(), rk, rv, &gr.n))) return fail(rc);
            gr.keys = rk.as<u64>(); gr.vals = rv.as<u64>();
        }
    }
    if (gl.n || gr.n) {
        if ((gl.n && (rc = seal_group(fl, gl))) || (gr.n && (rc = seal_group(fr, gr)))) {
            l->trash.push_back(fl); l->trash.push_back(fr);      // freed with l (vb_shuffle_free would re-lock the context here)
            return rc;
        }
        // kernel counters of the internal shuffles belong to the caller's statistics
        for (int k = 0; k < K_N; ++k) { l->klaunch[k] += fl->klaunch[k] + fr->klaunch[k]; }
        l->st.kernel_launches += fl->st.kernel_launches + fr->st.kernel_launches;
        l->st.table_slots = std::max<u64>(l->st.table_slots, std::max<u64>(cap, std::max(fl->st.table_slots, fr->st.table_slots)));
    }
    cudaStreamSynchronize(c->stream);
    l->filtered[cache_key] = std::make_pair(fl, fr);
    *fl_out = fl; *fr_out = fr;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_seal(vb_shuf *s)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    vb_ctx *c = s->ctx;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->freed) return set_err(VB_ERR_STATE, "seal of a freed shuffle");
        if (s->sealed) return VB_OK;
    }
    {
        std::unique_lock<std::mutex> g(s->mu);
        if (s->sealing) {           // concurrent seal: wait for the one in flight
            ++s->waiters;
            s->cv.wait(g, [&] { return !s->sealing || s->freed; });
            --s->waiters;
            s->cv.notify_all();
            if (s->sealed) return VB_OK;
            return set_err(VB_ERR_STATE, "shuffle %llu: the concurrent seal failed or the shuffle was freed", (unsigned long long)s->id);
        }
        if (s->sealed) return VB_OK;
        s->sealing = true;
    }
    int rc = VB_OK;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        cudaSetDevice(c->device);
        KLaunch call(s, -2);
        auto body = [&]() -> int {
            if (s->rep) {
                if (s->world == 1) TRY(seal_rep(s));
                else if (!s->exported) return set_err(VB_ERR_STATE, "shuffle %llu: a multi-rank repartition is sealed after vb_shuffle_exchange", (unsigned long long)s->id);
            } else if (s->world == 1) {
                for (u32 m = 0; m < s->n_map; ++m)
                    if (!s->maps[m].present) return set_err(VB_ERR_STATE, "shuffle %llu sealed but map %u was never submitted", (unsigned long long)s->id, m);
                if (s->str) {
                    TRY(seal_str(s));
                } else if (is_reduce_op(s->agg)) {
                    void *tab = nullptr; u32 log_cap = 0; u64 n_ins = 0;
                    TRY(merge_map_tables(s, &tab, &log_cap, &n_ins));
                    DevBuf guard(c); guard.p = tab;
                    TRY(finalize_reduce(s, tab, log_cap, n_ins));
                } else {
                    Gathered g;
                    TRY(gather_maps(s, &g));
                    if (s->agg == VB_AGG_SORT) TRY(seal_sort(s, g));
                    else if (s->agg == VB_AGG_COGROUP) TRY(seal_lazy(s, g, false));
                    else TRY(seal_group(s, g));
                }
            } else {
                if (!s->exported || !s->imported) return set_err(VB_ERR_STATE, "world > 1: seal needs export_prepare + import");
                if (s->str) {
                    TRY(seal_str_import(s));
                } else if (is_reduce_op(s->agg)) {
                    void *tab = nullptr; u32 log_cap = 0; u64 n_ins = 0;
                    if (s->imp_n) {
                        std::vector<AggInput> in(1);
                        in[0] = AggInput{s->multi ? IN_ACCS : IN_SOA, s->imp_keys, s->imp_vals, s->imp_n, VB_DEVICE};
                        TRY(build_table(s, K_MERGE, in, merge_opk(s), TX_NONE, s->hint, &tab, &log_cap, &n_ins, nullptr,
                                        s->multi ? &s->acc_imp : nullptr));
                    }
                    DevBuf guard(c); guard.p = tab;
                    TRY(finalize_reduce(s, tab, log_cap, n_ins));
                } else if (s->agg == VB_AGG_SORT) {
                    if (s->sort_part_rows.size() != s->n_reduce) return set_err(VB_ERR_STATE, "multi-rank sort_by_key goes through vb_shuffle_exchange");
                    Gathered g;
                    g.keys = s->imp_keys; g.vals = s->imp_vals; g.n = s->imp_n;
                    TRY(seal_sort(s, g));        // the received runs are key-range disjoint per partition: one stable sort orders them all
                    s->bucket_off.assign((size_t)s->n_reduce + 1, 0);
                    for (u32 p = 0; p < s->n_reduce; ++p) s->bucket_off[p + 1] = s->bucket_off[p] + s->sort_part_rows[p];
                } else {
                    Gathered g;
                    g.keys = s->imp_keys; g.vals = s->imp_vals; g.n = s->imp_n;
                    if (s->agg == VB_AGG_COGROUP) TRY(seal_lazy(s, g, s->imp_keys == s->imp_own_k && s->imp_own_k));
                    else TRY(seal_group(s, g));
                }
            }
            release_inputs(s);
            CU(cudaStreamSynchronize(c->stream));
            return VB_OK;
        };
        rc = body();
        call.done("seal");
    }
    std::lock_guard<std::mutex> g(s->mu);
    if (rc == VB_OK) s->sealed = true; else s->failed = true;
    s->sealing = false;
    s->cv.notify_all();
    return rc;
}

extern "C" int32_t vb_shuffle_is_sealed(vb_shuf *s) { return s && s->sealed ? 1 : 0; }

static int wait_sealed(vb_shuf *s, bool rep_call = false)
{
    if (s->rep && !rep_call) return reject_rep(s, "an integer-key reduce, join, cogroup or blob call");
    std::unique_lock<std::mutex> g(s->mu);
    ++s->waiters;
    s->cv.wait(g, [&] { return s->sealed || s->failed || s->freed; });
    --s->waiters;
    const bool ok = s->sealed && !s->freed;
    const unsigned long long id = s->id;
    s->cv.notify_all();            // vb_shuffle_free waits for waiters == 0 (s may be deleted once g is released)
    g.unlock();
    if (!ok) return set_err(VB_ERR_STATE, "shuffle %llu failed or was freed before it was sealed", id);
    return VB_OK;
}

extern "C" int32_t vb_shuffle_reduce_size(vb_shuf *s, uint32_t r, uint64_t *n_keys, uint64_t *n_vals)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (s->str) return invalid_str(s, "vb_shuffle_reduce_size (read it with vb_shuffle_reduce_str_size)");
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    TRY(wait_sealed(s));
    if (s->lazy) {                                   // first cogroup materialisation: group all rows now
        std::lock_guard<std::mutex> lk(s->ctx->mu);
        CU(cudaSetDevice(s->ctx->device));
        TRY(ensure_grouped(s));
    }
    if (n_keys) *n_keys = s->bucket_off[r + 1] - s->bucket_off[r];
    if (n_vals) *n_vals = is_group_op(s->agg) ? s->val_off[r + 1] - s->val_off[r] : 0;
    return VB_OK;
}

static int copy_out(vb_shuf *s, void *dst, const void *src, size_t bytes, int dst_loc)
{
    if (!dst || !bytes) return VB_OK;
    if (!src) return set_err(VB_ERR_STATE, "result array missing");
    CU(cudaMemcpyAsync(dst, src, bytes, dst_loc == VB_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, s->ctx->stream));
    if (dst_loc == VB_HOST) s->st.d2h_bytes += bytes;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_reduce(vb_shuf *s, uint32_t r, void *out_keys, void *out_combined, uint64_t *out_offsets,
                                     void *out_vals, int32_t dst_loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (s->str) return invalid_str(s, "vb_shuffle_reduce (read it with vb_shuffle_reduce_str)");
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    TRY(wait_sealed(s));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    TRY(ensure_grouped(s));
    const u64 b0 = s->bucket_off[r], nk = s->bucket_off[r + 1] - b0;
    TRY(copy_out(s, out_keys, s->res_keys ? s->res_keys + b0 : nullptr, nk * 8, dst_loc));
    if (is_group_op(s->agg)) {
        const u64 v0 = s->val_off[r], nv = s->val_off[r + 1] - v0;
        if (out_offsets) {
            if (nk == 0) {
                u64 zero = 0;
                CU(cudaMemcpyAsync(out_offsets, &zero, 8, dst_loc == VB_HOST ? cudaMemcpyHostToHost : cudaMemcpyHostToDevice, c->stream));
            } else {
                DevBuf tmp(c);
                TRY(tmp.alloc((nk + 1) * 8));
                KLaunch kl(s, K_MISC);
                rebase_kernel<<<(unsigned)((nk + 1 + 255) / 256), 256, 0, c->stream>>>(s->res_offs + b0, nk + 1, v0, tmp.as<u64>());
                TRY(kl.done("rebase_kernel"));
                TRY(copy_out(s, out_offsets, tmp.p, (nk + 1) * 8, dst_loc));
            }
        }
        TRY(copy_out(s, out_vals, s->res_vals ? s->res_vals + v0 : nullptr, nv * 8, dst_loc));
    } else if (out_combined && s->multi) {
        return set_err(VB_ERR_INVALID, "shuffle %llu has several aggregates per key: read them with vb_shuffle_reduce_cols", (unsigned long long)s->id);
    } else if (out_combined && nk) {
        if (!s->res_comb && s->agg == VB_AGG_SORT) return set_err(VB_ERR_INVALID, "key-only sort has no payload");
        TRY(copy_out(s, out_combined, s->res_comb + b0, nk * 8, dst_loc));
    }
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_reduce_cols(vb_shuf *s, uint32_t r, void *out_keys, void *const *out_aggs, int32_t dst_loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->multi) return set_err(VB_ERR_INVALID, "vb_shuffle_reduce_cols needs a shuffle from vb_shuffle_create_multi");
    if (s->str) return invalid_str(s, "vb_shuffle_reduce_cols (read it with vb_shuffle_reduce_str_cols)");
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    TRY(wait_sealed(s));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    const u64 b0 = s->bucket_off[r], nk = s->bucket_off[r + 1] - b0;
    TRY(copy_out(s, out_keys, s->res_keys ? s->res_keys + b0 : nullptr, nk * 8, dst_loc));
    for (u32 o = 0; out_aggs && o < s->outs.n; ++o)
        TRY(copy_out(s, out_aggs[o], s->res_cols ? s->res_cols + (u64)o * s->n_keys + b0 : nullptr, nk * 8, dst_loc));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// a reduce result as a cogroup / join side without a second shuffle (CoGroupedRdd::new's OneToOneDependency,
// co_grouped_rdd.rs:103-112)
// ---------------------------------------------------------------------------------------------
// Partition r of a reduce result already holds exactly the keys with hash % n_reduce == r, each once, so the view is a
// grouped COGROUP shuffle over the same placement: copies of the keys and of one result column, offsets 0..n (one value
// per key), and the key dictionary the joins probe, built by one narrow_dict_kernel pass (the keys are distinct, so there
// is no hash_agg, no id sort and no CSR build).  The table is keys only: dictionaries never read the accumulator half.
static int narrow_build(vb_shuf *v, const u64 *keys, const u64 *col, u64 n)
{
    vb_ctx *c = v->ctx;
    if (n == 0) return VB_OK;                         // an empty side: no arrays, no dictionary (as seal_group leaves it)
    DevBuf k(c), vals(c), offs(c), ctl(c);
    TRY(k.alloc(n * 8)); TRY(vals.alloc(n * 8)); TRY(offs.alloc((n + 1) * 8)); TRY(ctl.alloc(sizeof(TableCtl)));
    CU(cudaMemcpyAsync(k.p, keys, n * 8, cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaMemcpyAsync(vals.p, col, n * 8, cudaMemcpyDeviceToDevice, c->stream));
    // load <= 0.5 by construction; a probe chain longer than HA_MAX_PROBE buckets restarts the table larger, and at max_log,
    // where it cannot grow, inserts have no probe-round limit (chain_limit), so every insert succeeds
    const u32 max_log = std::min<u32>(MAX_LOG_CAP, std::max<u32>(4, ceil_log2_u64(2 * n)));
    u32 log_cap = choose_log_cap(n, n, false, max_log, c->l2_bytes);
    for (;;) {
        const u64 cap = 1ull << log_cap;
        DevBuf tab(c), dense(c);
        TRY(tab.alloc((cap + BUCKET) * 8));
        TRY(dense.alloc((cap + 1) * 4));
        CU(cudaMemsetAsync(tab.p, 0xFF, cap * 8, c->stream));                 // EMPTY_KEY
        CU(cudaMemsetAsync(tab.as<u64>() + cap, 0, BUCKET * 8, c->stream));   // special-slot marker: absent
        CU(cudaMemsetAsync(ctl.p, 0, sizeof(TableCtl), c->stream));
        {
            KLaunch kl(v, K_DICT, n);
            Table t = table_at(tab.p, log_cap);
            t.max_probe = chain_limit(log_cap < max_log || cap < 2 * n);
            narrow_dict_kernel<<<(unsigned)((n + 1 + 255) / 256), 256, 0, c->stream>>>(k.as<u64>(), n, t, dense.as<u32>(), offs.as<u64>(),
                                                                                      ctl.as<TableCtl>());
            TRY(kl.done("narrow_dict_kernel"));
        }
        TableCtl h;
        TRY(fetch_status_unlocked(c, ctl.p, &h, sizeof(h)));
        if (!h.abort) {
            v->dict = tab.release();
            v->dict_log_cap = log_cap;
            v->dense_of_slot = (u32 *)dense.release();
            v->st.table_slots = cap;
            break;
        }
        if (log_cap >= max_log) return set_err(VB_ERR_CUDA, "key dictionary overflow at maximum capacity 2^%u (internal error)", log_cap);
        log_cap = std::min(max_log, log_cap + 2);
        v->st.table_restarts++;
    }
    v->res_keys = (u64 *)k.release();
    v->res_vals = (u64 *)vals.release();
    v->res_offs = (u64 *)offs.release();
    return VB_OK;
}

extern "C" int32_t vb_shuffle_create_narrow(vb_shuf *p, uint32_t out_col, vb_shuf **out)
{
    if (!p || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_narrow: NULL argument");
    *out = nullptr;
    if (p->str) return invalid_str(p, "vb_shuffle_create_narrow");
    if (!is_reduce_op(p->agg))
        return set_err(VB_ERR_INVALID, "vb_shuffle_create_narrow: shuffle %llu is not a reduce-op or combine_by_key shuffle",
                       (unsigned long long)p->id);
    const u32 n_cols = p->multi ? p->outs.n : 1;
    if (out_col >= n_cols) return set_err(VB_ERR_INVALID, "vb_shuffle_create_narrow: output column %u of %u", out_col, n_cols);
    TRY(wait_sealed(p));
    vb_ctx *c = p->ctx;
    vb_shuf *v = make_internal_like(p);
    v->agg = VB_AGG_COGROUP;
    v->vdt = p->multi ? p->out_dt[out_col] : p->agg == VB_AGG_COUNT ? VB_U64 : p->vdt;
    v->rank = p->rank; v->world = p->world;
    v->bucket_off = p->bucket_off; v->val_off = p->bucket_off;
    v->n_keys = v->n_vals = v->st.rows_out = p->n_keys;
    int rc;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        rc = [&]() -> int {
            CU(cudaSetDevice(c->device));
            const u64 *col = p->multi ? (p->res_cols ? p->res_cols + (u64)out_col * p->n_keys : nullptr) : p->res_comb;
            TRY(narrow_build(v, p->res_keys, col, p->n_keys));
            CU(cudaStreamSynchronize(c->stream));
            return VB_OK;
        }();
    }
    if (rc != VB_OK) { vb_shuffle_free(v); return rc; }
    *out = v;
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// bincode blobs (N1)
// ---------------------------------------------------------------------------------------------
static u64 str_blob_bytes(const vb_shuf *s, u32 r);
static int str_reduce_blob_locked(vb_shuf *s, u32 r, unsigned char *dst);
static int str_map_blob(vb_shuf *s, u32 map_id, const void *blob, u64 n_bytes, int src_loc);
static int str_blob_check(const vb_shuf *s);

static u64 blob_bytes(const vb_shuf *s, u32 r)
{
    if (s->str) return str_blob_bytes(s, r);
    const u64 nk = s->bucket_off[r + 1] - s->bucket_off[r];
    if (is_group_op(s->agg)) return 8 + 16 * nk + 8 * (s->val_off[r + 1] - s->val_off[r]);
    return 8 + 16 * nk;
}

extern "C" int32_t vb_shuffle_reduce_blob_size(vb_shuf *s, uint32_t r, uint64_t *n_bytes)
{
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_reduce_blob_size");
    if (!s || !n_bytes) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "bincode blobs");
    if (s->str) TRY(str_blob_check(s));
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    TRY(wait_sealed(s));
    if (s->lazy) {
        std::lock_guard<std::mutex> lk(s->ctx->mu);
        CU(cudaSetDevice(s->ctx->device));
        TRY(ensure_grouped(s));
    }
    *n_bytes = blob_bytes(s, r);
    return VB_OK;
}

extern "C" int32_t vb_shuffle_reduce_blob(vb_shuf *s, uint32_t r, void *out_blob, int32_t dst_loc)
{
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_reduce_blob");
    if (!s || !out_blob) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "bincode blobs");
    if (s->str) TRY(str_blob_check(s));
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    if (s->str && dst_loc == VB_DEVICE && ((uintptr_t)out_blob & 15))
        return set_err(VB_ERR_INVALID, "a string-key blob's device destination must be 16-byte aligned");
    TRY(wait_sealed(s));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    TRY(ensure_grouped(s));
    const u64 bytes = blob_bytes(s, r);
    const u64 b0 = s->bucket_off[r], nk = s->bucket_off[r + 1] - b0;
    DevBuf tmp(c);
    u64 *dst = (u64 *)out_blob;
    if (dst_loc == VB_HOST) { TRY(tmp.alloc(bytes)); dst = tmp.as<u64>(); }
    const unsigned grid = (unsigned)std::min<u64>(std::max<u64>(1, (std::max(nk, s->val_off[r + 1] - s->val_off[r]) + 255) / 256), (u64)c->sm_count * 8);
    if (s->str) {
        TRY(str_reduce_blob_locked(s, r, (unsigned char *)dst));
    } else {
        KLaunch kl(s, K_MISC);
        if (is_group_op(s->agg)) {
            if (nk) blob_group_kernel<<<grid, 256, 0, c->stream>>>(s->res_keys + b0, s->res_offs + b0, nk, s->res_vals, dst);
            else CU(cudaMemsetAsync(dst, 0, 8, c->stream));
        } else {
            if (nk) blob_pairs_kernel<<<grid, 256, 0, c->stream>>>(s->res_keys + b0, s->res_comb ? s->res_comb + b0 : nullptr, nk, dst);
            else CU(cudaMemsetAsync(dst, 0, 8, c->stream));
        }
        TRY(kl.done("blob kernel"));
    }
    if (dst_loc == VB_HOST) TRY(copy_out(s, out_blob, dst, bytes, VB_HOST));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_map_blob(vb_shuf *s, uint32_t map_id, const void *blob, uint64_t n_bytes, int32_t src_loc)
{
    if (s && s->rep) return reject_rep(s, "vb_shuffle_map_blob");
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_map_blob");
    if (!s || !blob) return set_err(VB_ERR_INVALID, "NULL argument");
    if (s->multi) return reject_multi(s, "bincode blobs");
    if (s->str) {
        TRY(str_blob_check(s));
        if (s->world > 1) return reject_str(s, "vb_shuffle_map_blob across ranks (map tasks cross ranks through the exchange)");
        if (src_loc < VB_HOST || src_loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc");
        return str_map_blob(s, map_id, blob, n_bytes, src_loc);
    }
    if (src_loc < VB_HOST || src_loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc");
    if (s->agg == VB_AGG_SORT) return set_err(VB_ERR_UNSUPPORTED, "sort_by_key takes rows, not combined buckets");
    if (n_bytes < 8 || (n_bytes & 7)) return set_err(VB_ERR_INVALID, "corrupted blob: %llu bytes", (unsigned long long)n_bytes);
    vb_ctx *c = s->ctx;
    // the whole blob on the host: CPU-produced buckets arrive there anyway, and the record structure of
    // Vec<(K,Vec<V>)> is a linked list (each record's position depends on the previous lengths)
    std::vector<u64> host;
    const u64 *w = (const u64 *)blob;
    if (src_loc != VB_HOST) {
        host.resize(n_bytes / 8);
        std::lock_guard<std::mutex> lk(c->mu);
        CU(cudaSetDevice(c->device));
        CU(cudaMemcpyAsync(host.data(), blob, n_bytes, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        w = host.data();
    }
    const u64 words = n_bytes / 8, n = w[0];
    if (!is_group_op(s->agg)) {
        if (n > (words - 1) / 2 || words != 1 + 2 * n) return set_err(VB_ERR_INVALID, "corrupted blob: %llu records in %llu bytes", (unsigned long long)n, (unsigned long long)n_bytes);
        std::vector<u64> k(n), v(n);
        for (u64 i = 0; i < n; ++i) { k[i] = w[1 + 2 * i]; v[i] = w[2 + 2 * i]; }
        return shuffle_map(s, map_id, nullptr, k.data(), v.data(), n, VB_HOST, /*combined=*/true);
    }
    std::vector<u64> k, v;
    u64 pos = 1;
    for (u64 i = 0; i < n; ++i) {
        if (pos + 2 > words) return set_err(VB_ERR_INVALID, "corrupted blob: record %llu runs past the end", (unsigned long long)i);
        const u64 key = w[pos], len = w[pos + 1];
        if (len > words - pos - 2) return set_err(VB_ERR_INVALID, "corrupted blob: record %llu has length %llu", (unsigned long long)i, (unsigned long long)len);
        for (u64 j = 0; j < len; ++j) { k.push_back(key); v.push_back(w[pos + 2 + j]); }
        pos += 2 + len;
    }
    if (pos != words) return set_err(VB_ERR_INVALID, "corrupted blob: %llu trailing bytes", (unsigned long long)((words - pos) * 8));
    return shuffle_map(s, map_id, nullptr, k.data(), v.data(), k.size(), VB_HOST, false);
}

// ---------------------------------------------------------------------------------------------
// join
// ---------------------------------------------------------------------------------------------
static int exclusive_scan_u64(vb_shuf *s, const u64 *in, u64 *out, u64 n, u64 *d_total)
{
    vb_ctx *c = s->ctx;
    if (n == 0) return VB_OK;
    const u64 blocks = (n + SC_CHUNK - 1) / SC_CHUNK;
    if (blocks == 1) {
        KLaunch kl(s, K_JOIN);
        scan_apply_kernel<<<1, SC_THREADS, 0, c->stream>>>(in, out, n, nullptr, d_total);
        return kl.done("scan_apply_kernel");
    }
    DevBuf sums(c), offs(c);
    TRY(sums.alloc(blocks * 8));
    TRY(offs.alloc(blocks * 8));
    {
        KLaunch kl(s, K_JOIN);
        scan_reduce_kernel<<<(unsigned)blocks, SC_THREADS, 0, c->stream>>>(in, n, sums.as<u64>());
        TRY(kl.done("scan_reduce_kernel"));
    }
    TRY(exclusive_scan_u64(s, sums.as<u64>(), offs.as<u64>(), blocks, nullptr));
    KLaunch kl(s, K_JOIN);
    scan_apply_kernel<<<(unsigned)blocks, SC_THREADS, 0, c->stream>>>(in, out, n, offs.as<u64>(), d_total);
    return kl.done("scan_apply_kernel");
}

static int join_check(vb_shuf *l, vb_shuf *r, u32 rid)
{
    if (!l || !r) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (l->str || r->str) return invalid_str(l->str ? l : r, "a join or cogroup");
    if (!is_group_op(l->agg) || !is_group_op(r->agg)) return set_err(VB_ERR_INVALID, "join needs two GROUP/COGROUP shuffles");
    if (l->n_reduce != r->n_reduce || l->key_width != r->key_width) return set_err(VB_ERR_INVALID, "join sides use different partitioners");
    if (l->ctx != r->ctx) return set_err(VB_ERR_INVALID, "join sides live on different contexts");
    if (rid >= l->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", rid, l->n_reduce);
    TRY(wait_sealed(l));
    TRY(wait_sealed(r));
    return VB_OK;
}

static_assert(JK_LEFT == (int)VB_JOIN_LEFT && JK_RIGHT == (int)VB_JOIN_RIGHT && JK_FULL == (int)VB_JOIN_FULL, "join kinds");

// Row counts and output positions of partition rid for an outer kind.  Left-driven rows first: per left key |vs| * |ws|
// when the right side has the key, |vs| when it does not and the kind keeps the left side (LEFT / FULL), else 0.
// RIGHT / FULL then place the right-only keys (|ws| rows each, found by probing the left dictionary); one exclusive
// scan covers both.
static int join_plan(vb_shuf *l, vb_shuf *r, u32 rid, int kind, JoinPlan **out)
{
    vb_ctx *c = l->ctx;
    auto key = std::make_tuple(r->uid, rid, kind);    // by uid: a freed side's address may be reused
    auto it = l->join_plans.find(key);
    if (it != l->join_plans.end()) { *out = &it->second; return VB_OK; }
    JoinPlan p;
    const u64 lb = l->bucket_off[rid], le = l->bucket_off[rid + 1];
    p.nl = (u32)(le - lb);
    const u64 rb = r->bucket_off[rid], re = r->bucket_off[rid + 1];
    p.nr = (kind == JK_LEFT) ? 0 : (u32)(re - rb);
    const u64 n = (u64)p.nl + p.nr;
    if (n) {
        if ((r->n_keys && !r->dict) || (l->n_keys && !l->dict)) return set_err(VB_ERR_STATE, "join side without a key dictionary");
        const Table rtab = table_at(r->n_keys ? r->dict : nullptr, r->dict_log_cap);   // keys NULL: that side is empty
        const Table ltab = table_at(l->n_keys ? l->dict : nullptr, l->dict_log_cap);
        DevBuf cnt(c), pos(c), match(c), tot(c);
        TRY(cnt.alloc(n * 8));
        TRY(pos.alloc(n * 8));
        TRY(match.alloc(std::max<u64>(p.nl, 1) * 4));
        TRY(tot.alloc(8));
        if (p.nl) {
            KLaunch kl(l, K_JOIN);
            const unsigned g = (p.nl + 255) / 256;
            if (kind == JK_LEFT)
                join_probe_kernel<JK_LEFT><<<g, 256, 0, c->stream>>>(l->res_keys, l->res_offs, (u32)lb, (u32)le, rtab, r->dense_of_slot,
                                                                     r->res_offs, cnt.as<u64>(), match.as<u32>());
            else if (kind == JK_RIGHT)
                join_probe_kernel<JK_RIGHT><<<g, 256, 0, c->stream>>>(l->res_keys, l->res_offs, (u32)lb, (u32)le, rtab, r->dense_of_slot,
                                                                      r->res_offs, cnt.as<u64>(), match.as<u32>());
            else
                join_probe_kernel<JK_FULL><<<g, 256, 0, c->stream>>>(l->res_keys, l->res_offs, (u32)lb, (u32)le, rtab, r->dense_of_slot,
                                                                     r->res_offs, cnt.as<u64>(), match.as<u32>());
            TRY(kl.done("join_probe_kernel"));
        }
        if (p.nr) {
            KLaunch kl(l, K_JOIN);
            join_probe_right_kernel<<<(p.nr + 255) / 256, 256, 0, c->stream>>>(r->res_keys, r->res_offs, (u32)rb, (u32)re, ltab,
                                                                               cnt.as<u64>() + p.nl);
            TRY(kl.done("join_probe_right_kernel"));
        }
        TRY(exclusive_scan_u64(l, cnt.as<u64>(), pos.as<u64>(), n, tot.as<u64>()));
        u64 *h = (u64 *)c->h_scratch;
        CU(cudaMemcpyAsync(h, tot.p, 8, cudaMemcpyDeviceToHost, c->stream));
        if (p.nr) CU(cudaMemcpyAsync(h + 1, pos.as<u64>() + p.nl, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        p.total = h[0];
        p.total_left = p.nr ? h[1] : p.total;
        p.pos = (u64 *)pos.release();
        p.match = (u32 *)match.release();
    }
    auto ins = l->join_plans.emplace(key, p);
    *out = &ins.first->second;
    return VB_OK;
}

// the pair of shuffles whose CSR the join reads: the filtered internal pair while both sides are still lazy
static int join_sides(vb_shuf *&l, vb_shuf *&r, int kind)
{
    if (l->lazy && r->lazy && l != r) {
        vb_shuf *fl = nullptr, *fr = nullptr;
        TRY(filtered_pair(l, r, kind, &fl, &fr));
        l = fl; r = fr;
        return VB_OK;
    }
    TRY(ensure_grouped(l));
    TRY(ensure_grouped(r));
    return VB_OK;
}

static int join_size(vb_shuf *l, vb_shuf *r, uint32_t rid, int kind, uint64_t *n_out)
{
    TRY(join_check(l, r, rid));
    if (!n_out) return set_err(VB_ERR_INVALID, "n_out is NULL");
    std::lock_guard<std::mutex> lk(l->ctx->mu);
    CU(cudaSetDevice(l->ctx->device));
    TRY(join_sides(l, r, kind));
    JoinPlan *p = nullptr;
    TRY(join_plan(l, r, rid, kind, &p));
    *n_out = p->total;
    return VB_OK;
}

static int join_rows(vb_shuf *l, vb_shuf *r, uint32_t rid, int kind, void *out_k, void *out_v, void *out_w,
                     uint8_t *out_vv, uint8_t *out_wv, int32_t dst_loc)
{
    TRY(join_check(l, r, rid));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_ctx *c = l->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    TRY(join_sides(l, r, kind));
    JoinPlan *p = nullptr;
    TRY(join_plan(l, r, rid, kind, &p));
    const u64 total = p->total;
    int rc = VB_OK;
    if (total) {
        if (!out_k || !out_v || !out_w) return set_err(VB_ERR_INVALID, "NULL output with %llu rows to write", (unsigned long long)total);
        DevBuf bk(c), bv(c), bw(c), bvv(c), bwv(c);
        u64 *dk = (u64 *)out_k, *dv = (u64 *)out_v, *dw = (u64 *)out_w;
        unsigned char *dvv = out_vv, *dwv = out_wv;
        if (dst_loc == VB_HOST) {
            TRY(bk.alloc(total * 8)); TRY(bv.alloc(total * 8)); TRY(bw.alloc(total * 8));
            dk = bk.as<u64>(); dv = bv.as<u64>(); dw = bw.as<u64>();
            if (out_vv) { TRY(bvv.alloc(total)); dvv = bvv.as<unsigned char>(); }
            if (out_wv) { TRY(bwv.alloc(total)); dwv = bwv.as<unsigned char>(); }
        }
        const u64 lb = l->bucket_off[rid];
        const u64 total_left = p->total_left;
        if (total_left) {
            KLaunch kl(l, K_JOIN);
            u64 blocks = std::min<u64>((total_left + 255) / 256, (u64)c->sm_count * 8);
#define VB_JOIN_EXPAND(KIND) join_expand_kernel<KIND><<<(unsigned)blocks, 256, 0, c->stream>>>(p->pos, p->nl, total_left, l->res_keys, \
                                 l->res_offs, l->res_vals, (u32)lb, p->match, r->res_offs, r->res_vals, dk, dv, dw, dvv, dwv)
            switch (kind) {
            case JK_LEFT: VB_JOIN_EXPAND(JK_LEFT); break;
            case JK_RIGHT: VB_JOIN_EXPAND(JK_RIGHT); break;
            default: VB_JOIN_EXPAND(JK_FULL); break;
            }
#undef VB_JOIN_EXPAND
            rc = kl.done("join_expand_kernel");
        }
        if (rc == VB_OK && total > total_left) {
            KLaunch kl(l, K_JOIN);
            u64 blocks = std::min<u64>((total - total_left + 255) / 256, (u64)c->sm_count * 8);
            join_expand_right_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(p->pos + p->nl, p->nr, total, r->res_keys, r->res_offs,
                                                                              r->res_vals, (u32)r->bucket_off[rid], dk, dv, dw, dvv, dwv);
            rc = kl.done("join_expand_right_kernel");
        }
        if (rc == VB_OK && dst_loc == VB_HOST) {
            rc = copy_out(l, out_k, dk, total * 8, VB_HOST);
            if (rc == VB_OK) rc = copy_out(l, out_v, dv, total * 8, VB_HOST);
            if (rc == VB_OK) rc = copy_out(l, out_w, dw, total * 8, VB_HOST);
            if (rc == VB_OK) rc = copy_out(l, out_vv, dvv, total, VB_HOST);
            if (rc == VB_OK) rc = copy_out(l, out_wv, dwv, total, VB_HOST);
        }
        cudaStreamSynchronize(c->stream);
    }
    dev_free(c, p->pos);
    dev_free(c, p->match);
    l->join_plans.erase(std::make_tuple(r->uid, rid, kind));
    return rc;
}

static bool outer_kind(int32_t kind) { return kind == VB_JOIN_LEFT || kind == VB_JOIN_RIGHT || kind == VB_JOIN_FULL; }

extern "C" int32_t vb_join_outer_size(vb_shuf *l, vb_shuf *r, uint32_t rid, int32_t kind, uint64_t *n_out)
{
    if (!outer_kind(kind)) return set_err(VB_ERR_INVALID, "bad join kind %d", kind);
    return join_size(l, r, rid, kind, n_out);
}

extern "C" int32_t vb_join_outer(vb_shuf *l, vb_shuf *r, uint32_t rid, int32_t kind, void *out_k, void *out_v, void *out_w,
                                 uint8_t *out_v_valid, uint8_t *out_w_valid, int32_t dst_loc)
{
    if (!outer_kind(kind)) return set_err(VB_ERR_INVALID, "bad join kind %d", kind);
    return join_rows(l, r, rid, kind, out_k, out_v, out_w, out_v_valid, out_w_valid, dst_loc);
}

// ---------------------------------------------------------------------------------------------
// cogroup and inner join of n sides (CoGroupedRdd::compute with n parents, co_grouped_rdd.rs:206-249)
// Side i's keys are probed against every other side's dictionary by one launch per side (all sides' tables in one
// parameter struct): a key no earlier side has is new, and its row of the match matrix records its index on every side.
// The output keys are side 0's, then each later side's new keys taken by the stable compaction.  Side 0's lists are its
// partition's value slice as it is; side j's lists are its value segments gathered into output key order.  The join
// reads side 0's rows of the matrix only: the keys on every side are exactly the side-0 keys without a 0xFFFFFFFF.
// vb_cogroup_n* / vb_join_n* group every side whole.  vb_cogroup* / vb_join* are the two-side case over the pair
// join_sides picks: the FULL (cogroup) or INNER (join) filtered pair while both sides are still lazy.
// ---------------------------------------------------------------------------------------------
static_assert(CGN_MAX_SIDES == VB_MAX_COGROUP_SIDES, "cogroup side limit");

static void free_cogroup_n_plan(vb_ctx *c, CogroupNPlan &p)
{
    dev_free(c, p.new_keys); dev_free(c, p.match); dev_free(c, p.pos);
    dev_free(c, p.str_sel); dev_free(c, p.str_koff); dev_free(c, p.str_roff);
}

static int str_n_sides(vb_shuf *const *sides, u32 n, u32 rid, StrNSides *a);

// vb_cogroup's argument rules for every side; waits until every side is sealed
static int cogroup_n_check(vb_shuf *const *sides, u32 n, u32 rid)
{
    if (!sides) return set_err(VB_ERR_INVALID, "sides is NULL");
    if (n < 1 || n > VB_MAX_COGROUP_SIDES) return set_err(VB_ERR_INVALID, "n_sides %u is not in [1, %d]", n, VB_MAX_COGROUP_SIDES);
    for (u32 j = 0; j < n; ++j) {
        const vb_shuf *s = sides[j];
        if (!s) return set_err(VB_ERR_INVALID, "side %u is NULL", j);
        if (s->str) return invalid_str(s, "a join or cogroup");
        if (!is_group_op(s->agg)) return set_err(VB_ERR_INVALID, "side %u is not a GROUP/COGROUP shuffle", j);
        if (s->n_reduce != sides[0]->n_reduce || s->key_width != sides[0]->key_width)
            return set_err(VB_ERR_INVALID, "side %u uses a different partitioner than side 0", j);
        if (s->ctx != sides[0]->ctx) return set_err(VB_ERR_INVALID, "side %u lives on a different context than side 0", j);
    }
    if (rid >= sides[0]->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", rid, sides[0]->n_reduce);
    for (u32 j = 0; j < n; ++j) TRY(wait_sealed(sides[j]));
    return VB_OK;
}

// describe the grouped sides for the kernels
static int cogroup_n_sides(vb_shuf *const *sides, u32 n, u32 rid, CogroupNSides *a)
{
    *a = CogroupNSides{};
    a->n = n;
    for (u32 j = 0; j < n; ++j) {
        const vb_shuf *s = sides[j];
        if (s->n_keys && !s->dict && !s->str) return set_err(VB_ERR_STATE, "cogroup side without a key dictionary");
        a->tab[j] = table_at(s->n_keys ? s->dict : nullptr, s->dict_log_cap);
        a->dense[j] = s->dense_of_slot;
        a->keys[j] = s->res_keys; a->offs[j] = s->res_offs; a->vals[j] = s->res_vals;
        a->kb[j] = (u32)s->bucket_off[rid];
    }
    return VB_OK;
}

// kind: NP_COGROUP, NP_INNER, or an outer join's mask of required sides
static int cogroup_n_plan(vb_shuf *const *sides, u32 n, u32 rid, i64 kind, const CogroupNSides &a, CogroupNPlan **out)
{
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    std::vector<u64> uids(n);
    for (u32 j = 0; j < n; ++j) uids[j] = sides[j]->uid;
    auto key = std::make_tuple(uids, rid, kind);
    auto it = s0->n_plans.find(key);
    if (it != s0->n_plans.end()) { *out = &it->second; return VB_OK; }
    const bool join = kind != NP_COGROUP;
    // a join that requires side 0 has rows only for side 0's keys; every other plan takes the union of the keys
    const bool all_keys = kind == NP_COGROUP || (kind >= 0 && !(kind & 1));
    std::vector<u64> nk(n);
    u64 cap = 0;                                       // output keys at most
    for (u32 j = 0; j < n && (j == 0 || all_keys); ++j) {
        nk[j] = sides[j]->bucket_off[rid + 1] - sides[j]->bucket_off[rid];
        cap += nk[j];
    }
    if (cap >= 0xFFFFFFFFull) return set_err(VB_ERR_TOO_LARGE, "%llu keys in one cogroup partition", (unsigned long long)cap);
    CogroupNPlan p;
    DevBuf match(c), new_keys(c), pos(c);
    TRY(match.alloc(cap * n * 4));
    // string sides: the lookup reads each side's key index (the keys themselves are written from the match rows)
    const bool str = s0->str != nullptr;
    StrNSides sa;
    if (str) TRY(str_n_sides(sides, n, rid, &sa));
    auto probe = [&](u32 i, u32 *rows, unsigned char *flag, u64 *lidx) -> int {
        KLaunch kl(s0, K_JOIN);
        const unsigned g = (unsigned)((nk[i] + 255) / 256);
        if (str) {
            cogroup_n_str_probe_kernel<<<g, 256, 0, c->stream>>>(sa, i, (u32)nk[i], rows, flag, lidx);
            return kl.done("cogroup_n_str_probe_kernel");
        }
        cogroup_n_probe_kernel<<<g, 256, 0, c->stream>>>(a, i, (u32)nk[i], rows, flag, lidx);
        return kl.done("cogroup_n_probe_kernel");
    };
    if (nk[0]) TRY(probe(0, match.as<u32>(), nullptr, nullptr));
    p.n_keys = nk[0];
    if (all_keys && cap > nk[0]) {
        if (!str) TRY(new_keys.alloc((cap - nk[0]) * 8));
        for (u32 i = 1; i < n; ++i) {
            if (!nk[i]) continue;
            DevBuf rows(c), flag(c), lidx(c), ok(c), ov(c);
            TRY(rows.alloc(i + 1 < n ? nk[i] * n * 4 : 0)); TRY(flag.alloc(nk[i])); TRY(lidx.alloc(nk[i] * 8));
            TRY(probe(i, rows.as<u32>(), flag.as<unsigned char>(), lidx.as<u64>()));
            u64 m = 0;
            if (str)      // no key values: only the new keys' local indices (ov) are kept
                TRY(compact_rows(s0, lidx.as<u64>(), lidx.as<u64>(), nk[i], flag.as<unsigned char>(), ok, ov, &m));
            else
                TRY(compact_rows(s0, sides[i]->res_keys + a.kb[i], lidx.as<u64>(), nk[i], flag.as<unsigned char>(), ok, ov, &m,
                                 new_keys.as<u64>() + (p.n_keys - nk[0])));
            if (!m) continue;
            {
                KLaunch kl(s0, K_JOIN);
                const u64 blocks = std::min<u64>((m * n + 255) / 256, (u64)c->sm_count * 8);
                cogroup_n_take_rows_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(rows.as<u32>(), n, i, a.kb[i], ov.as<u64>(), m,
                                                                                    match.as<u32>() + p.n_keys * n);
                TRY(kl.done("cogroup_n_take_rows_kernel"));
            }
            p.n_keys += m;
        }
    }
    if (join && p.n_keys) {
        DevBuf cnt(c), flags(c);
        TRY(cnt.alloc(p.n_keys * 8)); TRY(pos.alloc(p.n_keys * 8)); TRY(flags.alloc(24));
        CU(cudaMemsetAsync(flags.p, 0, 24, c->stream));
        unsigned long long *sums = flags.as<unsigned long long>();
        u32 *too_large = (u32 *)(sums + 2);
        if (kind == NP_INNER) {
            KLaunch kl(s0, K_JOIN);
            join_n_count_kernel<<<(unsigned)((p.n_keys + 255) / 256), 256, 0, c->stream>>>(a, match.as<u32>(), (u32)p.n_keys,
                                                                                          cnt.as<u64>(), sums, too_large);
            TRY(kl.done("join_n_count_kernel"));
        } else {
            KLaunch kl(s0, K_JOIN);
            join_n_outer_count_kernel<<<(unsigned)((p.n_keys + 255) / 256), 256, 0, c->stream>>>(
                a, match.as<u32>(), (u32)p.n_keys, (u32)kind, cnt.as<u64>(), sums, too_large);
            TRY(kl.done("join_n_outer_count_kernel"));
        }
        TRY(exclusive_scan_u64(s0, cnt.as<u64>(), pos.as<u64>(), p.n_keys, nullptr));
        u64 *h = (u64 *)c->h_scratch;
        CU(cudaMemcpyAsync(h, flags.p, 24, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        const unsigned __int128 total = ((unsigned __int128)h[0] << 32) + h[1];
        if (*(u32 *)(h + 2) || total >> 63)
            return set_err(VB_ERR_TOO_LARGE, "partition %u of the join has 2^63 rows or more", rid);
        p.total = (u64)total;
    }
    CU(cudaStreamSynchronize(c->stream));
    p.match = (u32 *)match.release();
    p.new_keys = (u64 *)new_keys.release();
    p.pos = (u64 *)pos.release();
    *out = &s0->n_plans.emplace(key, p).first->second;
    return VB_OK;
}

static void drop_cogroup_n_plan(vb_shuf *const *sides, u32 n, u32 rid, i64 kind)
{
    std::vector<u64> uids(n);
    for (u32 j = 0; j < n; ++j) uids[j] = sides[j]->uid;
    auto it = sides[0]->n_plans.find(std::make_tuple(uids, rid, kind));
    if (it == sides[0]->n_plans.end()) return;
    free_cogroup_n_plan(sides[0]->ctx, it->second);
    sides[0]->n_plans.erase(it);
}

// The plan and the write of a cogroup / inner join, over sides that are grouped, with the context locked

static int cogroup_n_size(vb_shuf *const *sides, u32 n_sides, u32 rid, u64 *n_keys, u64 *n_vals)
{
    CogroupNSides a;
    TRY(cogroup_n_sides(sides, n_sides, rid, &a));
    CogroupNPlan *p = nullptr;
    TRY(cogroup_n_plan(sides, n_sides, rid, NP_COGROUP, a, &p));
    if (n_keys) *n_keys = p->n_keys;
    for (u32 j = 0; n_vals && j < n_sides; ++j) n_vals[j] = sides[j]->val_off[rid + 1] - sides[j]->val_off[rid];
    return VB_OK;
}

static int str_plan_keys(vb_shuf *const *sides, u32 n, u32 rid, i64 kind, CogroupNPlan *p);
static int str_write_keys(vb_shuf *const *sides, u32 n, u32 rid, i64 kind, CogroupNPlan *p, u64 *out_key_offsets,
                          void *out_key_bytes, int dst_loc);

// string sides: out_keys is the key bytes, out_key_offsets their offsets
static int cogroup_n_write(vb_shuf *const *sides, u32 n_sides, u32 rid, void *out_keys, u64 *const *out_offsets,
                           void *const *out_vals, int dst_loc, u64 *out_key_offsets = nullptr)
{
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    CogroupNSides a;
    TRY(cogroup_n_sides(sides, n_sides, rid, &a));
    CogroupNPlan *p = nullptr;
    TRY(cogroup_n_plan(sides, n_sides, rid, NP_COGROUP, a, &p));
    const u64 nk = p->n_keys, nk0 = s0->bucket_off[rid + 1] - s0->bucket_off[rid];
    int rc = [&]() -> int {
        if (s0->str) {
            TRY(str_write_keys(sides, n_sides, rid, NP_COGROUP, p, out_key_offsets, out_keys, dst_loc));
        } else {
            TRY(copy_out(s0, out_keys, s0->res_keys ? s0->res_keys + a.kb[0] : nullptr, nk0 * 8, dst_loc));
            TRY(copy_out(s0, out_keys ? (u64 *)out_keys + nk0 : nullptr, p->new_keys, (nk - nk0) * 8, dst_loc));
        }
        for (u32 j = 0; j < n_sides; ++j) {
            u64 *o_offs = out_offsets ? out_offsets[j] : nullptr;
            void *o_vals = out_vals ? out_vals[j] : nullptr;
            if (!o_offs && !o_vals) continue;
            vb_shuf *s = sides[j];
            const u64 nv = s->val_off[rid + 1] - s->val_off[rid];
            if (j == 0) {
                // side 0's lists are its partition's value slice as it is: its CSR offsets rebased, then flat (nv) for
                // the keys after side 0's
                if (o_offs) {
                    DevBuf tmp(c);
                    u64 *d = o_offs;
                    if (dst_loc == VB_HOST) { TRY(tmp.alloc((nk + 1) * 8)); d = tmp.as<u64>(); }
                    {
                        KLaunch kl(s0, K_JOIN);
                        cogroup_left_offsets_kernel<<<(unsigned)((nk + 1 + 255) / 256), 256, 0, c->stream>>>(s->res_offs, a.kb[0], (u32)nk0,
                                                                                                            nk + 1, s->val_off[rid], nv, d);
                        TRY(kl.done("cogroup_left_offsets_kernel"));
                    }
                    if (dst_loc == VB_HOST) TRY(copy_out(s0, o_offs, d, (nk + 1) * 8, VB_HOST));
                }
                if (o_vals && nv) TRY(copy_out(s0, o_vals, s->res_vals + s->val_off[rid], nv * 8, dst_loc));
                continue;
            }
            // side j's list offsets: the list lengths of the output keys, scanned (on the device even for a host output)
            DevBuf pos(c), cnt(c);
            u64 *d_pos = (o_offs && dst_loc == VB_DEVICE) ? o_offs : nullptr;
            if (!d_pos) { TRY(pos.alloc((nk + 1) * 8)); d_pos = pos.as<u64>(); }
            if (nk == 0) {
                CU(cudaMemsetAsync(d_pos, 0, 8, c->stream));
            } else {
                TRY(cnt.alloc(nk * 8));
                {
                    KLaunch kl(s0, K_JOIN);
                    cogroup_n_count_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, c->stream>>>(p->match, n_sides, j, (u32)nk,
                                                                                                s->res_offs, cnt.as<u64>());
                    TRY(kl.done("cogroup_n_count_kernel"));
                }
                TRY(exclusive_scan_u64(s0, cnt.as<u64>(), d_pos, nk, d_pos + nk));
            }
            if (o_offs && dst_loc == VB_HOST) TRY(copy_out(s0, o_offs, d_pos, (nk + 1) * 8, VB_HOST));
            if (!o_vals || !nv) continue;
            DevBuf tmp(c);
            u64 *d = (u64 *)o_vals;
            if (dst_loc == VB_HOST) { TRY(tmp.alloc(nv * 8)); d = tmp.as<u64>(); }
            {
                KLaunch kl(s0, K_JOIN);
                const u64 blocks = std::min<u64>((nv + 255) / 256, (u64)c->sm_count * 8);
                cogroup_n_gather_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(d_pos, (u32)nk, p->match, n_sides, j,
                                                                                s->res_offs, s->res_vals, d);
                TRY(kl.done("cogroup_n_gather_kernel"));
            }
            if (dst_loc == VB_HOST) TRY(copy_out(s0, o_vals, d, nv * 8, VB_HOST));
        }
        return VB_OK;
    }();
    cudaStreamSynchronize(c->stream);
    drop_cogroup_n_plan(sides, n_sides, rid, NP_COGROUP);
    return rc;
}

static int join_n_size(vb_shuf *const *sides, u32 n_sides, u32 rid, u64 *n_out)
{
    CogroupNSides a;
    TRY(cogroup_n_sides(sides, n_sides, rid, &a));
    CogroupNPlan *p = nullptr;
    TRY(cogroup_n_plan(sides, n_sides, rid, NP_INNER, a, &p));
    *n_out = p->total;
    return VB_OK;
}

static int join_n_write(vb_shuf *const *sides, u32 n_sides, u32 rid, void *out_k, void *const *out_vals, int dst_loc)
{
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    CogroupNSides a;
    TRY(cogroup_n_sides(sides, n_sides, rid, &a));
    CogroupNPlan *p = nullptr;
    TRY(cogroup_n_plan(sides, n_sides, rid, NP_INNER, a, &p));
    const u64 total = p->total;
    int rc = [&]() -> int {
        if (!total) return VB_OK;
        bool missing = !out_k || !out_vals;
        for (u32 j = 0; !missing && j < n_sides; ++j) missing = !out_vals[j];
        if (missing) return set_err(VB_ERR_INVALID, "NULL output with %llu rows to write", (unsigned long long)total);
        JoinNOut o{};
        DevBuf bufs[CGN_MAX_SIDES + 1];
        o.k = (u64 *)out_k;
        for (u32 j = 0; j < n_sides; ++j) o.v[j] = (u64 *)out_vals[j];
        if (dst_loc == VB_HOST) {
            for (u32 j = 0; j <= n_sides; ++j) { bufs[j].c = c; TRY(bufs[j].alloc(total * 8)); }
            o.k = bufs[n_sides].as<u64>();
            for (u32 j = 0; j < n_sides; ++j) o.v[j] = bufs[j].as<u64>();
        }
        {
            KLaunch kl(s0, K_JOIN);
            const u64 blocks = std::min<u64>((total + 255) / 256, (u64)c->sm_count * 8);
            join_n_expand_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(a, p->pos, (u32)p->n_keys, total, p->match, o);
            TRY(kl.done("join_n_expand_kernel"));
        }
        if (dst_loc == VB_HOST) {
            TRY(copy_out(s0, out_k, o.k, total * 8, VB_HOST));
            for (u32 j = 0; j < n_sides; ++j) TRY(copy_out(s0, out_vals[j], o.v[j], total * 8, VB_HOST));
        }
        return VB_OK;
    }();
    cudaStreamSynchronize(c->stream);
    drop_cogroup_n_plan(sides, n_sides, rid, NP_INNER);
    return rc;
}

// Outer join of n sides (a key is kept when every side of `required` has it; a missing optional side gives one None
// slot): the plan of the union of the keys (side 0's keys alone when side 0 is required), counted with max(len, 1)
static int join_n_outer_size(vb_shuf *const *sides, u32 n_sides, u32 rid, u32 required, u64 *n_out)
{
    CogroupNSides a;
    TRY(cogroup_n_sides(sides, n_sides, rid, &a));
    CogroupNPlan *p = nullptr;
    TRY(cogroup_n_plan(sides, n_sides, rid, required, a, &p));
    *n_out = p->total;
    return VB_OK;
}

// string sides: out_k is the key bytes of the keys with rows, out_key_offsets their offsets and out_row_offsets their
// rows; the rows carry no key
static int join_n_outer_write(vb_shuf *const *sides, u32 n_sides, u32 rid, u32 required, void *out_k, void *const *out_vals,
                              uint8_t *const *out_valid, int dst_loc, u64 *out_key_offsets = nullptr, u64 *out_row_offsets = nullptr)
{
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    const bool str = s0->str != nullptr;
    CogroupNSides a;
    TRY(cogroup_n_sides(sides, n_sides, rid, &a));
    CogroupNPlan *p = nullptr;
    TRY(cogroup_n_plan(sides, n_sides, rid, required, a, &p));
    const u64 total = p->total;
    int rc = [&]() -> int {
        if (!total) {
            if (str) TRY(str_write_keys(sides, n_sides, rid, required, p, out_key_offsets, out_k, dst_loc));
            if (str && out_row_offsets) TRY(copy_out(s0, out_row_offsets, p->str_roff, 8, dst_loc));
            return VB_OK;
        }
        bool missing = !out_vals;
        if (str) {
            TRY(str_plan_keys(sides, n_sides, rid, required, p));
            missing = missing || !out_key_offsets || !out_row_offsets || (p->str_nkb && !out_k);
        } else {
            missing = missing || !out_k;
        }
        for (u32 j = 0; !missing && j < n_sides; ++j) missing = !out_vals[j];
        if (missing) return set_err(VB_ERR_INVALID, "NULL output with %llu rows to write", (unsigned long long)total);
        JoinNOuterOut o{};
        DevBuf bufs[2 * CGN_MAX_SIDES + 1];     // host output: keys, values per side, validity per side
        if (!str) {
            o.k = (u64 *)out_k;
            o.new_keys = p->new_keys;
            o.nk0 = (u32)(s0->bucket_off[rid + 1] - s0->bucket_off[rid]);
        }
        for (u32 j = 0; j < n_sides; ++j) {
            o.v[j] = (u64 *)out_vals[j];
            o.valid[j] = out_valid ? out_valid[j] : nullptr;
        }
        if (dst_loc == VB_HOST) {
            for (u32 j = 0; j <= n_sides; ++j) {
                if (str && j == n_sides) continue;
                bufs[j].c = c;
                TRY(bufs[j].alloc(total * 8));
            }
            if (!str) o.k = bufs[n_sides].as<u64>();
            for (u32 j = 0; j < n_sides; ++j) {
                o.v[j] = bufs[j].as<u64>();
                if (!o.valid[j]) continue;
                DevBuf &b = bufs[n_sides + 1 + j];
                b.c = c;
                TRY(b.alloc(total));
                o.valid[j] = b.as<unsigned char>();
            }
        }
        {
            KLaunch kl(s0, K_JOIN);
            const u64 blocks = std::min<u64>((total + 255) / 256, (u64)c->sm_count * 8);
            if (str) {
                join_n_outer_expand_nokey_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(a, p->pos, (u32)p->n_keys, total, p->match, o);
                TRY(kl.done("join_n_outer_expand_nokey_kernel"));
            } else {
                join_n_outer_expand_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(a, p->pos, (u32)p->n_keys, total, p->match, o);
                TRY(kl.done("join_n_outer_expand_kernel"));
            }
        }
        if (str) {
            TRY(str_write_keys(sides, n_sides, rid, required, p, out_key_offsets, out_k, dst_loc));
            TRY(copy_out(s0, out_row_offsets, p->str_roff, (p->str_nk + 1) * 8, dst_loc));
        }
        if (dst_loc == VB_HOST) {
            if (!str) TRY(copy_out(s0, out_k, o.k, total * 8, VB_HOST));
            for (u32 j = 0; j < n_sides; ++j) {
                TRY(copy_out(s0, out_vals[j], o.v[j], total * 8, VB_HOST));
                if (o.valid[j]) TRY(copy_out(s0, out_valid[j], o.valid[j], total, VB_HOST));
            }
        }
        return VB_OK;
    }();
    cudaStreamSynchronize(c->stream);
    drop_cogroup_n_plan(sides, n_sides, rid, required);
    return rc;
}

extern "C" int32_t vb_cogroup_n_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint64_t *n_keys, uint64_t *n_vals)
{
    TRY(cogroup_n_check(sides, n_sides, rid));
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(ensure_grouped(sides[j]));
    return cogroup_n_size(sides, n_sides, rid, n_keys, n_vals);
}

extern "C" int32_t vb_cogroup_n(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, void *out_keys,
                                uint64_t *const *out_offsets, void *const *out_vals, int32_t dst_loc)
{
    TRY(cogroup_n_check(sides, n_sides, rid));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(ensure_grouped(sides[j]));
    return cogroup_n_write(sides, n_sides, rid, out_keys, out_offsets, out_vals, dst_loc);
}

extern "C" int32_t vb_join_n_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint64_t *n_out)
{
    TRY(cogroup_n_check(sides, n_sides, rid));
    if (!n_out) return set_err(VB_ERR_INVALID, "n_out is NULL");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(ensure_grouped(sides[j]));
    return join_n_size(sides, n_sides, rid, n_out);
}

extern "C" int32_t vb_join_n(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, void *out_k, void *const *out_vals,
                             int32_t dst_loc)
{
    TRY(cogroup_n_check(sides, n_sides, rid));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(ensure_grouped(sides[j]));
    return join_n_write(sides, n_sides, rid, out_k, out_vals, dst_loc);
}

// vb_cogroup_n's rules, and no required bit at or above n_sides
static int join_n_outer_check(vb_shuf *const *sides, u32 n_sides, u32 rid, u32 required)
{
    TRY(cogroup_n_check(sides, n_sides, rid));
    if (required >> n_sides)                           // n_sides <= 16 here
        return set_err(VB_ERR_INVALID, "required mask %#x names a side >= n_sides %u", required, n_sides);
    return VB_OK;
}

extern "C" int32_t vb_join_n_outer_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required,
                                        uint64_t *n_out)
{
    TRY(join_n_outer_check(sides, n_sides, rid, required));
    if (!n_out) return set_err(VB_ERR_INVALID, "n_out is NULL");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(ensure_grouped(sides[j]));
    return join_n_outer_size(sides, n_sides, rid, required, n_out);
}

extern "C" int32_t vb_join_n_outer(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required, void *out_k,
                                   void *const *out_vals, uint8_t *const *out_valid, int32_t dst_loc)
{
    TRY(join_n_outer_check(sides, n_sides, rid, required));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(ensure_grouped(sides[j]));
    return join_n_outer_write(sides, n_sides, rid, required, out_k, out_vals, out_valid, dst_loc);
}

// ---------------------------------------------------------------------------------------------
// semi and anti joins of n sides.  vega has no such op; this restates it over CoGroupedRdd::compute
// (co_grouped_rdd.rs:206-249): a key of side 0's partition r is kept when its side-0 list is non-empty, every side of
// `required` has it and no side of `excluded` does, and then gives the rows (k, v) for v in its side-0 list.  Only side
// 0's values are read.  The keys of the filter sides (required | excluded, a shuffle listed twice counted once) go into
// one presence dictionary with a side mask per slot; a lazy filter side gives its rows' keys and is never grouped.  A
// lazy side 0 is filtered row by row and only its kept rows are grouped; a grouped side 0 (GROUP, grouped COGROUP,
// narrow view) is probed once per key of the partition.  Either way the partition is a one-side join plan over a
// grouped source, written by join_n_expand_kernel.  Cost: linear in side 0's rows (or keys) and the filter sides' keys.
// ---------------------------------------------------------------------------------------------
static i64 semi_kind(u32 required, u32 excluded) { return NP_SEMI - (i64)(((u64)excluded << 16) | required); }

// the mask rules of vb_semi_join_n*, after the cogroup rules (so n_sides <= 16)
static int semi_masks_check(u32 n, u32 required, u32 excluded)
{
    if ((required | excluded) >> n)
        return set_err(VB_ERR_INVALID, "mask %#x names a side >= n_sides %u", (required | excluded), n);
    if ((required | excluded) & 1u) return set_err(VB_ERR_INVALID, "side 0 cannot be required or excluded: it is the side filtered");
    if (required & excluded) return set_err(VB_ERR_INVALID, "sides %#x are both required and excluded", required & excluded);
    return VB_OK;
}

static void semi_count_launches(vb_shuf *s0, const vb_shuf *t)
{
    for (int k = 0; k < K_N; ++k) s0->klaunch[k] += t->klaunch[k];
    s0->st.kernel_launches += t->st.kernel_launches;
    s0->st.table_slots = std::max(s0->st.table_slots, t->st.table_slots);
}

// The filter of (sides, required, excluded), built once and kept on side 0; the context is locked
static int semi_filter(vb_shuf *const *sides, u32 n, u32 required, u32 excluded, SemiFilter **out)
{
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    std::vector<u64> uids(n);
    for (u32 j = 0; j < n; ++j) uids[j] = sides[j]->uid;
    const auto key = std::make_tuple(uids, required, excluded);
    auto it = s0->semi.find(key);
    if (it != s0->semi.end()) { *out = &it->second; return VB_OK; }
    const u32 filter = required | excluded;
    SemiFilter f;
    if (!filter) {                                     // no filter side: side 0's rows as its reduce gives them
        TRY(ensure_grouped(s0));
        *out = &s0->semi.emplace(key, f).first->second;
        return VB_OK;
    }
    // 1. every filter shuffle once, with the bits of the sides it is; its keys (a lazy side's rows' keys)
    std::vector<vb_shuf *> fs;
    std::vector<u32> bits;
    for (u32 j = 1; j < n; ++j) {
        if (!(filter >> j & 1u)) continue;
        const size_t i = std::find(fs.begin(), fs.end(), sides[j]) - fs.begin();
        if (i == fs.size()) { fs.push_back(sides[j]); bits.push_back(0); }
        bits[i] |= 1u << j;
    }
    std::vector<AggInput> in;
    std::vector<u32> in_bits;
    u64 total = 0;
    for (size_t i = 0; i < fs.size(); ++i) {
        const vb_shuf *s = fs[i];
        const u64 m = s->lazy ? s->lz_n : s->n_keys;
        if (!m) continue;
        in.push_back(AggInput{IN_SOA, s->lazy ? s->lz_keys : s->res_keys, nullptr, m, VB_DEVICE});
        in_bits.push_back(bits[i]);
        total += m;
    }
    // 2. the presence dictionary: one table over all of them, then each input's bits ORed into its rows' slots
    DevBuf tab(c), mask(c);
    if (total) {
        DevBuf ids(c);
        TRY(ids.alloc(total * 4));
        u64 n_ins = 0;
        TRY(build_table(s0, K_DICT, in, OPK_DICT, TX_NONE, 0, &tab.p, &f.log_cap, &n_ins, ids.as<u32>()));
        const u64 slots = (1ull << f.log_cap) + 1 + 16;
        TRY(mask.alloc(slots * 4));
        CU(cudaMemsetAsync(mask.p, 0, slots * 4, c->stream));
        u64 at = 0;
        for (size_t i = 0; i < in.size(); ++i) {
            KLaunch kl(s0, K_JOIN, in[i].n);
            const unsigned g = (unsigned)std::min<u64>((in[i].n + 255) / 256, (u64)c->sm_count * 16);
            presence_mark_kernel<<<g, 256, 0, c->stream>>>(ids.as<u32>() + at, in[i].n, in_bits[i], mask.as<u32>());
            TRY(kl.done("presence_mark_kernel"));
            at += in[i].n;
        }
        s0->st.table_slots = std::max<u64>(s0->st.table_slots, 1ull << f.log_cap);
    }
    const Table t = table_at(tab.p, f.log_cap);
    if (s0->lazy) {
        // 3. a lazy side 0: keep its rows by the rule (stable), then group only those, in side 0's value order
        Gathered g;
        DevBuf keep(c), gk(c), gv(c);
        if (s0->lz_n) {
            TRY(keep.alloc(s0->lz_n));
            {
                KLaunch kl(s0, K_JOIN, s0->lz_n);
                const unsigned gr = (unsigned)std::min<u64>((s0->lz_n + 255) / 256, (u64)c->sm_count * 16);
                presence_probe_kernel<<<gr, 256, 0, c->stream>>>(s0->lz_keys, s0->lz_n, t, mask.as<u32>(), required, excluded,
                                                                 keep.as<unsigned char>());
                TRY(kl.done("presence_probe_kernel"));
            }
            TRY(compact_rows(s0, s0->lz_keys, s0->lz_vals, s0->lz_n, keep.as<unsigned char>(), gk, gv, &g.n));
            g.keys = gk.as<u64>(); g.vals = gv.as<u64>();
        }
        vb_shuf *k = make_internal_like(s0);
        k->bucket_off.assign((size_t)s0->n_reduce + 1, 0);
        k->val_off = k->bucket_off;
        if (g.n) {
            const int rc = seal_group(k, g);
            if (rc) { s0->trash.push_back(k); return rc; }   // freed with s0 (vb_shuffle_free would re-lock the context)
        }
        CU(cudaStreamSynchronize(c->stream));
        semi_count_launches(s0, k);
        f.kept = k;
    } else {
        CU(cudaStreamSynchronize(c->stream));
        f.tab = tab.release();
        f.mask = (u32 *)mask.release();
    }
    *out = &s0->semi.emplace(key, f).first->second;
    return VB_OK;
}

// The plan of partition rid: the kept keys' side-0 list lengths scanned (pos, total) over a one-side match (each key's
// own index), cached in side 0's n_plans.  *src: the grouped shuffle the plan indexes (side 0, or its kept rows).
static int semi_plan(vb_shuf *const *sides, u32 n, u32 rid, u32 required, u32 excluded, CogroupNPlan **out, vb_shuf **src)
{
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    const bool str = s0->str != nullptr;
    SemiFilter *f = nullptr;
    if (!str) TRY(semi_filter(sides, n, required, excluded, &f));
    vb_shuf *g = f && f->kept ? f->kept : s0;
    *src = g;
    std::vector<u64> uids(n);
    for (u32 j = 0; j < n; ++j) uids[j] = sides[j]->uid;
    const auto key = std::make_tuple(uids, rid, semi_kind(required, excluded));
    auto it = s0->n_plans.find(key);
    if (it != s0->n_plans.end()) { *out = &it->second; return VB_OK; }
    const u64 nk = g->bucket_off[rid + 1] - g->bucket_off[rid];
    if (nk >= 0xFFFFFFFFull) return set_err(VB_ERR_TOO_LARGE, "%llu keys in one semi-join partition", (unsigned long long)nk);
    CogroupNPlan p;
    p.n_keys = nk;
    if (nk) {
        DevBuf match(c), cnt(c), pos(c);
        TRY(match.alloc(nk * 4)); TRY(cnt.alloc(nk * 8)); TRY(pos.alloc((nk + 1) * 8));
        const u32 kb = (u32)g->bucket_off[rid];
        {
            KLaunch kl(s0, K_JOIN, nk);
            const unsigned gr = (unsigned)((nk + 255) / 256);
            if (str) {
                StrNSides sa;
                TRY(str_n_sides(sides, n, rid, &sa));
                semi_str_count_kernel<<<gr, 256, 0, c->stream>>>(sa, g->res_offs, (u32)nk, required, excluded, cnt.as<u64>(), match.as<u32>());
                TRY(kl.done("semi_str_count_kernel"));
            } else {
                // the kept rows were filtered already: every key of theirs is kept
                const bool all = f->kept != nullptr;
                presence_count_kernel<<<gr, 256, 0, c->stream>>>(g->res_keys, g->res_offs, kb, (u32)nk, table_at(f->tab, f->log_cap),
                                                                 f->mask, all ? 0 : required, all ? 0 : excluded, cnt.as<u64>(),
                                                                 match.as<u32>());
                TRY(kl.done("presence_count_kernel"));
            }
        }
        TRY(exclusive_scan_u64(s0, cnt.as<u64>(), pos.as<u64>(), nk, pos.as<u64>() + nk));
        CU(cudaMemcpyAsync(c->h_scratch, pos.as<u64>() + nk, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        p.total = *(u64 *)c->h_scratch;
        p.match = (u32 *)match.release();
        p.pos = (u64 *)pos.release();
    }
    *out = &s0->n_plans.emplace(key, p).first->second;
    return VB_OK;
}

// one side of the plan's grouped source, for join_n_expand_kernel / cogroup_n_gather_kernel
static CogroupNSides semi_side(const vb_shuf *g, u32 rid)
{
    CogroupNSides a{};
    a.n = 1;
    a.keys[0] = g->res_keys; a.offs[0] = g->res_offs; a.vals[0] = g->res_vals;
    a.kb[0] = (u32)g->bucket_off[rid];
    return a;
}

static int semi_write(vb_shuf *const *sides, u32 n, u32 rid, u32 required, u32 excluded, void *out_k, void *out_v, int dst_loc)
{
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    CogroupNPlan *p = nullptr;
    vb_shuf *g = nullptr;
    TRY(semi_plan(sides, n, rid, required, excluded, &p, &g));
    const u64 total = p->total;
    int rc = [&]() -> int {
        if (!total) return VB_OK;
        if (!out_k || !out_v) return set_err(VB_ERR_INVALID, "NULL output with %llu rows to write", (unsigned long long)total);
        JoinNOut o{};
        o.k = (u64 *)out_k; o.v[0] = (u64 *)out_v;
        DevBuf bk(c), bv(c);
        if (dst_loc == VB_HOST) {
            TRY(bk.alloc(total * 8)); TRY(bv.alloc(total * 8));
            o.k = bk.as<u64>(); o.v[0] = bv.as<u64>();
        }
        {
            KLaunch kl(s0, K_JOIN, total);
            const u64 blocks = std::min<u64>((total + 255) / 256, (u64)c->sm_count * 8);
            join_n_expand_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(semi_side(g, rid), p->pos, (u32)p->n_keys, total, p->match, o);
            TRY(kl.done("join_n_expand_kernel"));
        }
        if (dst_loc == VB_HOST) {
            TRY(copy_out(s0, out_k, o.k, total * 8, VB_HOST));
            TRY(copy_out(s0, out_v, o.v[0], total * 8, VB_HOST));
        }
        return VB_OK;
    }();
    cudaStreamSynchronize(c->stream);
    drop_cogroup_n_plan(sides, n, rid, semi_kind(required, excluded));
    return rc;
}

extern "C" int32_t vb_semi_join_n_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required,
                                       uint32_t excluded, uint64_t *n_rows)
{
    TRY(cogroup_n_check(sides, n_sides, rid));
    TRY(semi_masks_check(n_sides, required, excluded));
    if (!n_rows) return set_err(VB_ERR_INVALID, "n_rows is NULL");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    CogroupNPlan *p = nullptr;
    vb_shuf *g = nullptr;
    TRY(semi_plan(sides, n_sides, rid, required, excluded, &p, &g));
    *n_rows = p->total;
    return VB_OK;
}

extern "C" int32_t vb_semi_join_n(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required, uint32_t excluded,
                                  void *out_k, void *out_v, int32_t dst_loc)
{
    TRY(cogroup_n_check(sides, n_sides, rid));
    TRY(semi_masks_check(n_sides, required, excluded));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    return semi_write(sides, n_sides, rid, required, excluded, out_k, out_v, dst_loc);
}

extern "C" int32_t vb_cogroup_size(vb_shuf *l, vb_shuf *r, uint32_t rid, uint64_t *n_keys, uint64_t *n_left_vals,
                                   uint64_t *n_right_vals)
{
    TRY(join_check(l, r, rid));
    std::lock_guard<std::mutex> lk(l->ctx->mu);
    CU(cudaSetDevice(l->ctx->device));
    TRY(join_sides(l, r, JK_FULL));
    vb_shuf *const sides[2] = {l, r};
    u64 n_vals[2];
    TRY(cogroup_n_size(sides, 2, rid, n_keys, n_vals));
    if (n_left_vals) *n_left_vals = n_vals[0];
    if (n_right_vals) *n_right_vals = n_vals[1];
    return VB_OK;
}

extern "C" int32_t vb_cogroup(vb_shuf *l, vb_shuf *r, uint32_t rid, void *out_keys, uint64_t *out_left_offsets,
                              void *out_left_vals, uint64_t *out_right_offsets, void *out_right_vals, int32_t dst_loc)
{
    TRY(join_check(l, r, rid));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    std::lock_guard<std::mutex> lk(l->ctx->mu);
    CU(cudaSetDevice(l->ctx->device));
    TRY(join_sides(l, r, JK_FULL));
    vb_shuf *const sides[2] = {l, r};
    u64 *const out_offsets[2] = {out_left_offsets, out_right_offsets};
    void *const out_vals[2] = {out_left_vals, out_right_vals};
    return cogroup_n_write(sides, 2, rid, out_keys, out_offsets, out_vals, dst_loc);
}

extern "C" int32_t vb_join_size(vb_shuf *l, vb_shuf *r, uint32_t rid, uint64_t *n_out)
{
    TRY(join_check(l, r, rid));
    if (!n_out) return set_err(VB_ERR_INVALID, "n_out is NULL");
    std::lock_guard<std::mutex> lk(l->ctx->mu);
    CU(cudaSetDevice(l->ctx->device));
    TRY(join_sides(l, r, JK_INNER));
    vb_shuf *const sides[2] = {l, r};
    return join_n_size(sides, 2, rid, n_out);
}

extern "C" int32_t vb_join(vb_shuf *l, vb_shuf *r, uint32_t rid, void *out_k, void *out_v, void *out_w, int32_t dst_loc)
{
    TRY(join_check(l, r, rid));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    std::lock_guard<std::mutex> lk(l->ctx->mu);
    CU(cudaSetDevice(l->ctx->device));
    TRY(join_sides(l, r, JK_INNER));
    vb_shuf *const sides[2] = {l, r};
    void *const out_vals[2] = {out_v, out_w};
    return join_n_write(sides, 2, rid, out_k, out_vals, dst_loc);
}

// ---------------------------------------------------------------------------------------------
// string keys (vb_shuffle_create_str): byte-string keys placed like the reference's `String` keys
// ---------------------------------------------------------------------------------------------
// One shuffle's dictionary of distinct keys (strkeys.cuh: entries + arena + index), the map calls' rows as entry ids,
// and after seal the partition-major key column (Arrow-style offsets + bytes) beside the usual res_* arrays.
struct StrState {
    int kind = STRKEY_STR;                // how the keys hash (vb_shuffle_set_str_key): placement only
    StrDict d{};                          // device arrays; d.fp / d.id have 1 << d.log_cap slots
    u64 cap_e = 0, cap_a = 0;             // entries / arena bytes reserved
    u32 n_e = 0;                          // entries in use (ctl->n_entries after the last call)
    u64 n_a = 0;                          // arena bytes in use
    StrCtl *ctl = nullptr;
    std::vector<u32 *> ids;               // per map id: the rows' entry ids (owned)
    std::vector<const u64 *> vals;        // GROUP, per map id: the rows' values
    struct Cols { const u64 *c[MA_MAX_COLS]; };
    std::vector<Cols> cols;               // reduce ops and combine_by_key, per map id: the value columns of the spec
    std::vector<char> vals_owned;         // per map id: vals / cols are copies (else borrowed, VB_DEVICE_BORROWED)
    std::vector<char> blob;               // per map id: a bincode blob's partials in vals (vb_shuffle_map_blob), not rows
    u64 *key_off = nullptr;               // [n_keys + 1] byte offset of every result key (partition-major, from 0)
    unsigned char *key_bytes = nullptr;   // the result keys' bytes
    std::vector<u64> kb_off;              // [n_reduce + 1] first key byte of each partition
    // key index of the result keys (str_key_index), built by the first cogroup or join that reads the shuffle
    u64 *res_hash = nullptr;              // [n_keys] each key's hash
    u64 *ix_fp = nullptr;                 // [1 << ix_log_cap] fingerprints, 0 = empty
    u32 *ix_id = nullptr;                 // [1 << ix_log_cap] dense key id of each slot
    u32 ix_log_cap = 0;
    // across ranks (vb_shuffle_create_str_dist): the exported columns, destination-major, owned until seal ...
    u32 *x_lens = nullptr, *x_cnts = nullptr;
    unsigned char *x_bytes = nullptr;
    u64 *x_vals = nullptr;
    // ... and the imported ones, source-rank major: borrowed until seal, or received by vb_shuffle_exchange (i_own).
    // Reduce ops and combine_by_key: x_vals / i_vals are the accumulators [n_acc][keys], in plain value form
    const u32 *i_lens = nullptr, *i_cnts = nullptr;
    const unsigned char *i_bytes = nullptr;
    const u64 *i_vals = nullptr;
    u64 i_nk = 0, i_nkb = 0, i_nv = 0;
    void *i_own[4] = {};
    // sort_by_key (vb_shuffle_create_str_sort): after seal key_off / key_bytes hold the D distinct keys in rank order,
    // res_vals the payload in row order, and partition r is rows [bucket_off[r], bucket_off[r + 1]), ranks
    // [rank_cut[r], rank_cut[r + 1]) and key bytes [kb_off[r], kb_off[r + 1])
    bool sort = false, sort_vals = false;   // a sort shuffle; with a payload column
    u64 *row_off = nullptr;                 // [D + 1] first row of each rank (the CSR), row_off[D] = rows
    u64 *row_boff = nullptr;                // [D + 1] first key byte of each rank's rows (each row carries its key)
    std::vector<u64> rank_cut;              // [n_reduce + 1]
};

constexpr u32 STR_MAX_LOG_CAP = 33;       // index slots: < 2^31 distinct keys at load <= 0.6

// VEGA_B200_STR_FP_BITS=k keeps k bits of the hash in the index fingerprint (test switch: forces equal fingerprints of
// distinct keys, which must then be told apart by their bytes).  Placement always uses the full hash.
static u64 str_fp_mask()
{
    static const u64 m = [] {
        const char *e = getenv("VEGA_B200_STR_FP_BITS");
        const int k = e ? atoi(e) : 64;
        return (k <= 0 || k >= 64) ? ~0ull : ((1ull << k) - 1);
    }();
    return m;
}

static void free_str_map(vb_shuf *s, u32 m)
{
    StrState *t = s->str;
    dev_free(s->ctx, t->ids[m]);
    if (t->vals_owned[m]) {
        dev_free(s->ctx, t->vals[m]);
        for (const u64 *p : t->cols[m].c) dev_free(s->ctx, p);
    }
    t->ids[m] = nullptr;
    t->vals[m] = nullptr;
    t->cols[m] = StrState::Cols{};
    t->vals_owned[m] = 0;
    t->blob[m] = 0;
}

static void free_str_dict(vb_shuf *s)
{
    StrState *t = s->str;
    vb_ctx *c = s->ctx;
    dev_free(c, t->d.fp); dev_free(c, t->d.id);
    dev_free(c, t->d.e_hash); dev_free(c, t->d.e_off); dev_free(c, t->d.e_len); dev_free(c, t->d.arena);
    dev_free(c, t->ctl);
    t->d.fp = nullptr; t->d.id = nullptr;
    t->d.e_hash = t->d.e_off = nullptr; t->d.e_len = nullptr; t->d.arena = nullptr;
    t->ctl = nullptr;
    t->cap_e = t->cap_a = 0;
}

static void free_str_xchg(vb_shuf *s)
{
    StrState *t = s->str;
    vb_ctx *c = s->ctx;
    dev_free(c, t->x_lens); dev_free(c, t->x_cnts); dev_free(c, t->x_bytes); dev_free(c, t->x_vals);
    t->x_lens = t->x_cnts = nullptr; t->x_bytes = nullptr; t->x_vals = nullptr;
    for (void *&p : t->i_own) { dev_free(c, p); p = nullptr; }
    t->i_lens = t->i_cnts = nullptr; t->i_bytes = nullptr; t->i_vals = nullptr;
    t->i_nk = t->i_nkb = t->i_nv = 0;
}

static void free_str(vb_shuf *s)
{
    StrState *t = s->str;
    if (!t) return;
    for (u32 m = 0; m < s->n_map; ++m) free_str_map(s, m);
    free_str_dict(s);
    free_str_xchg(s);
    dev_free(s->ctx, t->key_off);
    dev_free(s->ctx, t->key_bytes);
    dev_free(s->ctx, t->res_hash);
    dev_free(s->ctx, t->ix_fp);
    dev_free(s->ctx, t->ix_id);
    dev_free(s->ctx, t->row_off);
    dev_free(s->ctx, t->row_boff);
    delete t;
    s->str = nullptr;
}

// A fresh string state (empty dictionary, no map output) for a new shuffle
static StrState *str_attach(vb_shuf *s)
{
    StrState *t = new StrState();
    t->ids.assign(s->n_map, nullptr);
    t->vals.assign(s->n_map, nullptr);
    t->cols.assign(s->n_map, StrState::Cols{});
    t->vals_owned.assign(s->n_map, 0);
    t->blob.assign(s->n_map, 0);
    t->d.fp_mask = str_fp_mask();
    s->str = t;
    return t;
}

extern "C" int32_t vb_shuffle_create_str(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t vdt, int32_t agg,
                                         vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_str: NULL argument");
    *out = nullptr;
    if (agg != VB_AGG_SUM && agg != VB_AGG_MIN && agg != VB_AGG_MAX && agg != VB_AGG_COUNT && agg != VB_AGG_GROUP)
        return set_err(VB_ERR_UNSUPPORTED, "string keys: agg %d is not supported (SUM, MIN, MAX, COUNT and GROUP are)", agg);
    TRY(vb_shuffle_create(c, shuffle_id, n_map, n_reduce, VB_U64, vdt, agg, VB_PART_HASH_METRO64, out));
    if (is_reduce_op(agg)) {       // a reduce op is the combine of one value column with one aggregate
        const vb_agg_col one{agg, 0};
        MultiSpec ms;
        const int rc = multi_spec(1, &vdt, 1, &one, &ms);
        if (rc != VB_OK) { vb_shuffle_free(*out); *out = nullptr; return rc; }
        set_spec(*out, ms);
    }
    str_attach(*out);
    return VB_OK;
}

// sort_by_key over string keys: a VB_AGG_SORT / VB_PART_RANGE shuffle with a string dictionary (val_dtype -1: key-only)
extern "C" int32_t vb_shuffle_create_str_sort(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t val_dtype,
                                              vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_str_sort: NULL argument");
    *out = nullptr;
    if (val_dtype != -1 && (val_dtype < VB_U64 || val_dtype > VB_F64))
        return set_err(VB_ERR_INVALID, "vb_shuffle_create_str_sort: val_dtype %d (VB_U64, VB_I64, VB_F64, or -1 for key-only)", val_dtype);
    TRY(vb_shuffle_create(c, shuffle_id, n_map, n_reduce, VB_U64, val_dtype < 0 ? VB_U64 : val_dtype, VB_AGG_SORT, VB_PART_RANGE, out));
    StrState *t = str_attach(*out);
    t->sort = true;
    t->sort_vals = val_dtype >= 0;
    return VB_OK;
}

// sort_by_key over string keys with a byte-string payload: the shuffle of vb_shuffle_create_str_sort, mapped with
// vb_shuffle_map_str_bytes; its payload column holds the references, moved by the sort as any u64 payload
extern "C" int32_t vb_shuffle_create_str_sort_bytes(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_str_sort_bytes: NULL argument");
    *out = nullptr;
    TRY(vb_shuffle_create(c, shuffle_id, n_map, n_reduce, VB_U64, VB_BYTES, VB_AGG_SORT, VB_PART_RANGE, out));
    StrState *t = str_attach(*out);
    t->sort = true;
    t->sort_vals = true;
    return VB_OK;
}

// How the keys of a string shuffle hash: as `String` (the default) or as a byte slice (`Vec<u8>`).  Only the placement
// changes, so the kind may be chosen until the first map, blob or import call, and not after.
extern "C" int32_t vb_shuffle_set_str_key(vb_shuf *s, int32_t kind)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->str) return set_err(VB_ERR_INVALID, "vb_shuffle_set_str_key: shuffle %llu has no string keys (vb_shuffle_create_str*)", (unsigned long long)s->id);
    if (kind != VB_STRKEY_STR && kind != VB_STRKEY_BYTES)
        return set_err(VB_ERR_INVALID, "vb_shuffle_set_str_key: kind %d (VB_STRKEY_STR or VB_STRKEY_BYTES)", kind);
    std::lock_guard<std::mutex> g(s->mu);
    bool started = s->exported || s->imported || s->sealed || s->sealing || s->freed;
    for (const MapOut &m : s->maps) started = started || m.present;
    if (started) return set_err(VB_ERR_STATE, "vb_shuffle_set_str_key: shuffle %llu already has map output", (unsigned long long)s->id);
    s->str->kind = kind == VB_STRKEY_BYTES ? STRKEY_BYTES : STRKEY_STR;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_set_value_order(vb_shuf *s, int32_t order)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    const bool group = s->str ? s->agg == VB_AGG_GROUP && !s->str->sort : is_group_op(s->agg);
    if (!group || s->internal || s->rep)
        return set_err(VB_ERR_INVALID, "vb_shuffle_set_value_order: shuffle %llu is not a GROUP or COGROUP shuffle", (unsigned long long)s->id);
    if (order != VB_VALORDER_INPUT && order != VB_VALORDER_ASC)
        return set_err(VB_ERR_INVALID, "vb_shuffle_set_value_order: order %d (VB_VALORDER_INPUT or VB_VALORDER_ASC)", order);
    if (s->vdt == VB_BYTES) return set_err(VB_ERR_UNSUPPORTED, "vb_shuffle_set_value_order: byte-string values have no value order");
    std::lock_guard<std::mutex> g(s->mu);
    bool started = s->exported || s->imported || s->sealed || s->sealing || s->freed;
    for (const MapOut &m : s->maps) started = started || m.present;
    if (started) return set_err(VB_ERR_STATE, "vb_shuffle_set_value_order: shuffle %llu already has map output", (unsigned long long)s->id);
    s->vorder = order;
    return VB_OK;
}

// Reallocate one device array to `cap` elements of `sz` bytes, keeping the first `keep`.
template <typename T>
static int str_regrow(vb_ctx *c, T **p, u64 cap, u64 keep)
{
    DevBuf nb(c);
    TRY(nb.alloc(cap * sizeof(T)));
    if (keep) CU(cudaMemcpyAsync(nb.p, *p, keep * sizeof(T), cudaMemcpyDeviceToDevice, c->stream));
    dev_free(c, *p);
    *p = (T *)nb.release();
    return VB_OK;
}

// Entries and arena for the worst case of the next call (every row a new key), growing by doubling.
static int str_reserve(vb_shuf *s, u64 want_e, u64 want_a)
{
    StrState *t = s->str;
    vb_ctx *c = s->ctx;
    if (want_e > t->cap_e || !t->d.e_hash) {
        const u64 cap = std::max<u64>(want_e, std::max<u64>(2 * t->cap_e, 1024));
        TRY(str_regrow(c, &t->d.e_hash, cap, t->n_e));
        TRY(str_regrow(c, &t->d.e_off, cap, t->n_e));
        TRY(str_regrow(c, &t->d.e_len, cap, t->n_e));
        t->cap_e = cap;
    }
    if (want_a > t->cap_a || !t->d.arena) {
        const u64 cap = std::max<u64>(want_a, std::max<u64>(2 * t->cap_a, 1 << 16));
        TRY(str_regrow(c, &t->d.arena, cap, t->n_a));
        t->cap_a = cap;
    }
    return VB_OK;
}

// A new index of at least 2^log_cap slots holding every entry (larger if the entries do not fit).
static int str_index_build(vb_shuf *s, u32 log_cap)
{
    StrState *t = s->str;
    vb_ctx *c = s->ctx;
    for (;;) {
        if (log_cap > STR_MAX_LOG_CAP) return set_err(VB_ERR_TOO_LARGE, "string-key index beyond 2^%u slots", STR_MAX_LOG_CAP);
        const u64 cap = 1ull << log_cap;
        DevBuf fp(c), id(c);
        TRY(fp.alloc(cap * 8));
        TRY(id.alloc(cap * 4));
        CU(cudaMemsetAsync(fp.p, 0, cap * 8, c->stream));
        CU(cudaMemsetAsync(id.p, 0xFF, cap * 4, c->stream));
        StrDict nd = t->d;
        nd.fp = fp.as<u64>();
        nd.id = id.as<u32>();
        nd.log_cap = log_cap;
        u32 abort = 0;
        if (t->n_e) {
            CU(cudaMemsetAsync(&t->ctl->abort, 0, 4, c->stream));
            KLaunch kl(s, K_DICT, t->n_e);
            const u64 blocks = std::min<u64>((t->n_e + 255) / 256, (u64)c->sm_count * 8);
            str_index_rebuild_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(nd, t->n_e, t->ctl);
            TRY(kl.done("str_index_rebuild_kernel"));
            TRY(fetch_status_unlocked(c, &t->ctl->abort, &abort, 4));
        }
        if (!abort) {
            dev_free(c, t->d.fp);
            dev_free(c, t->d.id);
            t->d = nd;
            fp.release();
            id.release();
            s->st.table_slots = std::max<u64>(s->st.table_slots, cap);
            return VB_OK;
        }
        ++log_cap;
    }
}

// Key offsets of one call: VB_ERR_INVALID when decreasing or beyond n_bytes, VB_ERR_TOO_LARGE for a key of 2^32 bytes
// or more.  Host offsets are checked here, device offsets by str_check_offsets_kernel.  *first / *last: offs[0], offs[n].
static int str_check_offsets(vb_shuf *s, const u64 *offs, u64 n, u64 n_bytes, int loc, u64 *first, u64 *last)
{
    vb_ctx *c = s->ctx;
    u32 flags = 0;
    if (loc == VB_HOST) {
        for (u64 i = 0; i <= n; ++i) {
            if (offs[i] > n_bytes) flags |= 1u;
            if (i < n) {
                if (offs[i + 1] < offs[i]) flags |= 1u;
                else if (offs[i + 1] - offs[i] >= (1ull << 32)) flags |= 2u;
            }
        }
        *first = offs[0];
        *last = offs[n];
    } else {
        DevBuf f(c);
        TRY(f.alloc(4));
        CU(cudaMemsetAsync(f.p, 0, 4, c->stream));
        {
            KLaunch kl(s, K_MISC, n);
            const u64 blocks = std::min<u64>((n + 256) / 256, (u64)c->sm_count * 8);
            str_check_offsets_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(offs, n, n_bytes, f.as<u32>());
            TRY(kl.done("str_check_offsets_kernel"));
        }
        u64 *h = (u64 *)c->h_scratch;
        CU(cudaMemcpyAsync(h, offs, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(h + 1, offs + n, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(h + 2, f.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        *first = h[0];
        *last = h[1];
        flags = (u32)h[2];
    }
    if (flags & 1u) return set_err(VB_ERR_INVALID, "key offsets decrease or exceed n_bytes %llu", (unsigned long long)n_bytes);
    if (flags & 2u) return set_err(VB_ERR_TOO_LARGE, "a key of 2^32 bytes or more");
    return VB_OK;
}

// Entry ids of n keys (key i is bytes[offs[i] - first .. offs[i + 1] - first), n_bytes in all) in the shuffle's
// dictionary, creating the entries of new keys.  A missing index is first sized from (guess, hint); when it fills,
// it grows and the whole call reruns.
//
// Growth rule.  Load: an index holds at most 0.6 of its slots (max_entries), and a call that would pass that grows it
// at least 4x.  Chains: a probe gives up after STR_MAX_PROBE buckets.  Keys that share their full hash share their home
// bucket at every index size, so growth cannot shorten their chain, and keys can be crafted so (MetroHash64_1 is not
// seeded: placement must equal the reference's HashPartitioner).  So a chain abort grows the index at most once per
// call, and only while it holds fewer than twice the call's worst-case key count (entries before the call plus its
// rows); then the call reruns with the probe limit lifted to the bucket count, for the rest of the call.  The load
// bound leaves an empty slot, so every lifted probe ends within the bucket count; equal-hash keys cost their chain's
// length in byte compares, never a failure.  Random keys practically never chain past STR_MAX_PROBE buckets at load
// <= 0.6, so their index sizes are those of the load rule alone.
static int str_encode(vb_shuf *s, const u64 *offs, const unsigned char *bytes, u64 first, u64 n, u64 n_bytes, u64 guess, u64 hint,
                      u32 *ids)
{
    StrState *t = s->str;
    vb_ctx *c = s->ctx;
    TRY(str_reserve(s, (u64)t->n_e + n, t->n_a + n_bytes));
    if (!t->ctl) {
        DevBuf ctl(c);
        TRY(ctl.alloc(sizeof(StrCtl)));
        CU(cudaMemsetAsync(ctl.p, 0, sizeof(StrCtl), c->stream));
        t->ctl = (StrCtl *)ctl.release();
    }
    if (!t->d.fp) TRY(str_index_build(s, choose_log_cap(guess, hint, false, STR_MAX_LOG_CAP, c->l2_bytes, 12)));
    const u64 worst = (u64)t->n_e + n;         // keys the dictionary can hold after this call
    bool lifted = (1ull << t->d.log_cap) >= 2 * worst;
    for (;;) {
        const u64 cap = 1ull << t->d.log_cap, nb = cap / BUCKET;
        const u32 max_entries = (u32)std::min<u64>((cap / 10) * 6, 0xFFFFFFFFull);
        const u32 max_probe = (u32)(lifted || nb < STR_MAX_PROBE ? nb : STR_MAX_PROBE);
        CU(cudaMemsetAsync(&t->ctl->abort, 0, 4, c->stream));
        {
            KLaunch kl(s, K_DICT, n);
            const u64 blocks = std::min<u64>((n + 255) / 256, (u64)c->sm_count * 8);
            if (t->kind == STRKEY_BYTES)
                str_encode_kernel<STRKEY_BYTES><<<(unsigned)blocks, 256, 0, c->stream>>>(offs, bytes, first, n, t->d, t->ctl, max_entries,
                                                                                         max_probe, ids);
            else
                str_encode_kernel<STRKEY_STR><<<(unsigned)blocks, 256, 0, c->stream>>>(offs, bytes, first, n, t->d, t->ctl, max_entries,
                                                                                       max_probe, ids);
            TRY(kl.done("str_encode_kernel"));
        }
        StrCtl h;
        TRY(fetch_status_unlocked(c, t->ctl, &h, sizeof(StrCtl)));
        t->n_e = h.n_entries;
        t->n_a = h.n_arena;
        if (!h.abort) return VB_OK;
        s->st.table_restarts++;                // rerun the whole call, in a larger index or with the limit lifted
        // Below max_entries the abort was a chain of max_probe full buckets; a walk of every bucket fails only when the
        // index is full, which the count then shows.
        const bool chain = h.n_entries < max_entries;
        if (chain) lifted = true;
        if (!chain || cap < 2 * worst) TRY(str_index_build(s, std::max<u32>(t->d.log_cap + 2, ceil_log2_u64(3 * (u64)t->n_e))));
    }
}

// One map call of a string shuffle after the argument checks: the keys' entry ids, and the value columns in[0 .. n_in)
// (a NULL column is neither read nor copied), copied, or borrowed for VB_DEVICE_BORROWED.  A single-column shuffle
// passes its one column (none for COUNT), a combine_by_key shuffle every column an aggregate reads.  Reduce ops keep
// them as the spec's value columns (cols), GROUP as its values (vals).
static int str_map_state(vb_shuf *s)
{
    std::lock_guard<std::mutex> g(s->mu);
    if (s->sealed || s->sealing || s->freed) return set_err(VB_ERR_STATE, "shuffle %llu: map after seal", (unsigned long long)s->id);
    if (s->exported) return set_err(VB_ERR_STATE, "shuffle %llu: map after export", (unsigned long long)s->id);
    return VB_OK;
}

static int str_map_locked(vb_shuf *s, u32 map_id, const uint64_t *key_offsets, const void *key_bytes, u64 n_bytes, const u64 *const *in,
                          u32 n_in, u64 n, int loc, DevBuf *own_vals)
{
    vb_ctx *c = s->ctx;
    KLaunch call(s, -1);
    StrState *t = s->str;
    u64 others = 0;
    for (u32 j = 0; j < s->n_map; ++j)
        if (j != map_id && s->maps[j].present) others += s->maps[j].n_rows;
    if (others + n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "shuffle of %llu rows on one device", (unsigned long long)(others + n));
    DevBuf d_offs(c), d_bytes(c), ids(c);
    DevBuf d_vals[MA_MAX_COLS];
    for (DevBuf &b : d_vals) b.c = c;
    const u64 *offs = key_offsets;
    const unsigned char *bytes = (const unsigned char *)key_bytes;
    u64 first = 0, last = 0;
    if (n) {
        TRY(str_check_offsets(s, key_offsets, n, n_bytes, loc, &first, &last));
        if ((u64)t->n_e + n > 0xFFFFFFFFull) return set_err(VB_ERR_TOO_LARGE, "more than 2^32 - 1 string keys submitted to one shuffle");
        if (loc == VB_HOST) {       // the encode kernel reads key i at bytes + (offs[i] - first)
            TRY(d_offs.alloc((n + 1) * 8));
            TRY(d_bytes.alloc(last - first));
            CU(cudaMemcpyAsync(d_offs.p, key_offsets, (n + 1) * 8, cudaMemcpyHostToDevice, c->stream));
            if (last > first) CU(cudaMemcpyAsync(d_bytes.p, bytes + first, last - first, cudaMemcpyHostToDevice, c->stream));
            s->st.h2d_bytes += (n + 1) * 8 + (last - first);
            offs = d_offs.as<u64>();
            bytes = d_bytes.as<unsigned char>();
        } else {
            bytes = bytes ? bytes + first : nullptr;
        }
        TRY(ids.alloc(n * 4));
        TRY(str_encode(s, offs, bytes, first, n, last - first, n * std::max<u32>(1, s->n_map), s->hint, ids.as<u32>()));
        for (u32 j = 0; j < n_in && loc != VB_DEVICE_BORROWED; ++j) {
            if (!in[j]) continue;
            TRY(d_vals[j].alloc(n * 8));
            CU(cudaMemcpyAsync(d_vals[j].p, in[j], n * 8, loc == VB_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream));
            if (loc == VB_HOST) s->st.h2d_bytes += n * 8;
        }
    }
    MapOut &m = s->maps[map_id];
    if (m.present) {                               // stage resubmission: the new rows replace the old ones
        s->st.rows_in -= m.n_rows;
        free_str_map(s, map_id);
    }
    t->ids[map_id] = (u32 *)ids.release();
    if (n && n_in) {
        t->vals_owned[map_id] = loc != VB_DEVICE_BORROWED;
        for (u32 j = 0; j < n_in; ++j) {
            const u64 *p = loc == VB_DEVICE_BORROWED ? in[j] : (const u64 *)d_vals[j].release();
            if (is_reduce_op(s->agg)) t->cols[map_id].c[j] = p;
            else t->vals[map_id] = p;
        }
    }
    if (n && own_vals) {                           // byte-string values: the references, owned whatever loc is
        t->vals[map_id] = (const u64 *)own_vals->release();
        t->vals_owned[map_id] = 1;
    }
    m.present = true;
    m.n_rows = n;
    s->st.rows_in += n;
    CU(cudaStreamSynchronize(c->stream));          // the caller's key column is free again when the call returns
    TRY(call.done("map"));
    return VB_OK;
}

static int str_map(vb_shuf *s, u32 map_id, const uint64_t *key_offsets, const void *key_bytes, u64 n_bytes, const u64 *const *in, u32 n_in,
                   u64 n, int loc, DevBuf *own_vals = nullptr)
{
    TRY(str_map_state(s));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    return str_map_locked(s, map_id, key_offsets, key_bytes, n_bytes, in, n_in, n, loc, own_vals);
}

// ---- bincode blobs of string reduce ops (Vec<(String, C)>; strkeys.cuh, str_blob_encode_kernel) -------------------
static unsigned str_grid(const vb_ctx *c, u64 x);

// String GROUP and sort shuffles have no blob format yet: a GROUP's Vec<(String, Vec<V>)> would need its own encoder,
// and a sort takes rows, not combined buckets
static int str_blob_check(const vb_shuf *s)
{
    if (s->str->sort || !is_reduce_op(s->agg)) return reject_str(s, "bincode blobs of a GROUP or sort shuffle");
    return VB_OK;
}

static u64 str_blob_bytes(const vb_shuf *s, u32 r)
{
    return 8 + 16 * (s->bucket_off[r + 1] - s->bucket_off[r]) + (s->str->kb_off[r + 1] - s->str->kb_off[r]);
}

// Partition r's blob into dst (device, 16-byte aligned): one output-driven kernel; an empty partition is 8 zero bytes.
// The caller holds c->mu.
static int str_reduce_blob_locked(vb_shuf *s, u32 r, unsigned char *dst)
{
    vb_ctx *c = s->ctx;
    const StrState *t = s->str;
    const u64 b0 = s->bucket_off[r], nk = s->bucket_off[r + 1] - b0, bytes = str_blob_bytes(s, r);
    KLaunch kl(s, K_MISC, nk);
    if (nk) str_blob_encode_kernel<<<str_grid(c, (bytes + 15) / 16), 256, 0, c->stream>>>(t->key_off + b0, t->key_bytes, s->res_cols + b0, nk, bytes, dst);
    else CU(cudaMemsetAsync(dst, 0, 8, c->stream));
    return kl.done("str_blob_encode_kernel");
}

// One map task's combined bucket Vec<(String, C)> of a string reduce op (world == 1).  The host walks the length
// fields (each record's position depends on the lengths before it) and rejects a malformed blob before allocating or
// launching anything; then the blob and its u32 key lengths go to the device, a scan gives the key offsets, and
// str_blob_decode_kernel writes the key bytes and the partials column.  The keys are encoded as a map call's are, and
// the partials kept as the map task's (blob[m]: the seal merges them with the import spec, as it does received
// partials).  A blob replaces an earlier submission of the map id, rows or blob, and rows replace a blob.
static int str_map_blob(vb_shuf *s, u32 map_id, const void *blob, u64 n_bytes, int src_loc)
{
    if (map_id >= s->n_map) return set_err(VB_ERR_INVALID, "map_id %u >= n_map %u", map_id, s->n_map);
    if (n_bytes < 8) return set_err(VB_ERR_INVALID, "corrupted blob: %llu bytes", (unsigned long long)n_bytes);
    vb_ctx *c = s->ctx;
    std::vector<unsigned char> host;
    const unsigned char *b = (const unsigned char *)blob;
    if (src_loc != VB_HOST) {
        host.resize(n_bytes);
        std::lock_guard<std::mutex> lk(c->mu);
        CU(cudaSetDevice(c->device));
        CU(cudaMemcpyAsync(host.data(), blob, n_bytes, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        b = host.data();
    }
    u64 n = 0;
    memcpy(&n, b, 8);
    if (n > (n_bytes - 8) / 16) return set_err(VB_ERR_INVALID, "corrupted blob: %llu records in %llu bytes", (unsigned long long)n, (unsigned long long)n_bytes);
    std::vector<u32> lens(n);
    u64 pos = 8;
    for (u64 i = 0; i < n; ++i) {
        if (n_bytes - pos < 16) return set_err(VB_ERR_INVALID, "corrupted blob: record %llu runs past the end", (unsigned long long)i);
        u64 len = 0;
        memcpy(&len, b + pos, 8);
        if (len > n_bytes - pos - 16) return set_err(VB_ERR_INVALID, "corrupted blob: record %llu has a key of %llu bytes", (unsigned long long)i, (unsigned long long)len);
        if (len >= (1ull << 32)) return set_err(VB_ERR_TOO_LARGE, "a key of 2^32 bytes or more");
        lens[i] = (u32)len;
        pos += 16 + len;
    }
    if (pos != n_bytes) return set_err(VB_ERR_INVALID, "corrupted blob: %llu trailing bytes", (unsigned long long)(n_bytes - pos));
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "map partition of %llu rows", (unsigned long long)n);
    TRY(str_map_state(s));
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    const u64 nkb = n_bytes - 8 - 16 * n;
    DevBuf d_blob(c), d_lens(c), wide(c), koff(c), kbytes(c), vals(c);
    if (n) {
        const unsigned char *db = (const unsigned char *)blob;
        if (src_loc == VB_HOST) {
            TRY(d_blob.alloc(n_bytes));
            CU(cudaMemcpyAsync(d_blob.p, blob, n_bytes, cudaMemcpyHostToDevice, c->stream));
            s->st.h2d_bytes += n_bytes;
            db = d_blob.as<unsigned char>();
        }
        TRY(d_lens.alloc(n * 4));
        CU(cudaMemcpyAsync(d_lens.p, lens.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
        s->st.h2d_bytes += n * 4;
        TRY(wide.alloc(n * 8));
        TRY(koff.alloc((n + 1) * 8));
        {
            KLaunch kl(s, K_MISC, n);
            str_widen_u32_kernel<<<str_grid(c, n), 256, 0, c->stream>>>(d_lens.as<u32>(), n, wide.as<u64>());
            TRY(kl.done("str_widen_u32_kernel"));
        }
        TRY(exclusive_scan_u64(s, wide.as<u64>(), koff.as<u64>(), n, koff.as<u64>() + n));
        TRY(kbytes.alloc((nkb + 15) & ~15ull));
        TRY(vals.alloc(n * 8));
        {
            KLaunch kl(s, K_MISC, n);
            str_blob_decode_kernel<<<str_grid(c, std::max<u64>(n, (nkb + 15) / 16)), 256, 0, c->stream>>>(db, koff.as<u64>(), n, kbytes.as<unsigned char>(),
                                                                                                      vals.as<u64>());
            TRY(kl.done("str_blob_decode_kernel"));
        }
    }
    TRY(str_map_locked(s, map_id, koff.as<u64>(), kbytes.p, nkb, nullptr, 0, n, VB_DEVICE, &vals));
    s->str->blob[map_id] = 1;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_map_str(vb_shuf *s, uint32_t map_id, const uint64_t *key_offsets, const void *key_bytes, uint64_t n_bytes,
                                      const void *vals, uint64_t n, int32_t loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->str) return set_err(VB_ERR_INVALID, "vb_shuffle_map_str needs a shuffle from vb_shuffle_create_str");
    if (s->multi) return set_err(VB_ERR_INVALID, "shuffle %llu has several aggregates per key: map it with vb_shuffle_map_str_cols", (unsigned long long)s->id);
    if (s->vdt == VB_BYTES) return set_err(VB_ERR_INVALID, "shuffle %llu has byte-string values: map it with vb_shuffle_map_str_bytes", (unsigned long long)s->id);
    if (map_id >= s->n_map) return set_err(VB_ERR_INVALID, "map_id %u >= n_map %u", map_id, s->n_map);
    if (loc < VB_HOST || loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc %d", loc);
    if (n && !key_offsets) return set_err(VB_ERR_INVALID, "NULL key_offsets with n_rows > 0");
    if (n && n_bytes && !key_bytes) return set_err(VB_ERR_INVALID, "NULL key_bytes with n_bytes > 0");
    const bool sort = s->str->sort;
    if (sort && !s->str->sort_vals && vals) return set_err(VB_ERR_INVALID, "shuffle %llu sorts keys only: vals must be NULL", (unsigned long long)s->id);
    if (n && !vals && (sort ? s->str->sort_vals : s->agg != VB_AGG_COUNT)) return set_err(VB_ERR_INVALID, "values required for this aggregator");
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "map partition of %llu rows", (unsigned long long)n);
    const u64 *col = (const u64 *)vals;
    const u32 n_in = sort ? (s->str->sort_vals ? 1u : 0u) : (s->agg != VB_AGG_COUNT ? 1u : 0u);
    return str_map(s, map_id, key_offsets, key_bytes, n_bytes, &col, n_in, n, loc);
}

extern "C" int32_t vb_shuffle_map_str_cols(vb_shuf *s, uint32_t map_id, const uint64_t *key_offsets, const void *key_bytes, uint64_t n_bytes,
                                           const void *const *vals, uint64_t n, int32_t loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->str || !s->multi) return set_err(VB_ERR_INVALID, "vb_shuffle_map_str_cols needs a shuffle from vb_shuffle_create_str_multi");
    if (map_id >= s->n_map) return set_err(VB_ERR_INVALID, "map_id %u >= n_map %u", map_id, s->n_map);
    if (loc < VB_HOST || loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc %d", loc);
    if (n && !key_offsets) return set_err(VB_ERR_INVALID, "NULL key_offsets with n_rows > 0");
    if (n && n_bytes && !key_bytes) return set_err(VB_ERR_INVALID, "NULL key_bytes with n_bytes > 0");
    const u64 *cols[MA_MAX_COLS] = {};
    bool read[MA_MAX_COLS] = {};
    for (u32 a = 0; a < s->acc_map.n; ++a)
        if (spec_at(s->acc_map.op, a) != OPK_COUNT) read[spec_at(s->acc_map.src, a)] = true;
    for (u32 i = 0; vals && i < s->n_cols; ++i) cols[i] = read[i] ? (const u64 *)vals[i] : nullptr;   // an unread column is not copied
    for (u32 i = 0; i < s->n_cols; ++i)
        if (n && read[i] && !cols[i]) return set_err(VB_ERR_INVALID, "value column %u is read by an aggregate but NULL", i);
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "map partition of %llu rows", (unsigned long long)n);
    return str_map(s, map_id, key_offsets, key_bytes, n_bytes, cols, s->n_cols, n, loc);
}

// ---------------------------------------------------------------------------------------------
// byte-string values (bytevals.cuh): a map call copies its values into a store of the shuffle and maps the rows'
// references as ordinary u64 values; vb_shuffle_gather_bytes* turn references back into bytes
// ---------------------------------------------------------------------------------------------
static int bytes_check_args(vb_shuf *s, u32 map_id, const u64 *val_offsets, const void *val_bytes, u64 n_val_bytes, u64 n, int loc)
{
    if (map_id >= s->n_map) return set_err(VB_ERR_INVALID, "map_id %u >= n_map %u", map_id, s->n_map);
    if (loc < VB_HOST || loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc %d", loc);
    if (n && !val_offsets) return set_err(VB_ERR_INVALID, "NULL val_offsets with n_rows > 0");
    if (n && n_val_bytes && !val_bytes) return set_err(VB_ERR_INVALID, "NULL val_bytes with n_val_bytes > 0");
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "map partition of %llu rows", (unsigned long long)n);
    std::lock_guard<std::mutex> g(s->mu);
    if (s->sealed || s->sealing || s->freed) return set_err(VB_ERR_STATE, "shuffle %llu: map after seal", (unsigned long long)s->id);
    if (s->exported) return set_err(VB_ERR_STATE, "shuffle %llu: map after export", (unsigned long long)s->id);
    return VB_OK;
}

// One map task's values: the checked offsets rebased to 0 and the bytes, copied into *st, and the task's references
// ((map_id + 1) << 32 | row) in refs.  The caller's buffers are free again when it returns.
static int bytes_store(vb_shuf *s, u32 map_id, const u64 *val_offsets, const void *val_bytes, u64 n_val_bytes, u64 n, int loc,
                       ByteSrc *st, DevBuf &refs)
{
    *st = ByteSrc{nullptr, nullptr, 0};
    if (n == 0) return VB_OK;
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    const int in = loc == VB_HOST ? VB_HOST : VB_DEVICE;
    u64 first = 0, last = 0;
    const int rc = str_check_offsets(s, val_offsets, n, n_val_bytes, in, &first, &last);
    if (rc == VB_ERR_INVALID) return set_err(rc, "value offsets decrease or exceed n_val_bytes %llu", (unsigned long long)n_val_bytes);
    if (rc == VB_ERR_TOO_LARGE) return set_err(rc, "a value of 2^32 bytes or more");
    TRY(rc);
    const cudaMemcpyKind kind = in == VB_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
    DevBuf offs(c), bytes(c), staged(c);
    TRY(offs.alloc((n + 1) * 8));
    TRY(bytes.alloc(last - first));
    TRY(refs.alloc(n * 8));
    const u64 *src_offs = val_offsets;
    if (in == VB_HOST) {
        TRY(staged.alloc((n + 1) * 8));
        CU(cudaMemcpyAsync(staged.p, val_offsets, (n + 1) * 8, kind, c->stream));
        s->st.h2d_bytes += (n + 1) * 8 + (last - first);
        src_offs = staged.as<u64>();
    }
    if (last > first) CU(cudaMemcpyAsync(bytes.p, (const unsigned char *)val_bytes + first, last - first, kind, c->stream));
    {
        KLaunch kl(s, K_MISC, n);
        rebase_kernel<<<(unsigned)((n + 256) / 256), 256, 0, c->stream>>>(src_offs, n + 1, first, offs.as<u64>());   // one thread per offset
        TRY(kl.done("rebase_kernel"));
    }
    {
        KLaunch kl(s, K_MISC, n);
        const unsigned blocks = (unsigned)std::min<u64>((n + 255) / 256, (u64)c->sm_count * 8);
        bytes_refs_kernel<<<blocks, 256, 0, c->stream>>>((u64)(map_id + 1) << 32, n, refs.as<u64>());
        TRY(kl.done("bytes_refs_kernel"));
    }
    CU(cudaStreamSynchronize(c->stream));
    *st = ByteSrc{(const u64 *)offs.release(), (const unsigned char *)bytes.release(), n};
    return VB_OK;
}

// After the map call: on success the new store replaces the map id's old one, otherwise it is dropped
static int bytes_keep(vb_shuf *s, u32 map_id, const ByteSrc &st, int rc)
{
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    cudaSetDevice(c->device);
    const ByteSrc &drop = rc == VB_OK ? s->bvals[map_id] : st;
    dev_free(c, drop.offs);
    dev_free(c, drop.bytes);
    if (rc == VB_OK) s->bvals[map_id] = st;
    return rc;
}

extern "C" int32_t vb_shuffle_map_bytes(vb_shuf *s, uint32_t map_id, const void *keys, const uint64_t *val_offsets, const void *val_bytes,
                                        uint64_t n_val_bytes, uint64_t n, int32_t loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (s->vdt != VB_BYTES || s->str || s->bvals.size() < s->n_map)
        return set_err(VB_ERR_INVALID, "vb_shuffle_map_bytes needs an integer-key shuffle of VB_BYTES values");
    if (n && !keys) return set_err(VB_ERR_INVALID, "NULL keys with n_rows > 0");
    TRY(bytes_check_args(s, map_id, val_offsets, val_bytes, n_val_bytes, n, loc));
    ByteSrc st;
    DevBuf refs(s->ctx);
    TRY(bytes_store(s, map_id, val_offsets, val_bytes, n_val_bytes, n, loc, &st, refs));
    return bytes_keep(s, map_id, st, shuffle_map(s, map_id, nullptr, (const u64 *)keys, nullptr, n, loc, false, nullptr, &refs));
}

extern "C" int32_t vb_shuffle_map_str_bytes(vb_shuf *s, uint32_t map_id, const uint64_t *key_offsets, const void *key_bytes, uint64_t n_key_bytes,
                                            const uint64_t *val_offsets, const void *val_bytes, uint64_t n_val_bytes, uint64_t n, int32_t loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (s->vdt != VB_BYTES || !s->str || s->multi || s->bvals.size() < s->n_map)
        return set_err(VB_ERR_INVALID, "vb_shuffle_map_str_bytes needs a string-key shuffle of VB_BYTES values");
    if (n && !key_offsets) return set_err(VB_ERR_INVALID, "NULL key_offsets with n_rows > 0");
    if (n && n_key_bytes && !key_bytes) return set_err(VB_ERR_INVALID, "NULL key_bytes with n_key_bytes > 0");
    TRY(bytes_check_args(s, map_id, val_offsets, val_bytes, n_val_bytes, n, loc));
    ByteSrc st;
    DevBuf refs(s->ctx);
    TRY(bytes_store(s, map_id, val_offsets, val_bytes, n_val_bytes, n, loc, &st, refs));
    const u64 *none = nullptr;   // the value column is the references (refs), not a caller column
    return bytes_keep(s, map_id, st, str_map(s, map_id, key_offsets, key_bytes, n_key_bytes, &none, 1, n, loc, &refs));
}

// Lengths of n references (copied to the device first when on the host) into lens, and their exclusive scan into
// offs [n + 1]; VB_ERR_INVALID, with offs untouched, when one of them was not issued by s.  Caller holds c->mu.
static int bytes_offsets(vb_shuf *s, const u64 *refs_in, u64 n, int src_loc, DevBuf &refs, u64 *offs, u64 *total)
{
    vb_ctx *c = s->ctx;
    *total = 0;
    if (!s->bvals_dev) {
        DevBuf t(c);
        TRY(t.alloc(s->bvals.size() * sizeof(ByteSrc)));
        CU(cudaMemcpyAsync(t.p, s->bvals.data(), s->bvals.size() * sizeof(ByteSrc), cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));   // pageable source
        s->bvals_dev = t.as<ByteSrc>();
        t.release();
    }
    if (n == 0) { CU(cudaMemsetAsync(offs, 0, 8, c->stream)); return VB_OK; }
    const u64 *r = refs_in;
    if (src_loc == VB_HOST) {
        TRY(refs.alloc(n * 8));
        CU(cudaMemcpyAsync(refs.p, refs_in, n * 8, cudaMemcpyHostToDevice, c->stream));
        s->st.h2d_bytes += n * 8;
        r = refs.as<u64>();
    }
    DevBuf lens(c), bad(c);
    TRY(lens.alloc(n * 8));
    TRY(bad.alloc(4));
    CU(cudaMemsetAsync(bad.p, 0, 4, c->stream));
    {
        KLaunch kl(s, K_MISC, n);
        const unsigned blocks = (unsigned)std::min<u64>((n + 255) / 256, (u64)c->sm_count * 8);
        bytes_len_kernel<<<blocks, 256, 0, c->stream>>>(r, n, s->bvals_dev, (u32)s->bvals.size(), lens.as<u64>(), bad.as<u32>());
        TRY(kl.done("bytes_len_kernel"));
    }
    u32 h_bad = 0;
    TRY(fetch_status_unlocked(c, bad.p, &h_bad, 4));
    if (h_bad) return set_err(VB_ERR_INVALID, "shuffle %llu: a reference it did not issue", (unsigned long long)s->id);
    TRY(exclusive_scan_u64(s, lens.as<u64>(), offs, n, offs + n));
    return fetch_status_unlocked(c, offs + n, total, 8);
}

// out [total] = the values of the n device references refs at the offsets offs (bytes_offsets)
static int bytes_gather_launch(vb_shuf *s, const u64 *refs, u64 n, const u64 *offs, u64 total, unsigned char *out)
{
    vb_ctx *c = s->ctx;
    const u64 tiles = (n + total + GB_ITEMS - 1) / GB_ITEMS;
    const u64 grid = std::min<u64>(tiles, (u64)c->sm_count * occupancy(c, bytes_gather_kernel, GB_THREADS, 0));
    KLaunch kl(s, K_MISC, n);
    bytes_gather_kernel<<<(unsigned)grid, GB_THREADS, 0, c->stream>>>(refs, n, offs, total, s->bvals_dev, (u32)s->bvals.size(), out);
    return kl.done("bytes_gather_kernel");
}

static int bytes_gather_check(vb_shuf *s, const void *refs, u64 n, int src_loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (s->vdt != VB_BYTES || s->bvals.size() < s->n_map) return set_err(VB_ERR_INVALID, "shuffle %llu has no byte-string values", (unsigned long long)s->id);
    if (n && !refs) return set_err(VB_ERR_INVALID, "NULL refs with n > 0");
    if (src_loc < VB_HOST || src_loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc %d", src_loc);
    return wait_sealed(s);
}

extern "C" int32_t vb_shuffle_gather_bytes_size(vb_shuf *s, const uint64_t *refs, uint64_t n, int32_t src_loc, uint64_t *n_bytes)
{
    if (!n_bytes) return set_err(VB_ERR_INVALID, "NULL n_bytes");
    TRY(bytes_gather_check(s, refs, n, src_loc));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    DevBuf r(c), offs(c);
    TRY(offs.alloc((n + 1) * 8));
    u64 total = 0;
    TRY(bytes_offsets(s, refs, n, src_loc, r, offs.as<u64>(), &total));
    *n_bytes = total;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_gather_bytes(vb_shuf *s, const uint64_t *refs, uint64_t n, int32_t src_loc, uint64_t *out_offsets,
                                           void *out_bytes, int32_t dst_loc)
{
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    if (!out_offsets) return set_err(VB_ERR_INVALID, "NULL out_offsets");
    TRY(bytes_gather_check(s, refs, n, src_loc));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    DevBuf r(c), offs_tmp(c), bytes_tmp(c);
    // the offsets go straight to a device caller only when nothing can fail after them: with out_bytes NULL the
    // total decides whether the call is valid, so they are scanned into a buffer of the library first
    u64 *offs = out_offsets;
    const bool staged = dst_loc == VB_HOST || !out_bytes;
    if (staged) { TRY(offs_tmp.alloc((n + 1) * 8)); offs = offs_tmp.as<u64>(); }
    u64 total = 0;
    TRY(bytes_offsets(s, refs, n, src_loc, r, offs, &total));
    if (total && !out_bytes) return set_err(VB_ERR_INVALID, "NULL out_bytes for %llu bytes", (unsigned long long)total);
    unsigned char *dst = (unsigned char *)out_bytes;
    if (total && dst_loc == VB_HOST) { TRY(bytes_tmp.alloc(total)); dst = bytes_tmp.as<unsigned char>(); }
    if (total) TRY(bytes_gather_launch(s, src_loc == VB_HOST ? r.as<u64>() : refs, n, offs, total, dst));
    if (staged) {
        TRY(copy_out(s, out_offsets, offs, (n + 1) * 8, dst_loc));
    }
    if (dst_loc == VB_HOST) {
        TRY(copy_out(s, out_bytes, dst, total, VB_HOST));
    }
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// repartition (Rdd::repartition = coalesce(n, shuffle = true), rdd.rs:386-418): row i of map m is placed by
// HashPartitioner::<usize> at position start_m + 1 + i.  The seal is one stable multisplit whose loader computes each
// row's position from its index (LD_POS): no key column exists, and each partition holds its rows in map-id, then
// input order.
// ---------------------------------------------------------------------------------------------
struct RepMapIn {
    bool present = false;
    bool owned = false;          // the columns are copies owned by the shuffle (not VB_DEVICE_BORROWED)
    u64 n_rows = 0;
    u64 start = 0;               // first_position
    const u64 *cols[2] = {};
};

struct RepState {
    u32 n_cols = 0;
    bool bytes = false;
    std::vector<RepMapIn> maps;
    u64 n = 0;                   // sealed rows
    u64 *cols = nullptr;         // [n_cols][n] item columns, partition r at rows [bucket_off[r], bucket_off[r + 1])
    u64 *refs = nullptr;         // bytes: [n] row references in the same order, gathered by the byte-string copy path
};

static int reject_rep(const vb_shuf *s, const char *what)
{
    return set_err(VB_ERR_INVALID, "shuffle %llu is a repartition shuffle: %s does not apply to it", (unsigned long long)s->id, what);
}

static void free_rep_map(vb_ctx *c, RepMapIn &m)
{
    if (m.owned) { dev_free(c, m.cols[0]); dev_free(c, m.cols[1]); }
    m = RepMapIn();
}

static void free_rep(vb_shuf *s)
{
    if (!s->rep) return;
    for (RepMapIn &m : s->rep->maps) free_rep_map(s->ctx, m);
    dev_free(s->ctx, s->rep->cols);
    dev_free(s->ctx, s->rep->refs);
    delete s->rep;
    s->rep = nullptr;
}

extern "C" int32_t vb_shuffle_create_repartition_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t n_cols,
                                                      int32_t has_bytes, uint32_t rank, uint32_t world, vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_repartition: NULL argument");
    *out = nullptr;
    if (world < 1 || world > 256 || rank >= world) return set_err(VB_ERR_INVALID, "vb_shuffle_create_repartition_dist: bad rank %u / world %u", rank, world);
    if (n_reduce < 1) return set_err(VB_ERR_INVALID, "vb_shuffle_create_repartition: n_reduce must be >= 1");
    if (has_bytes != 0 && has_bytes != 1) return set_err(VB_ERR_INVALID, "vb_shuffle_create_repartition: has_bytes must be 0 or 1");
    if (n_cols > 2 || (n_cols == 0 && !has_bytes))
        return set_err(VB_ERR_INVALID, "vb_shuffle_create_repartition: items are 0 to 2 64-bit columns plus an optional byte-string column, at least one column in all");
    if (n_reduce > 65536) return set_err(VB_ERR_UNSUPPORTED, "more than 65536 reduce partitions");
    vb_shuf *s = new vb_shuf();
    s->uid = next_uid.fetch_add(1);
    s->ctx = c;
    s->id = shuffle_id;
    s->n_map = n_map;
    s->n_reduce = n_reduce;
    s->kdt = VB_U64;
    s->vdt = VB_U64;
    s->agg = -1;                  // no aggregator: every GROUP / reduce / sort path refuses the shuffle
    s->part = VB_PART_HASH_METRO64;
    s->rep = new RepState();
    s->rep->n_cols = n_cols;
    s->rep->bytes = has_bytes == 1;
    s->rep->maps.resize(n_map);
    if (has_bytes) s->bvals.assign(n_map, ByteSrc{nullptr, nullptr, 0});
    s->rank = rank;
    s->world = world;
    *out = s;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_create_repartition(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t n_cols,
                                                 int32_t has_bytes, vb_shuf **out)
{
    return vb_shuffle_create_repartition_dist(c, shuffle_id, n_map, n_reduce, n_cols, has_bytes, 0, 1, out);
}

extern "C" int32_t vb_shuffle_map_repartition(vb_shuf *s, uint32_t map_id, uint64_t first_position, const void *const *cols,
                                              const uint64_t *val_offsets, const void *val_bytes, uint64_t n_val_bytes, uint64_t n,
                                              int32_t loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->rep) return set_err(VB_ERR_INVALID, "vb_shuffle_map_repartition needs a shuffle from vb_shuffle_create_repartition");
    RepState *rs = s->rep;
    if (map_id >= s->n_map) return set_err(VB_ERR_INVALID, "map_id %u >= n_map %u", map_id, s->n_map);
    if (loc < VB_HOST || loc > VB_DEVICE_BORROWED) return set_err(VB_ERR_INVALID, "bad src_loc %d", loc);
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->exported) return set_err(VB_ERR_STATE, "shuffle %llu: map after exchange", (unsigned long long)s->id);
    }
    for (u32 k = 0; k < rs->n_cols; ++k)
        if (n && (!cols || !cols[k])) return set_err(VB_ERR_INVALID, "NULL item column %u with n_rows > 0", k);
    if (rs->bytes && n && !val_offsets) return set_err(VB_ERR_INVALID, "NULL val_offsets with n_rows > 0");
    if (rs->bytes && n && n_val_bytes && !val_bytes) return set_err(VB_ERR_INVALID, "NULL val_bytes with n_val_bytes > 0");
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "map partition of %llu rows", (unsigned long long)n);
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->sealing || s->freed) return set_err(VB_ERR_STATE, "shuffle %llu: map after seal", (unsigned long long)s->id);
    }
    vb_ctx *c = s->ctx;
    ByteSrc st{nullptr, nullptr, 0};
    if (rs->bytes) {
        DevBuf refs(c);   // bytes_store's references are not kept: a repartition computes them from the row index
        TRY(bytes_store(s, map_id, val_offsets, val_bytes, n_val_bytes, n, loc, &st, refs));
    }
    auto columns = [&]() -> int {
        std::lock_guard<std::mutex> lk(c->mu);
        CU(cudaSetDevice(c->device));
        RepMapIn in;
        in.present = true;
        in.n_rows = n;
        in.start = first_position;
        if (n && loc == VB_DEVICE_BORROWED) {
            for (u32 k = 0; k < rs->n_cols; ++k) in.cols[k] = (const u64 *)cols[k];
        } else if (n && rs->n_cols) {
            const cudaMemcpyKind kind = loc == VB_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
            DevBuf b0(c), b1(c);
            DevBuf *b[2] = {&b0, &b1};
            for (u32 k = 0; k < rs->n_cols; ++k) {
                TRY(b[k]->alloc(n * 8));
                CU(cudaMemcpyAsync(b[k]->p, cols[k], n * 8, kind, c->stream));
                if (loc == VB_HOST) s->st.h2d_bytes += n * 8;
            }
            CU(cudaStreamSynchronize(c->stream));      // the caller may reuse its buffers on return
            for (u32 k = 0; k < rs->n_cols; ++k) in.cols[k] = (const u64 *)b[k]->release();
            in.owned = true;
        }
        RepMapIn &m = rs->maps[map_id];
        if (m.present) s->st.rows_in -= m.n_rows;     // resubmission: the last submission wins
        free_rep_map(c, m);
        m = in;
        s->st.rows_in += n;
        return VB_OK;
    };
    const int rc = columns();
    return rs->bytes ? bytes_keep(s, map_id, st, rc) : rc;
}

// out[k * n + i] = item column k of the row with reference refs[i]; src[k * n_map + m] is map m's column k
__global__ void rep_gather_kernel(const u64 *__restrict__ refs, u64 n, const u64 *const *__restrict__ src, u32 n_map, u32 n_cols,
                                  u64 *__restrict__ out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u64 ref = refs[i];
        const u32 m = (u32)(ref >> 32) - 1;
        const u64 r = ref & 0xFFFFFFFFull;
        for (u32 k = 0; k < n_cols; ++k) out[(u64)k * n + i] = src[(u64)k * n_map + m][r];
    }
}

// One stable multisplit of every row by the partition of its position (multisplit: one pass for <= 256 partitions,
// two LSD passes over the 16-bit partition id above).  An item of one 64-bit column moves as the pass's value; any
// other item moves as its row reference, and a gather then reads its columns.
static int seal_rep(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    RepState *rs = s->rep;
    const u32 M = s->n_map, R = s->n_reduce;
    const bool direct = rs->n_cols == 1 && !rs->bytes;
    std::vector<RepMap> h((size_t)M + 1);
    u64 n = 0;
    for (u32 m = 0; m < M; ++m) {
        const RepMapIn &mi = rs->maps[m];
        if (!mi.present && s->world == 1) return set_err(VB_ERR_STATE, "shuffle %llu sealed but map %u was never submitted", (unsigned long long)s->id, m);
        h[m] = RepMap{n, mi.start, direct ? mi.cols[0] : nullptr};
        n += mi.n_rows;
    }
    h[M] = RepMap{n, 0, nullptr};
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "shuffle of %llu rows on one device", (unsigned long long)n);
    s->bucket_off.assign((size_t)R + 1, 0);
    rs->n = n;
    if (n == 0) return VB_OK;
    DevBuf tab(c), pos(c), vals(c);
    TRY(tab.alloc(h.size() * sizeof(RepMap)));
    CU(cudaMemcpyAsync(tab.p, h.data(), h.size() * sizeof(RepMap), cudaMemcpyHostToDevice, c->stream));
    TRY(pos.alloc(n * 8));
    TRY(vals.alloc(n * 8));
    TRY(multisplit(s, Loader{LD_POS, tab.p, nullptr, M}, n, DG_BUCKET, R, n, pos.as<u64>(), vals.as<u64>(), s->bucket_off));
    if (direct) {
        rs->cols = vals.as<u64>();
        vals.release();
    } else {
        if (rs->n_cols) {
            std::vector<const u64 *> hs((size_t)rs->n_cols * M);
            for (u32 k = 0; k < rs->n_cols; ++k)
                for (u32 m = 0; m < M; ++m) hs[(size_t)k * M + m] = rs->maps[m].cols[k];
            DevBuf src(c), out(c);
            TRY(src.alloc(hs.size() * sizeof(u64 *)));
            TRY(out.alloc((u64)rs->n_cols * n * 8));
            CU(cudaMemcpyAsync(src.p, hs.data(), hs.size() * sizeof(u64 *), cudaMemcpyHostToDevice, c->stream));
            {
                KLaunch kl(s, K_MISC, n);
                const unsigned blocks = (unsigned)std::min<u64>((n + 255) / 256, (u64)c->sm_count * 8);
                rep_gather_kernel<<<blocks, 256, 0, c->stream>>>(vals.as<u64>(), n, (const u64 *const *)src.p, M, rs->n_cols, out.as<u64>());
                TRY(kl.done("rep_gather_kernel"));
            }
            CU(cudaStreamSynchronize(c->stream));      // pageable sources of the two tables
            rs->cols = out.as<u64>();
            out.release();
        }
        if (rs->bytes) { rs->refs = vals.as<u64>(); vals.release(); }
    }
    CU(cudaStreamSynchronize(c->stream));
    for (RepMapIn &m : rs->maps) {             // the items now live in the result (the byte stores stay for the gather)
        if (m.owned) { dev_free(c, m.cols[0]); dev_free(c, m.cols[1]); }
        m.cols[0] = m.cols[1] = nullptr;
        m.owned = false;
    }
    s->st.rows_out = n;
    return VB_OK;
}

// Across ranks (vb_shuffle_exchange): the rank's own map tasks are split by output partition with the one-process seal,
// every partition's run goes to its owner (p % world) in one grouped send/recv, as the sort exchange sends them, and the
// owner appends the runs in source-rank order, which is map-id order because map ids are assigned in contiguous blocks
// by rank.  The count all-gather carries each rank's rows, n_cols and has_bytes; a second all-gather carries the rows
// (and bytes) of every partition.  Every limit and the agreement of n_cols and has_bytes are checked on every rank from
// the gathered counts, so all ranks return the same code before any send.
static int exchange_rep_locked(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    RepState *rs = s->rep;
    const u32 W = m->world, me = m->rank, R = s->n_reduce, K = rs->n_cols;
    auto clk = std::chrono::steady_clock::now();
    u64 n_local = 0;
    for (const RepMapIn &mi : rs->maps) n_local += mi.present ? mi.n_rows : 0;
    const u64 row[3] = {n_local, K, rs->bytes ? 1ull : 0ull};
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, row, 3, &mat));
    s->xst.counts_wall_ms += lap(clk);
    for (u32 r = 0; r < W; ++r) {
        if (mat[3 * r + 1] != K || mat[3 * r + 2] != row[2])
            return set_err(VB_ERR_INVALID, "repartition across ranks: rank %u has %llu columns and has_bytes %llu, rank %u %u and %llu", r,
                           (unsigned long long)mat[3 * r + 1], (unsigned long long)mat[3 * r + 2], me, K, (unsigned long long)row[2]);
        if (mat[3 * r] >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "rank %u maps %llu rows", r, (unsigned long long)mat[3 * r]);
    }
    // 1. the local split: partition p's rows at [bucket_off[p], bucket_off[p + 1]) of rs->cols / rs->refs
    TRY(seal_rep(s));
    const u64 nl = rs->n;
    const std::vector<u64> cut = s->bucket_off;
    std::vector<u64> bat;
    if (rs->bytes) TRY(bytes_pack(s, rs->refs, nl, cut, bat));
    s->xst.prepare_wall_ms += lap(clk);
    // 2. rows (and bytes) of every partition on every rank
    const u32 SR = rs->bytes ? 2 * R : R;
    std::vector<u64> seg(SR), segall((size_t)W * SR);
    for (u32 p = 0; p < R; ++p) {
        seg[p] = cut[p + 1] - cut[p];
        if (rs->bytes) seg[R + p] = bat[p + 1] - bat[p];
    }
    DevBuf d_seg(c), d_segall(c);
    TRY(d_seg.alloc((size_t)SR * 8));
    TRY(d_segall.alloc((size_t)W * SR * 8));
    CU(cudaMemcpyAsync(d_seg.p, seg.data(), (size_t)SR * 8, cudaMemcpyHostToDevice, c->stream));
    NC(g_nccl.AllGather(d_seg.p, d_segall.p, SR, ncclUint64, m->comm, c->stream));
    CU(cudaMemcpyAsync(segall.data(), d_segall.p, (size_t)W * SR * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (u32 d = 0; d < W; ++d) {                 // every rank's receive total, so that all ranks refuse alike
        u64 nd = 0;
        for (u32 p = d; p < R; p += W)
            for (u32 r = 0; r < W; ++r) nd += segall[(size_t)r * SR + p];
        if (nd >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "rank %u would receive %llu rows", d, (unsigned long long)nd);
    }
    std::vector<u64> off((size_t)R + 1, 0);
    u64 nb_recv = 0;
    for (u32 p = 0; p < R; ++p) {
        u64 np = 0;
        if (p % W == me)
            for (u32 r = 0; r < W; ++r) {
                np += segall[(size_t)r * SR + p];
                if (rs->bytes) nb_recv += segall[(size_t)r * SR + R + p];
            }
        off[p + 1] = off[p] + np;
    }
    const u64 n_recv = off[R];
    // 3. one grouped send/recv: partition-major, source-rank-major at the owner
    DevBuf rc(c), rl(c), rb(c), refs(c);
    TRY(rc.alloc((u64)K * n_recv * 8));
    if (rs->bytes) { TRY(rl.alloc(n_recv * 4)); TRY(rb.alloc(nb_recv)); }
    std::vector<Xfer> xs;
    u64 sent = 0, own = 0;
    for (u32 p = 0; p < R; ++p) {
        for (u32 k = 0; k < K; ++k) xs.push_back(Xfer{true, p % W, rs->cols + (u64)k * nl + cut[p], seg[p], ncclUint64});
        if (rs->bytes) {
            xs.push_back(Xfer{true, p % W, s->bx_lens + cut[p], seg[p], ncclUint32});
            xs.push_back(Xfer{true, p % W, s->bx_bytes + bat[p], seg[R + p], ncclUint8});
        }
        (p % W == me ? own : sent) += seg[p];
    }
    u64 boff = 0;
    for (u32 p = me; p < R; p += W) {
        u64 o = off[p];
        for (u32 r = 0; r < W; ++r) {
            const u64 cnt = segall[(size_t)r * SR + p];
            for (u32 k = 0; k < K; ++k) xs.push_back(Xfer{false, r, rc.as<u64>() + (u64)k * n_recv + o, cnt, ncclUint64});
            if (rs->bytes) {
                const u64 nb = segall[(size_t)r * SR + R + p];
                xs.push_back(Xfer{false, r, rl.as<u32>() + o, cnt, ncclUint32});
                xs.push_back(Xfer{false, r, rb.as<unsigned char>() + boff, nb, ncclUint8});
                boff += nb;
            }
            o += cnt;
        }
    }
    TRY(post_group(s, xs));
    if (rs->bytes) TRY(bytes_adopt(s, rl.as<u32>(), n_recv, rb, nb_recv, refs));   // synchronises the stream
    CU(cudaStreamSynchronize(c->stream));
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_NCCL, sent, n_recv - own);
    dev_free(c, rs->cols);
    dev_free(c, rs->refs);
    dev_free(c, s->bx_lens);
    dev_free(c, s->bx_bytes);
    s->bx_lens = nullptr;
    s->bx_bytes = nullptr;
    rs->cols = K ? rc.as<u64>() : nullptr;
    if (K) rc.release();
    rs->refs = rs->bytes ? refs.as<u64>() : nullptr;
    if (rs->bytes) refs.release();
    rs->n = n_recv;
    s->bucket_off = off;
    s->st.rows_out = n_recv;
    std::lock_guard<std::mutex> g(s->mu);
    s->exported = s->imported = true;
    return VB_OK;
}

static int exchange_rep(vb_shuf *s, int mode)
{
    vb_ctx *c = s->ctx;
    if (mode < VB_XCHG_AUTO || mode > VB_XCHG_P2P) return set_err(VB_ERR_INVALID, "bad exchange mode");
    if (mode == VB_XCHG_P2P) return set_err(VB_ERR_UNSUPPORTED, "repartition: the fused P2P exchange (VB_XCHG_NCCL is supported)");
    if (s->world < 2) return set_err(VB_ERR_STATE, "vb_shuffle_exchange of a one-process repartition (vb_shuffle_create_repartition_dist has world > 1)");
    if (!c->comm) return set_err(VB_ERR_STATE, "vb_shuffle_exchange needs vb_ctx_comm_init");
    if (c->comm->world != s->world || c->comm->rank != s->rank) return set_err(VB_ERR_INVALID, "shuffle rank/world differ from the communicator's");
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->sealing || s->exported || s->freed) return set_err(VB_ERR_STATE, "shuffle %llu: exchange after seal/exchange", (unsigned long long)s->id);
    }
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    return exchange_rep_locked(s);
}

static int rep_reduce_check(vb_shuf *s, u32 r, const char *what)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->rep) return set_err(VB_ERR_INVALID, "%s needs a shuffle from vb_shuffle_create_repartition", what);
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    return wait_sealed(s, true);
}

extern "C" int32_t vb_shuffle_reduce_repartition_size(vb_shuf *s, uint32_t r, uint64_t *n_rows, uint64_t *n_bytes)
{
    TRY(rep_reduce_check(s, r, "vb_shuffle_reduce_repartition_size"));
    const u64 b0 = s->bucket_off[r], nk = s->bucket_off[r + 1] - b0;
    if (n_rows) *n_rows = nk;
    if (!n_bytes) return VB_OK;
    *n_bytes = 0;
    if (!s->rep->bytes || nk == 0) return VB_OK;
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    DevBuf rr(c), offs(c);
    TRY(offs.alloc((nk + 1) * 8));
    return bytes_offsets(s, s->rep->refs + b0, nk, VB_DEVICE, rr, offs.as<u64>(), n_bytes);
}

extern "C" int32_t vb_shuffle_reduce_repartition(vb_shuf *s, uint32_t r, void *const *out_cols, uint64_t *out_offsets, void *out_bytes,
                                                 int32_t dst_loc)
{
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    TRY(rep_reduce_check(s, r, "vb_shuffle_reduce_repartition"));
    vb_ctx *c = s->ctx;
    RepState *rs = s->rep;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    const u64 b0 = s->bucket_off[r], nk = s->bucket_off[r + 1] - b0;
    DevBuf rr(c), offs(c), tmp(c);
    u64 total = 0;
    const bool want_bytes = rs->bytes && (out_offsets || out_bytes);
    if (want_bytes) {                           // the offsets first: a NULL out_bytes for a partition with bytes writes nothing
        TRY(offs.alloc((nk + 1) * 8));
        TRY(bytes_offsets(s, rs->refs ? rs->refs + b0 : nullptr, nk, VB_DEVICE, rr, offs.as<u64>(), &total));
        if (total && !out_bytes) return set_err(VB_ERR_INVALID, "NULL out_bytes for %llu bytes", (unsigned long long)total);
    }
    for (u32 k = 0; out_cols && k < rs->n_cols; ++k)
        if (nk) TRY(copy_out(s, out_cols[k], rs->cols + (u64)k * rs->n + b0, nk * 8, dst_loc));
    if (want_bytes) {
        unsigned char *dst = (unsigned char *)out_bytes;
        if (total && dst_loc == VB_HOST) { TRY(tmp.alloc(total)); dst = tmp.as<unsigned char>(); }
        if (total) TRY(bytes_gather_launch(s, rs->refs + b0, nk, offs.as<u64>(), total, dst));
        TRY(copy_out(s, out_offsets, offs.p, (nk + 1) * 8, dst_loc));
        if (dst_loc == VB_HOST) TRY(copy_out(s, out_bytes, dst, total, VB_HOST));
    }
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

template <int OPK, int TX>
static int launch_str_reduce(vb_shuf *s, const u32 *ids, const u64 *vals, u64 n, const u32 *dense, u64 *acc)
{
    vb_ctx *c = s->ctx;
    auto kern = str_reduce_kernel<OPK, TX>;
    const int occ = occupancy(c, kern, 256, 0);
    const u64 blocks = std::min<u64>((n + 255) / 256, (u64)c->sm_count * occ);
    KLaunch kl(s, K_HASH_AGG, n);
    kern<<<(unsigned)blocks, 256, 0, c->stream>>>(ids, vals, n, dense, acc);
    return kl.done("str_reduce_kernel");
}

static int str_reduce_rows(vb_shuf *s, int opk, int tx, const u32 *ids, const u64 *vals, u64 n, const u32 *dense, u64 *acc)
{
    switch (opk) {
    case OPK_ADD_U64: return launch_str_reduce<OPK_ADD_U64, TX_NONE>(s, ids, vals, n, dense, acc);
    case OPK_ADD_F64: return launch_str_reduce<OPK_ADD_F64, TX_NONE>(s, ids, vals, n, dense, acc);
    case OPK_COUNT: return launch_str_reduce<OPK_COUNT, TX_NONE>(s, ids, vals, n, dense, acc);
    case OPK_MIN_U64:
        if (tx == TX_I64) return launch_str_reduce<OPK_MIN_U64, TX_I64>(s, ids, vals, n, dense, acc);
        if (tx == TX_F64) return launch_str_reduce<OPK_MIN_U64, TX_F64>(s, ids, vals, n, dense, acc);
        return launch_str_reduce<OPK_MIN_U64, TX_NONE>(s, ids, vals, n, dense, acc);
    case OPK_MAX_U64:
        if (tx == TX_I64) return launch_str_reduce<OPK_MAX_U64, TX_I64>(s, ids, vals, n, dense, acc);
        if (tx == TX_F64) return launch_str_reduce<OPK_MAX_U64, TX_F64>(s, ids, vals, n, dense, acc);
        return launch_str_reduce<OPK_MAX_U64, TX_NONE>(s, ids, vals, n, dense, acc);
    }
    return set_err(VB_ERR_UNSUPPORTED, "string keys: op %d", s->agg);
}

// Rows as dictionary entry ids and their values: one map task's, or the rows a rank imported.  Reduce ops and
// combine_by_key: a map task's value columns in cols (in = IN_SOA), or partials [n_acc][n] in vals (IN_ACCS): the
// accumulators a rank imported, or a map task's bincode blob.
struct StrRun {
    const u32 *ids;
    const u64 *vals;
    u64 n;
    StrState::Cols cols{};
    int in = IN_SOA;
};

static std::vector<StrRun> str_map_runs(const vb_shuf *s)
{
    std::vector<StrRun> runs;
    for (u32 m = 0; m < s->n_map; ++m)
        if (s->maps[m].n_rows)
            runs.push_back(StrRun{s->str->ids[m], s->str->vals[m], s->maps[m].n_rows, s->str->cols[m], s->str->blob[m] ? IN_ACCS : IN_SOA});
    return runs;
}

static unsigned str_grid(const vb_ctx *c, u64 x) { return (unsigned)std::min<u64>((x + 255) / 256, (u64)c->sm_count * 8); }

// out[i] = a[at[i]] for host positions at[] (one gather, one D2H)
static int str_read_at(vb_shuf *s, const u64 *a, const std::vector<u64> &at, std::vector<u64> &out)
{
    vb_ctx *c = s->ctx;
    const u32 n = (u32)at.size();
    out.assign(n, 0);
    DevBuf idx(c), o(c);
    TRY(idx.alloc((size_t)n * 8));
    TRY(o.alloc((size_t)n * 8));
    CU(cudaMemcpyAsync(idx.p, at.data(), (size_t)n * 8, cudaMemcpyHostToDevice, c->stream));
    {
        KLaunch kl(s, K_MISC);
        gather_u64_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(a, idx.as<u64>(), n, o.as<u64>());
        TRY(kl.done("gather_u64_kernel"));
    }
    CU(cudaMemcpyAsync(out.data(), o.p, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

// Steps 1-2 of a string seal over `runs`: mark the entries the rows reference (a key only a replaced submission had is
// dropped), split them by h % n_reduce into dense ids laid out partition by partition in the order `order` (a
// permutation of [0, n_reduce)), and lay the keys' bytes out in that order.  cnt[r]: keys of partition r; base[r]: its
// first dense id, base[n_reduce] = D; dense [entries]: each entry's dense id; koff [D + 1]: byte offsets from 0.
static int str_dense_keys(vb_shuf *s, const std::vector<StrRun> &runs, const std::vector<u32> &order, std::vector<u64> &cnt,
                          std::vector<u64> &base, DevBuf &dense, DevBuf &koff, DevBuf &kbytes)
{
    vb_ctx *c = s->ctx;
    StrState *t = s->str;
    const u32 R = s->n_reduce, ne = t->n_e;
    DevBuf live(c), part(c), dcnt(c), cur(c), dbase(c), eod(c), klen(c);
    TRY(live.alloc((u64)ne * 4));
    CU(cudaMemsetAsync(live.p, 0, (u64)ne * 4, c->stream));
    for (const StrRun &r : runs) {
        KLaunch kl(s, K_MISC, r.n);
        str_mark_live_kernel<<<str_grid(c, r.n), 256, 0, c->stream>>>(r.ids, r.n, live.as<u32>());
        TRY(kl.done("str_mark_live_kernel"));
    }
    TRY(part.alloc((u64)ne * 4));
    TRY(dcnt.alloc((u64)R * 4));
    TRY(cur.alloc((u64)R * 4));
    CU(cudaMemsetAsync(dcnt.p, 0, (u64)R * 4, c->stream));
    CU(cudaMemsetAsync(cur.p, 0, (u64)R * 4, c->stream));
    {
        KLaunch kl(s, K_MISC, ne);
        str_part_count_kernel<<<(ne + 255) / 256, 256, 0, c->stream>>>(t->d.e_hash, live.as<u32>(), ne, make_fastmod(R), part.as<u32>(), dcnt.as<u32>());
        TRY(kl.done("str_part_count_kernel"));
    }
    std::vector<u32> hc(R);
    CU(cudaMemcpyAsync(hc.data(), dcnt.p, (size_t)R * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    cnt.assign(R, 0);
    base.assign((size_t)R + 1, 0);
    u64 D = 0;
    for (u32 r : order) {
        cnt[r] = hc[r];
        base[r] = D;
        D += hc[r];
    }
    base[R] = D;
    if (D >= (1ull << 31)) return set_err(VB_ERR_TOO_LARGE, "%llu distinct string keys (fewer than 2^31 are supported)", (unsigned long long)D);
    TRY(dbase.alloc(((u64)R + 1) * 8));
    CU(cudaMemcpyAsync(dbase.p, base.data(), ((size_t)R + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    TRY(dense.alloc((u64)ne * 4));
    TRY(eod.alloc(D * 4));
    TRY(klen.alloc(D * 8));
    TRY(koff.alloc((D + 1) * 8));
    {
        KLaunch kl(s, K_MISC, ne);
        str_dense_kernel<<<(ne + 255) / 256, 256, 0, c->stream>>>(live.as<u32>(), part.as<u32>(), ne, dbase.as<u64>(), cur.as<u32>(), t->d.e_len,
                                                                  dense.as<u32>(), eod.as<u32>(), klen.as<u64>());
        TRY(kl.done("str_dense_kernel"));
    }
    TRY(exclusive_scan_u64(s, klen.as<u64>(), koff.as<u64>(), D, koff.as<u64>() + D));
    u64 nb = 0;
    CU(cudaMemcpyAsync(c->h_scratch, koff.as<u64>() + D, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (D) nb = *(u64 *)c->h_scratch;
    TRY(kbytes.alloc(nb));
    {
        KLaunch kl(s, K_MISC, D);
        str_gather_bytes_kernel<<<(unsigned)((D * 32 + 255) / 256), 256, 0, c->stream>>>(eod.as<u32>(), (u32)D, t->d.e_off, koff.as<u64>(), t->d.arena,
                                                                                        kbytes.as<unsigned char>());
        TRY(kl.done("str_gather_bytes_kernel"));
    }
    return VB_OK;
}

// Reduce ops and combine_by_key: acc [n_acc][D] = every accumulator of the spec folded over the rows of `runs`, by
// dense id, in the spec's order transform, each run with the spec of its input kind (IN_SOA: the map rows and the map
// spec; IN_ACCS: partials and the import spec, whose merge ops have the map ops' identities).  A spec of one accumulator (every reduce op, and a combine of one aggregate) folds with
// str_reduce_kernel, whose 26-28 registers keep about twice the warps of str_reduce_multi_kernel resident (DESIGN
// §3.5, §5.2).
__global__ void range_kernel(u64 *__restrict__ out, u64 start, u64 step, u64 n);

static int str_fold_multi(vb_shuf *s, const std::vector<StrRun> &runs, const u32 *dense, u64 D, DevBuf &acc)
{
    vb_ctx *c = s->ctx;
    const AccSpec &ms = s->acc_map;
    TRY(acc.alloc(D * 8 * ms.n));
    for (u32 a = 0; a < ms.n; ++a) {
        KLaunch kl(s, K_MISC);
        str_fill_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(acc.as<u64>() + (u64)a * D, D, op_identity(spec_at(ms.op, a)));
        TRY(kl.done("str_fill_kernel"));
    }
    for (const StrRun &r : runs) {
        const int in = r.in;
        const AccSpec &sp = in == IN_ACCS ? s->acc_imp : s->acc_map;
        if (sp.n == 1) {               // a COUNT reads no column (its c[0] may be NULL)
            const u64 *vals = in == IN_ACCS ? r.vals : r.cols.c[spec_at(sp.src, 0)];
            TRY(str_reduce_rows(s, spec_at(sp.op, 0), spec_at(sp.tx, 0), r.ids, vals, r.n, dense, acc.as<u64>()));
            continue;
        }
        MaCols mc{};
        if (in == IN_ACCS) {
            mc.c[0] = r.vals;
            mc.stride = r.n;
        } else {
            std::copy(r.cols.c, r.cols.c + MA_MAX_COLS, mc.c);
        }
        auto kern = in == IN_ACCS ? str_reduce_multi_kernel<IN_ACCS> : str_reduce_multi_kernel<IN_SOA>;
        const int occ = occupancy(c, kern, 256, 0);
        const u64 blocks = std::min<u64>((r.n + 255) / 256, (u64)c->sm_count * occ);
        KLaunch kl(s, K_HASH_AGG, r.n);
        kern<<<(unsigned)blocks, 256, 0, c->stream>>>(r.ids, mc, r.n, dense, sp, D, acc.as<u64>());
        TRY(kl.done("str_reduce_multi_kernel"));
    }
    return VB_OK;
}

// The output columns [outs.n][D] of the folded accumulators: multi_finalize_kernel's rules (inverse order transform;
// MEAN = sum / count) over dense ids, read through an identity index.
static int str_finalize_multi(vb_shuf *s, const u64 *acc, u64 D, DevBuf &out)
{
    vb_ctx *c = s->ctx;
    DevBuf idx(c);
    TRY(idx.alloc(D * 8));
    TRY(out.alloc(D * 8 * s->outs.n));
    {
        KLaunch kl(s, K_MISC);
        range_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(idx.as<u64>(), 0, 1, D);
        TRY(kl.done("range_kernel"));
    }
    KLaunch kl(s, K_MISC);
    multi_finalize_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(acc, D, idx.as<u64>(), D, s->outs, out.as<u64>());
    return kl.done("multi_finalize_kernel");
}

// GROUP: the n rows of `runs`, concatenated in run order and stably sorted by dense id (seal_group's steps 4-7):
// offs [D + 1] (the CSR) and vals [n].
static int str_group_values(vb_shuf *s, const std::vector<StrRun> &runs, u64 n, const u32 *dense, u64 D, DevBuf &offs, DevBuf &vals)
{
    vb_ctx *c = s->ctx;
    DevBuf cids(c), cvals(c);
    TRY(cids.alloc(n * 4));
    TRY(cvals.alloc(n * 8));
    u64 at = 0;
    for (const StrRun &r : runs) {
        CU(cudaMemcpyAsync(cids.as<u32>() + at, r.ids, r.n * 4, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(cvals.as<u64>() + at, r.vals, r.n * 8, cudaMemcpyDeviceToDevice, c->stream));
        at += r.n;
    }
    TRY(offs.alloc((D + 1) * 8));
    CU(cudaMemsetAsync(offs.p, 0xFF, (D + 1) * 8, c->stream));
    u32 *sorted_ids = nullptr;
    u64 *sorted_vals = nullptr;
    bool csr_done = false;
    TRY(sort_id_pairs(s, cids.as<u32>(), Loader{LD_KEY32_VAL_SOA, nullptr, cvals.as<u64>(), 0}, n, ceil_log2_u64(std::max<u64>(D, 2)), &sorted_ids,
                      &sorted_vals, dense, offs.as<u64>(), &csr_done));
    DevBuf sid_guard(c);
    if (sorted_ids != cids.as<u32>()) sid_guard.p = sorted_ids;
    vals.reset();
    vals.p = sorted_vals;
    if (csr_done) {
        CU(cudaMemcpyAsync(offs.as<u64>() + D, &n, 8, cudaMemcpyHostToDevice, c->stream));
    } else {
        KLaunch kl(s, K_MISC);
        csr_bounds_kernel<<<str_grid(c, n), 256, 0, c->stream>>>(sorted_ids, n, offs.as<u64>(), D);
        TRY(kl.done("csr_bounds_kernel"));
    }
    return VB_OK;
}

// The reduce side of a string-key shuffle over `runs`:
//   1. mark the entries the rows reference;
//   2. split the live entries by h % n_reduce into partition-major dense ids, and lay their bytes out in that order;
//   3. reduce ops and combine_by_key: one RED per (warp, distinct id) into acc[accumulator][dense id] for every
//      accumulator of the spec (each run's `in`: map rows, or imported or blob partials), then the output columns;  GROUP: the rows in
//      run order (map-id order, or source-rank major), stably sorted by dense id, then the CSR (seal_group's steps
//      4-7).
// The per-map ids and the dictionary are freed at the end.
static int seal_str_runs(vb_shuf *s, const std::vector<StrRun> &runs)
{
    vb_ctx *c = s->ctx;
    StrState *t = s->str;
    const u32 R = s->n_reduce;
    s->bucket_off.assign((size_t)R + 1, 0);
    s->val_off.assign((size_t)R + 1, 0);
    t->kb_off.assign((size_t)R + 1, 0);
    u64 n = 0;
    for (const StrRun &r : runs) n += r.n;
    if (n && t->n_e) {
        std::vector<u32> order(R);
        for (u32 r = 0; r < R; ++r) order[r] = r;
        std::vector<u64> cnt;
        DevBuf dense(c), koff(c), kbytes(c);
        TRY(str_dense_keys(s, runs, order, cnt, s->bucket_off, dense, koff, kbytes));
        const u64 D = s->bucket_off[R];
        TRY(str_read_at(s, koff.as<u64>(), s->bucket_off, t->kb_off));
        if (is_reduce_op(s->agg)) {    // fold every accumulator, then the output columns
            DevBuf acc(c), out(c);
            TRY(str_fold_multi(s, runs, dense.as<u32>(), D, acc));
            TRY(str_finalize_multi(s, acc.as<u64>(), D, out));
            s->res_cols = (u64 *)out.release();
            s->st.rows_out = D;
        } else {
            DevBuf offs(c), vals(c);
            TRY(str_group_values(s, runs, n, dense.as<u32>(), D, offs, vals));
            TRY(sort_segments(s, offs.as<u64>(), D, vals.as<u64>(), n));
            TRY(str_read_at(s, offs.as<u64>(), s->bucket_off, s->val_off));
            s->n_vals = n;
            s->res_offs = (u64 *)offs.release();
            s->res_vals = (u64 *)vals.release();
            s->st.rows_out = n;
        }
        s->n_keys = D;
        t->key_off = (u64 *)koff.release();
        t->key_bytes = (unsigned char *)kbytes.release();
        CU(cudaStreamSynchronize(c->stream));
    }
    for (u32 m = 0; m < s->n_map; ++m) free_str_map(s, m);
    free_str_dict(s);
    return VB_OK;
}

static int seal_str_sort(vb_shuf *s, const std::vector<StrRun> &runs, const std::vector<u64> *part_rows = nullptr);

// Seal of a string-key shuffle (world == 1, every map present)
static int seal_str(vb_shuf *s) { return s->str->sort ? seal_str_sort(s, str_map_runs(s)) : seal_str_runs(s, str_map_runs(s)); }

// ---------------------------------------------------------------------------------------------
// sort_by_key over string keys (vb_shuffle_create_str_sort): the string map side (dictionary encode, per-map entry
// ids), the distinct keys ordered by their bytes on the device (strkeys.cuh, "sort_by_key over string keys"), and the
// rows stably sorted by key rank with the id sort of GROUP.  Partitions are sort_cuts_kernel's contiguous ranges.
// ---------------------------------------------------------------------------------------------

// OR ^ AND of keys[0 .. n): the radix digits on which not every key agrees
static int str_varying_bits(vb_shuf *s, const u64 *keys, u64 n, u64 *bits_dev, u64 *varying)
{
    vb_ctx *c = s->ctx;
    const unsigned long long init[2] = {0ull, ~0ull};
    CU(cudaMemcpyAsync(bits_dev, init, 16, cudaMemcpyHostToDevice, c->stream));
    {
        KLaunch kl(s, K_MISC);
        key_bits_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(keys, 1, n, TX_NONE, (unsigned long long *)bits_dev);
        TRY(kl.done("key_bits_kernel"));
    }
    u64 *h = (u64 *)c->h_scratch;
    CU(cudaMemcpyAsync(h, bits_dev, 16, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    *varying = h[0] ^ h[1];
    return VB_OK;
}

// Step 2 of the sort's seal: rank_of[e] for the D live entries live[0 .. D), in byte-wise lexicographic order of their
// keys.  Round w over the na active entries (all of them at first, each with start 0):
//   a. each entry's round-w sort key (str_sort_key: 7 key bytes and how the key goes on);
//   b. LSD radix passes over the digits of the key on which the active entries differ, then (w > 0) over those of their
//      starts: a stable sort by (start, key), entry ids as values;
//   c. run heads (same start and key) and group heads (same start); new start = start + (run head − group head);
//      a run of one is final, the others are compacted stably and go to round w + 1.
// Rounds: 1 + ceil(longest prefix two distinct keys share / 7); each touches only the keys still tied.
static int str_sort_order(vb_shuf *s, const u64 *live, u64 D, u32 *rank_of)
{
    vb_ctx *c = s->ctx;
    StrState *t = s->str;
    const u64 ne = t->n_e;
    DevBuf ka(c), kb(c), va(c), vb(c), key_of(c), start_of(c), head(c), hx(c), stay(c), spos(c), gpos(c), runpos(c), hist(c), aux(c);
    TRY(ka.alloc(D * 8)); TRY(kb.alloc(D * 8)); TRY(va.alloc(D * 8)); TRY(vb.alloc(D * 8));
    TRY(key_of.alloc(ne * 8)); TRY(start_of.alloc(ne * 4));
    TRY(head.alloc(D * 8)); TRY(hx.alloc(D * 8)); TRY(stay.alloc(D * 8)); TRY(spos.alloc(D * 8));
    TRY(gpos.alloc(D * 4)); TRY(runpos.alloc(D * 4));
    TRY(aux.alloc(32));                                   // [0, 2): key bits; [2]: runs; [3]: entries that stay
    CU(cudaMemsetAsync(start_of.p, 0, ne * 4, c->stream));
    u64 *bits = aux.as<u64>(), *n_runs = aux.as<u64>() + 2, *n_stay = aux.as<u64>() + 3;
    auto other_k = [&](const u64 *p) { return p == ka.as<u64>() ? kb.as<u64>() : ka.as<u64>(); };
    auto other_v = [&](const u64 *p) { return p == va.as<u64>() ? vb.as<u64>() : va.as<u64>(); };
    const u64 *act = live;
    u64 na = D;
    for (u32 w = 0; na; ++w) {
        if (7ull * w > t->n_a + 7) return set_err(VB_ERR_STATE, "string sort: round %u is past the longest key", w);
        {
            KLaunch kl(s, K_MISC, na);
            str_sort_word_kernel<<<str_grid(c, na), 256, 0, c->stream>>>(act, na, t->d.e_off, t->d.e_len, t->d.arena, w, ka.as<u64>(),
                                                                           key_of.as<u64>());
            TRY(kl.done("str_sort_word_kernel"));
        }
        const u64 *k = ka.as<u64>(), *v = act;
        const PassPlan plan = plan_pass<u64, true>(c, na);
        TRY(hist.alloc(plan.hist_bytes()));
        auto passes = [&](u64 varying) -> int {
            for (u32 p = 0; p < 8; ++p) {
                if (!((varying >> (8 * p)) & 0xFFull)) continue;
                u64 *dk = other_k(k), *dv = other_v(v);
                Digit dg{};
                dg.mode = DG_BITS; dg.shift = 8 * p; dg.mask = 0xFF; dg.tx = TX_NONE;
                TRY((radix_pass<u64, true>(s, Loader{LD_SOA64, k, v, 0}, dg, na, dk, dv, hist.as<u32>(), plan)));
                k = dk;
                v = dv;
            }
            return VB_OK;
        };
        u64 varying = 0;
        TRY(str_varying_bits(s, k, na, bits, &varying));
        TRY(passes(varying));
        if (w > 0) {                                      // round 0: every start is 0
            u64 *sk = other_k(k);
            {
                KLaunch kl(s, K_MISC, na);
                str_sort_start_kernel<<<str_grid(c, na), 256, 0, c->stream>>>(v, na, start_of.as<u32>(), sk);
                TRY(kl.done("str_sort_start_kernel"));
            }
            k = sk;
            TRY(str_varying_bits(s, k, na, bits, &varying));
            TRY(passes(varying));
        }
        {
            KLaunch kl(s, K_MISC, na);
            str_sort_heads_kernel<<<str_grid(c, na), 256, 0, c->stream>>>(v, na, key_of.as<u64>(), start_of.as<u32>(), head.as<u64>(),
                                                                            gpos.as<u32>());
            TRY(kl.done("str_sort_heads_kernel"));
        }
        TRY(exclusive_scan_u64(s, head.as<u64>(), hx.as<u64>(), na, n_runs));
        {
            KLaunch kl(s, K_MISC, na);
            str_sort_runpos_kernel<<<str_grid(c, na), 256, 0, c->stream>>>(head.as<u64>(), hx.as<u64>(), na, runpos.as<u32>());
            TRY(kl.done("str_sort_runpos_kernel"));
        }
        {
            KLaunch kl(s, K_MISC, na);
            str_sort_split_kernel<<<str_grid(c, na), 256, 0, c->stream>>>(v, head.as<u64>(), hx.as<u64>(), na, runpos.as<u32>(), n_runs,
                                                                            gpos.as<u32>(), start_of.as<u32>(), rank_of, stay.as<u64>());
            TRY(kl.done("str_sort_split_kernel"));
        }
        TRY(exclusive_scan_u64(s, stay.as<u64>(), spos.as<u64>(), na, n_stay));
        u64 next = 0;
        CU(cudaMemcpyAsync(&next, n_stay, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        if (next) {
            u64 *dst = other_v(v);
            KLaunch kl(s, K_MISC, na);
            str_compact_kernel<<<str_grid(c, na), 256, 0, c->stream>>>(stay.as<u64>(), spos.as<u64>(), v, na, dst);
            TRY(kl.done("str_compact_kernel"));
            act = dst;
        }
        na = next;
    }
    return VB_OK;
}

// The seal of a string sort over `runs` (map-id order):
//   1. mark the entries the rows reference, and compact the D live ones stably;
//   2. order them (str_sort_order): rank_of[entry];
//   3. the keys once, in rank order: offsets (scan of the lengths) and bytes (str_gather_bytes_kernel);
//   4. the rows' CSR by rank: with a payload, the rows in run order stably sorted by rank with their values (GROUP's
//      str_group_values over ranks); key-only, each rank's row count (the COUNT fold of str_reduce_kernel), scanned;
//   5. partition cuts (first CSR boundary at or after floor(p·n/R), or with part_rows, the owner's seal of a sort
//      across ranks: the boundaries after each partition's given row count) and per-partition key bytes (scan of
//      count · len).
// The per-map ids and the dictionary are freed at the end.
static int seal_str_sort(vb_shuf *s, const std::vector<StrRun> &runs, const std::vector<u64> *part_rows)
{
    vb_ctx *c = s->ctx;
    StrState *t = s->str;
    const u32 R = s->n_reduce;
    const u64 ne = t->n_e;
    s->bucket_off.assign((size_t)R + 1, 0);
    s->val_off.assign((size_t)R + 1, 0);
    t->kb_off.assign((size_t)R + 1, 0);
    t->rank_cut.assign((size_t)R + 1, 0);
    u64 n = 0;
    for (const StrRun &r : runs) n += r.n;
    if (n && ne) {
        DevBuf live(c), flag(c), pos(c), list(c), tot(c), rank_of(c);
        TRY(live.alloc(ne * 4));
        TRY(flag.alloc(ne * 8));
        TRY(pos.alloc(ne * 8));
        TRY(tot.alloc(8));
        CU(cudaMemsetAsync(live.p, 0, ne * 4, c->stream));
        for (const StrRun &r : runs) {
            KLaunch kl(s, K_MISC, r.n);
            str_mark_live_kernel<<<str_grid(c, r.n), 256, 0, c->stream>>>(r.ids, r.n, live.as<u32>());
            TRY(kl.done("str_mark_live_kernel"));
        }
        {
            KLaunch kl(s, K_MISC, ne);
            str_widen_u32_kernel<<<str_grid(c, ne), 256, 0, c->stream>>>(live.as<u32>(), ne, flag.as<u64>());
            TRY(kl.done("str_widen_u32_kernel"));
        }
        TRY(exclusive_scan_u64(s, flag.as<u64>(), pos.as<u64>(), ne, tot.as<u64>()));
        u64 D = 0;
        CU(cudaMemcpyAsync(&D, tot.p, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        if (D >= (1ull << 31)) return set_err(VB_ERR_TOO_LARGE, "%llu distinct string keys (fewer than 2^31 are supported)", (unsigned long long)D);
        TRY(list.alloc(D * 8));
        {
            KLaunch kl(s, K_MISC, ne);
            str_compact_kernel<<<str_grid(c, ne), 256, 0, c->stream>>>(flag.as<u64>(), pos.as<u64>(), nullptr, ne, list.as<u64>());
            TRY(kl.done("str_compact_kernel"));
        }
        flag.reset();
        pos.reset();
        TRY(rank_of.alloc(ne * 4));
        s->kclass_as = K_STR_ORDER;
        const int rc = str_sort_order(s, list.as<u64>(), D, rank_of.as<u32>());
        s->kclass_as = -1;
        TRY(rc);
        // 3. the keys in rank order
        DevBuf eor(c), klen(c), koff(c), kbytes(c);
        TRY(eor.alloc(D * 4));
        TRY(klen.alloc(D * 8));
        TRY(koff.alloc((D + 1) * 8));
        {
            KLaunch kl(s, K_MISC, D);
            str_sort_rank_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(list.as<u64>(), D, rank_of.as<u32>(), t->d.e_len, eor.as<u32>(),
                                                                         klen.as<u64>());
            TRY(kl.done("str_sort_rank_kernel"));
        }
        TRY(exclusive_scan_u64(s, klen.as<u64>(), koff.as<u64>(), D, koff.as<u64>() + D));
        u64 nb = 0;
        CU(cudaMemcpyAsync(&nb, koff.as<u64>() + D, 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        TRY(kbytes.alloc(nb));
        {
            KLaunch kl(s, K_MISC, D);
            str_gather_bytes_kernel<<<(unsigned)((D * 32 + 255) / 256), 256, 0, c->stream>>>(eor.as<u32>(), (u32)D, t->d.e_off, koff.as<u64>(),
                                                                                            t->d.arena, kbytes.as<unsigned char>());
            TRY(kl.done("str_gather_bytes_kernel"));
        }
        // 4. the rows' CSR by rank, and the payload in row order
        DevBuf roff(c), vals(c);
        if (t->sort_vals) {
            TRY(str_group_values(s, runs, n, rank_of.as<u32>(), D, roff, vals));
        } else {
            DevBuf cnt(c);
            TRY(cnt.alloc(D * 8));
            CU(cudaMemsetAsync(cnt.p, 0, D * 8, c->stream));
            for (const StrRun &r : runs) TRY(str_reduce_rows(s, OPK_COUNT, TX_NONE, r.ids, nullptr, r.n, rank_of.as<u32>(), cnt.as<u64>()));
            TRY(roff.alloc((D + 1) * 8));
            TRY(exclusive_scan_u64(s, cnt.as<u64>(), roff.as<u64>(), D, roff.as<u64>() + D));
        }
        // 5. cuts, and the key bytes of every partition
        DevBuf rb(c), boff(c), starts(c), rcut(c);
        TRY(rb.alloc(D * 8));
        TRY(boff.alloc((D + 1) * 8));
        TRY(starts.alloc(((u64)R + 1) * 8));
        TRY(rcut.alloc(((u64)R + 1) * 8));
        {
            KLaunch kl(s, K_MISC, D);
            str_sort_row_bytes_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(roff.as<u64>(), koff.as<u64>(), D, rb.as<u64>());
            TRY(kl.done("str_sort_row_bytes_kernel"));
        }
        TRY(exclusive_scan_u64(s, rb.as<u64>(), boff.as<u64>(), D, boff.as<u64>() + D));
        std::vector<u64> target;
        if (part_rows) {
            DevBuf tg(c);
            target.assign((size_t)R + 1, 0);
            for (u32 p = 0; p < R; ++p) target[p + 1] = target[p] + (*part_rows)[p];
            TRY(tg.alloc(((u64)R + 1) * 8));
            CU(cudaMemcpyAsync(tg.p, target.data(), ((size_t)R + 1) * 8, cudaMemcpyHostToDevice, c->stream));
            KLaunch kl(s, K_MISC);
            str_sort_cuts_at_kernel<<<(R + 1 + 255) / 256, 256, 0, c->stream>>>(roff.as<u64>(), D, tg.as<u64>(), R, starts.as<u64>(), rcut.as<u64>());
            TRY(kl.done("str_sort_cuts_at_kernel"));
        } else {
            KLaunch kl(s, K_MISC);
            str_sort_cuts_kernel<<<(R + 1 + 255) / 256, 256, 0, c->stream>>>(roff.as<u64>(), D, n, R, starts.as<u64>(), rcut.as<u64>());
            TRY(kl.done("str_sort_cuts_kernel"));
        }
        CU(cudaMemcpyAsync(s->bucket_off.data(), starts.p, ((size_t)R + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(t->rank_cut.data(), rcut.p, ((size_t)R + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        if (part_rows && s->bucket_off != target) return set_err(VB_ERR_STATE, "string sort: the received partitions do not end at key boundaries");
        TRY(str_read_at(s, boff.as<u64>(), t->rank_cut, t->kb_off));
        s->n_keys = D;
        s->st.rows_out = n;
        t->key_off = (u64 *)koff.release();
        t->key_bytes = (unsigned char *)kbytes.release();
        t->row_off = (u64 *)roff.release();
        t->row_boff = (u64 *)boff.release();
        if (t->sort_vals) s->res_vals = (u64 *)vals.release();
        CU(cudaStreamSynchronize(c->stream));
    }
    for (u32 m = 0; m < s->n_map; ++m) free_str_map(s, m);
    free_str_dict(s);
    return VB_OK;
}

static int copy_out_rebased(vb_shuf *s, u64 *dst, const u64 *src, u64 nk, u64 base, int dst_loc);

// vb_shuffle_reduce_str of a string sort: partition r's rows in key order, each with its key (offsets from
// str_sort_expand_kernel, bytes by str_gather_bytes_kernel over the row ranks), and the payload slice.
static int str_sort_out(vb_shuf *s, uint32_t r, uint64_t *out_key_offsets, void *out_key_bytes, void *out_vals, int32_t dst_loc)
{
    TRY(wait_sealed(s));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    StrState *t = s->str;
    const u64 row0 = s->bucket_off[r], nr = s->bucket_off[r + 1] - row0;
    const u64 byte0 = t->kb_off[r], nb = t->kb_off[r + 1] - byte0;
    if (nr == 0) {
        TRY(copy_out_rebased(s, out_key_offsets, nullptr, 0, 0, dst_loc));
        CU(cudaStreamSynchronize(c->stream));
        return VB_OK;
    }
    if (out_key_offsets || (out_key_bytes && nb)) {
        DevBuf off(c), rk(c), kb(c);
        TRY(off.alloc((nr + 1) * 8));
        TRY(rk.alloc(nr * 4));
        {
            KLaunch kl(s, K_MISC, nr);
            str_sort_expand_kernel<<<str_grid(c, nr), 256, 0, c->stream>>>(t->row_off, t->row_boff, t->key_off, t->rank_cut[r], t->rank_cut[r + 1],
                                                                             row0, nr, byte0, off.as<u64>(), rk.as<u32>());
            TRY(kl.done("str_sort_expand_kernel"));
        }
        TRY(copy_out(s, out_key_offsets, off.p, (nr + 1) * 8, dst_loc));
        if (out_key_bytes && nb) {
            unsigned char *dst = (unsigned char *)out_key_bytes;
            if (dst_loc == VB_HOST) {
                TRY(kb.alloc(nb));
                dst = kb.as<unsigned char>();
            }
            {
                KLaunch kl(s, K_MISC, nr);
                str_gather_bytes_kernel<<<(unsigned)((nr * 32 + 255) / 256), 256, 0, c->stream>>>(rk.as<u32>(), (u32)nr, t->key_off, off.as<u64>(),
                                                                                                 t->key_bytes, dst);
                TRY(kl.done("str_gather_bytes_kernel"));
            }
            if (dst_loc == VB_HOST) TRY(copy_out(s, out_key_bytes, kb.p, nb, dst_loc));
        }
    }
    TRY(copy_out(s, out_vals, s->res_vals ? s->res_vals + row0 : nullptr, nr * 8, dst_loc));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// string keys across ranks (vb_shuffle_create_str_dist): the map side of each rank is exported as key columns, packed
// by destination rank; the owner imports every rank's columns into a fresh dictionary and seals them as one run.
// ---------------------------------------------------------------------------------------------
// Export: steps 1-2 of the seal with the partitions laid out destination-major (rank 0's partitions, then rank 1's,
// ...), so the dense ids come out grouped by destination; then the values of step 3, as every accumulator of the
// spec per key in plain value form (reduce ops and combine_by_key) or each key's values in map order (GROUP).  The
// per-map ids and the dictionary are freed.  The caller holds c->mu.
static int export_str_locked(vb_shuf *s, u64 *n_keys, u64 *n_key_bytes, u64 *n_vals, u64 *n_val_bytes)
{
    vb_ctx *c = s->ctx;
    StrState *t = s->str;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->sealing || s->exported || s->freed) return set_err(VB_ERR_STATE, "export after seal/export");
    }
    const u32 W = s->world, R = s->n_reduce;
    for (u32 d = 0; d < W; ++d) n_keys[d] = n_key_bytes[d] = n_vals[d] = 0;
    if (n_val_bytes) std::fill(n_val_bytes, n_val_bytes + W, 0);
    const std::vector<StrRun> runs = str_map_runs(s);
    u64 n = 0;
    for (const StrRun &r : runs) n += r.n;
    if (n && t->n_e) {
        std::vector<u32> order;
        for (u32 d = 0; d < W; ++d)
            for (u32 r = d; r < R; r += W) order.push_back(r);
        std::vector<u64> cnt, base;
        DevBuf dense(c), koff(c), kbytes(c), lens(c);
        TRY(str_dense_keys(s, runs, order, cnt, base, dense, koff, kbytes));
        const u64 D = base[R];
        std::vector<u64> cut((size_t)W + 1, 0), at;                  // first dense id of each destination
        for (u32 d = 0; d < W; ++d) {
            u64 k = 0;
            for (u32 r = d; r < R; r += W) k += cnt[r];
            cut[d + 1] = cut[d] + k;
            n_keys[d] = k;
        }
        TRY(str_read_at(s, koff.as<u64>(), cut, at));
        for (u32 d = 0; d < W; ++d) n_key_bytes[d] = at[d + 1] - at[d];
        TRY(lens.alloc(D * 4));
        {
            KLaunch kl(s, K_MISC, D);
            str_diff_u32_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(koff.as<u64>(), D, lens.as<u32>());
            TRY(kl.done("str_diff_u32_kernel"));
        }
        if (is_reduce_op(s->agg)) {
            DevBuf acc(c);
            TRY(str_fold_multi(s, runs, dense.as<u32>(), D, acc));
            for (u32 a = 0; a < s->acc_map.n; ++a) {
                const int tx = spec_at(s->acc_map.tx, a);
                if (tx == TX_NONE) continue;
                KLaunch kl(s, K_MISC);
                tx_inv_kernel<<<(unsigned)((D + 255) / 256), 256, 0, c->stream>>>(acc.as<u64>() + (u64)a * D, D, tx);
                TRY(kl.done("tx_inv_kernel"));
            }
            for (u32 d = 0; d < W; ++d) n_vals[d] = n_keys[d];
            t->x_vals = (u64 *)acc.release();
        } else {
            DevBuf offs(c), vals(c), cnts(c);
            TRY(str_group_values(s, runs, n, dense.as<u32>(), D, offs, vals));
            TRY(cnts.alloc(D * 4));
            {
                KLaunch kl(s, K_MISC, D);
                str_diff_u32_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(offs.as<u64>(), D, cnts.as<u32>());
                TRY(kl.done("str_diff_u32_kernel"));
            }
            TRY(str_read_at(s, offs.as<u64>(), cut, at));
            for (u32 d = 0; d < W; ++d) n_vals[d] = at[d + 1] - at[d];
            if (s->bdist) {                     // byte-string values: their bytes travel in the values' order
                std::vector<u64> bat;
                TRY(bytes_pack(s, vals.as<u64>(), n, at, bat));
                for (u32 d = 0; d < W; ++d) n_val_bytes[d] = bat[d + 1] - bat[d];
            }
            t->x_cnts = (u32 *)cnts.release();
            t->x_vals = (u64 *)vals.release();
        }
        t->x_lens = (u32 *)lens.release();
        t->x_bytes = (unsigned char *)kbytes.release();
        CU(cudaStreamSynchronize(c->stream));
    }
    for (u32 m = 0; m < s->n_map; ++m) free_str_map(s, m);
    free_str_dict(s);
    std::lock_guard<std::mutex> g(s->mu);
    s->exported = true;
    return VB_OK;
}

// The limits of one import, from its totals: rows (accumulators, or GROUP values) and received keys
static int str_import_limits(const vb_shuf *s, u64 nk, u64 nv)
{
    const u64 rows = is_reduce_op(s->agg) ? nk : nv;
    if (rows >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "import of %llu rows (fewer than 2^32 - 2 are supported)", (unsigned long long)rows);
    if (nk >= (1ull << 31)) return set_err(VB_ERR_TOO_LARGE, "import of %llu keys (fewer than 2^31 are supported)", (unsigned long long)nk);
    return VB_OK;
}

// Seal of an imported string shuffle: the received keys' byte offsets (widened lengths, one scan), a fresh dictionary
// of them (str_encode_kernel; the received key count bounds the distinct keys), for GROUP each key's entry id over its
// run of values, then seal_str_runs over the rows as one source-rank-major run: reduce ops merge the accumulators with
// the import spec (COUNT as ADD), GROUP keeps source-rank order, which is map-id order.
static int seal_str_import(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    StrState *t = s->str;
    const u64 nk = t->i_nk, nkb = t->i_nkb, nv = t->i_nv;
    const bool group = !is_reduce_op(s->agg);
    std::vector<StrRun> runs;
    DevBuf wide(c), koff(c), voff(c), ids(c), row_ids(c);
    if (nk) {
        TRY(wide.alloc(nk * 8));
        TRY(koff.alloc((nk + 1) * 8));
        {
            KLaunch kl(s, K_MISC, nk);
            str_widen_u32_kernel<<<str_grid(c, nk), 256, 0, c->stream>>>(t->i_lens, nk, wide.as<u64>());
            TRY(kl.done("str_widen_u32_kernel"));
        }
        TRY(exclusive_scan_u64(s, wide.as<u64>(), koff.as<u64>(), nk, koff.as<u64>() + nk));
        u64 *h = (u64 *)c->h_scratch;
        CU(cudaMemcpyAsync(h, koff.as<u64>() + nk, 8, cudaMemcpyDeviceToHost, c->stream));
        if (group) {
            TRY(voff.alloc((nk + 1) * 8));
            {
                KLaunch kl(s, K_MISC, nk);
                str_widen_u32_kernel<<<str_grid(c, nk), 256, 0, c->stream>>>(t->i_cnts, nk, wide.as<u64>());
                TRY(kl.done("str_widen_u32_kernel"));
            }
            TRY(exclusive_scan_u64(s, wide.as<u64>(), voff.as<u64>(), nk, voff.as<u64>() + nk));
            CU(cudaMemcpyAsync(h + 1, voff.as<u64>() + nk, 8, cudaMemcpyDeviceToHost, c->stream));
        }
        CU(cudaStreamSynchronize(c->stream));
        if (h[0] != nkb) return set_err(VB_ERR_INVALID, "imported key lengths add up to %llu bytes, %llu announced", (unsigned long long)h[0], (unsigned long long)nkb);
        if (group && h[1] != nv) return set_err(VB_ERR_INVALID, "imported value counts add up to %llu, %llu announced", (unsigned long long)h[1], (unsigned long long)nv);
        t->n_e = 0;
        t->n_a = 0;
        TRY(ids.alloc(nk * 4));
        TRY(str_encode(s, koff.as<u64>(), t->i_bytes, 0, nk, nkb, nk, nk, ids.as<u32>()));
        if (group) {
            if (nv) {
                TRY(row_ids.alloc(nv * 4));
                KLaunch kl(s, K_MISC, nv);
                const int occ = occupancy(c, str_expand_ids_kernel, 256, 0);
                const u64 blocks = std::min<u64>((nv + 255) / 256, (u64)c->sm_count * occ);
                str_expand_ids_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(voff.as<u64>(), nk, ids.as<u32>(), nv, row_ids.as<u32>());
                TRY(kl.done("str_expand_ids_kernel"));
                runs.push_back(StrRun{row_ids.as<u32>(), t->i_vals, nv});
            }
        } else {
            runs.push_back(StrRun{ids.as<u32>(), t->i_vals, nk, {}, IN_ACCS});
        }
    }
    if (t->sort) {
        if (s->sort_part_rows.size() != s->n_reduce) return set_err(VB_ERR_STATE, "sort_by_key over string keys across ranks goes through vb_shuffle_exchange");
        TRY(seal_str_sort(s, runs, &s->sort_part_rows));
    } else {
        TRY(seal_str_runs(s, runs));
    }
    free_str_xchg(s);
    return VB_OK;
}

extern "C" int32_t vb_shuffle_create_str_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t vdt, int32_t agg,
                                              uint32_t rank, uint32_t world, vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_str_dist: NULL argument");
    *out = nullptr;
    if (vdt == VB_BYTES) return set_err(VB_ERR_UNSUPPORTED, "vb_shuffle_create_str_dist: byte-string values do not cross ranks yet");
    if (world < 1 || world > 256 || rank >= world) return set_err(VB_ERR_INVALID, "bad rank %u / world %u (1 <= world <= 256)", rank, world);
    TRY(vb_shuffle_create_str(c, shuffle_id, n_map, n_reduce, vdt, agg, out));
    (*out)->rank = rank;
    (*out)->world = world;
    return VB_OK;
}

// the checks every string export / import call makes first
static int str_dist_check(const vb_shuf *s, const char *what)
{
    if (!s->str || s->multi) return set_err(VB_ERR_INVALID, "%s needs a shuffle from vb_shuffle_create_str_dist", what);
    if (s->str->sort) return set_err(VB_ERR_UNSUPPORTED, "%s: sort_by_key over string keys across ranks goes through vb_shuffle_exchange (vb_ctx_comm_init)", what);
    if (s->world < 2) return set_err(VB_ERR_STATE, "%s needs a string shuffle of world > 1 (vb_shuffle_create_str_dist)", what);
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_str_prepare(vb_shuf *s, uint64_t *n_keys, uint64_t *n_key_bytes, uint64_t *n_vals)
{
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_export_str_prepare");
    if (!s || !n_keys || !n_key_bytes || !n_vals) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(str_dist_check(s, "vb_shuffle_export_str_prepare"));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    TRY(export_str_locked(s, n_keys, n_key_bytes, n_vals));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_str_buffers(vb_shuf *s, uint32_t **key_lens, void **key_bytes, uint32_t **val_counts, uint64_t **vals)
{
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_export_str_buffers");
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    TRY(str_dist_check(s, "vb_shuffle_export_str_buffers"));
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (!s->exported || s->sealed || s->freed) return set_err(VB_ERR_STATE, "vb_shuffle_export_str_buffers needs vb_shuffle_export_str_prepare first and no seal yet");
    }
    const StrState *t = s->str;
    if (key_lens) *key_lens = t->x_lens;
    if (key_bytes) *key_bytes = t->x_bytes;
    if (val_counts) *val_counts = t->x_cnts;
    if (vals) *vals = t->x_vals;
    return VB_OK;
}

// The columns a rank received, source-rank major, kept until seal (cnts: GROUP only); the shuffle is then imported.
static void str_take_import(vb_shuf *s, const u32 *lens, const void *bytes, const u32 *cnts, const u64 *vals, u64 nk, u64 nkb, u64 nv)
{
    StrState *t = s->str;
    t->i_lens = lens; t->i_bytes = (const unsigned char *)bytes; t->i_cnts = cnts; t->i_vals = vals;
    t->i_nk = nk; t->i_nkb = nkb; t->i_nv = nv;
    std::lock_guard<std::mutex> g(s->mu);
    s->imported = true;
}

// vb_shuffle_import_str and vb_shuffle_import_str_cols after their argument checks: the totals nk, nkb and nv (reduce
// ops: one accumulator row per key) are checked, and the caller's columns are borrowed until seal.
static int str_import(vb_shuf *s, const char *what, const char *prepare, const uint32_t *key_lens, const void *key_bytes,
                      const uint32_t *val_counts, const uint64_t *vals, u64 nk, u64 nkb, u64 nv)
{
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (!s->exported || s->imported || s->sealed || s->sealing || s->freed)
            return set_err(VB_ERR_STATE, "%s needs %s first, once, and no seal yet", what, prepare);
    }
    const bool group = !is_reduce_op(s->agg);
    if ((nk && !key_lens) || (nkb && !key_bytes) || (group && nk && !val_counts) || (nv && !vals))
        return set_err(VB_ERR_INVALID, "NULL column with a non-zero count");
    if (!group && nv != nk) return set_err(VB_ERR_INVALID, "reduce ops import one accumulator per key (%llu keys, %llu values)", (unsigned long long)nk, (unsigned long long)nv);
    TRY(str_import_limits(s, nk, nv));
    str_take_import(s, key_lens, key_bytes, group ? val_counts : nullptr, vals, nk, nkb, nv);
    return VB_OK;
}

extern "C" int32_t vb_shuffle_import_str(vb_shuf *s, const uint32_t *key_lens, const void *key_bytes, const uint32_t *val_counts,
                                         const uint64_t *vals, const uint64_t *n_keys, const uint64_t *n_key_bytes, const uint64_t *n_vals)
{
    if (s && s->vdt == VB_BYTES) return reject_bytes(s, "vb_shuffle_import_str");
    if (!s || !n_keys || !n_key_bytes || !n_vals) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(str_dist_check(s, "vb_shuffle_import_str"));
    u64 nk = 0, nkb = 0, nv = 0;
    for (u32 r = 0; r < s->world; ++r) { nk += n_keys[r]; nkb += n_key_bytes[r]; nv += n_vals[r]; }
    return str_import(s, "vb_shuffle_import_str", "vb_shuffle_export_str_prepare", key_lens, key_bytes, val_counts, vals, nk, nkb, nv);
}

// vb_shuffle_exchange of a GROUP string shuffle: export, then the exchange of four columns: u32 key lengths and u32
// value counts split by the key counts, key bytes by the byte counts, u64 values by the value counts.  The gathered
// row is the three count vectors (keys, key bytes, values to every destination).  The received columns are owned by
// the shuffle until seal.  A string sort takes its own path (exchange_str_sort_locked).
static int exchange_str_locked(vb_shuf *s)
{
    if (s->str->sort) return exchange_str_sort_locked(s);
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    StrState *t = s->str;
    const u32 W = m->world, me = m->rank;
    // byte-string values: a fourth count vector (value bytes), and u32 value lengths plus the bytes in place of the values
    const bool bx = s->bdist;
    const size_t len = (bx ? 4 : 3) * (size_t)W;   // n_keys[W], n_key_bytes[W], n_vals[W] (, n_val_bytes[W])
    std::vector<u64> row(len, 0);
    auto clk = std::chrono::steady_clock::now();
    TRY(export_str_locked(s, row.data(), row.data() + W, row.data() + 2 * (size_t)W, bx ? row.data() + 3 * (size_t)W : nullptr));
    s->xst.prepare_wall_ms += lap(clk);
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, row.data(), len, &mat));
    s->xst.counts_wall_ms += lap(clk);
    for (u32 d = 0; d < W; ++d) TRY(str_import_limits(s, xsplit(mat, len, W, d, 0).roff[W], xsplit(mat, len, W, d, 2).roff[W]));
    std::vector<XSplit> sp{xsplit(mat, len, W, me, 0), xsplit(mat, len, W, me, 1), xsplit(mat, len, W, me, 2)};
    if (bx) sp.push_back(xsplit(mat, len, W, me, 3));
    const u64 nk = sp[0].roff[W], nkb = sp[1].roff[W], nv = sp[2].roff[W], nvb = bx ? sp[3].roff[W] : 0;
    DevBuf lens(c), bytes(c), cnts(c), vals(c), vlens(c), vbytes(c);
    TRY(lens.alloc(nk * 4));
    TRY(bytes.alloc(nkb));
    TRY(cnts.alloc(nk * 4));
    if (bx) { TRY(vlens.alloc(nv * 4)); TRY(vbytes.alloc(nvb)); }
    else TRY(vals.alloc(nv * 8));
    std::vector<XCol> cols{{ncclUint32, t->x_lens, lens.p, 0}, {ncclUint8, t->x_bytes, bytes.p, 1}, {ncclUint32, t->x_cnts, cnts.p, 0}};
    if (bx) { cols.push_back({ncclUint32, s->bx_lens, vlens.p, 2}); cols.push_back({ncclUint8, s->bx_bytes, vbytes.p, 3}); }
    else cols.push_back({ncclUint64, t->x_vals, vals.p, 2});
    TRY(post_group(s, xfers(sp, cols, W)));
    if (bx) TRY(bytes_adopt(s, vlens.as<u32>(), nv, vbytes, nvb, vals));
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_NCCL, sp[2].soff[W] - sp[2].send[me], nv - sp[2].recv[me]);
    void **own = t->i_own;
    own[0] = lens.release(); own[1] = bytes.release(); own[2] = cnts.release(); own[3] = vals.release();
    str_take_import(s, (const u32 *)own[0], own[1], (const u32 *)own[2], (const u64 *)own[3], nk, nkb, nv);
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// sort_by_key over string keys across ranks (vb_shuffle_create_str_sort_dist + vb_shuffle_exchange).  The integer
// sort's shape (exchange_sort_locked) with byte-string cut keys:
//   1. one all-gather of (local rows, val_dtype, n_reduce): a rank that differs is refused on every rank;
//   2. the local sort (seal_str_sort over this rank's maps): distinct keys in rank order, the rows' CSR by key rank,
//      the payload in row order;
//   3. the exact cut keys s_p = the key of global row floor(p·N/R) - 1, agreed word by word for all cuts in lockstep
//      (str_cut_round_kernel): per word one round gathers every rank's smallest and largest word in the cut's
//      interval; if they differ, the ranks bisect [min, max] for the smallest word v whose global row count
//      Σ row_off[upper bound of v] reaches the target, one round per probe.  A word whose tail says the key ends is
//      final; otherwise the interval narrows to that word and the next one follows.  Only words and counts cross;
//   4. one all-gather of every rank's (keys, key bytes, rows) per partition; the receive limits are checked for every
//      rank from it, so all ranks refuse alike;
//   5. one grouped send/recv of the String GROUP wire columns cut by partition (u32 key lengths, key bytes, u32 row
//      counts per key, the u64 payload), received partition-major, then source-rank-major;
//   6. seal_str_import re-encodes them and seal_str_sort re-sorts them as one run (equal keys meet only within a
//      partition, in source-rank = map-id order), cut at the received partition totals.
// ---------------------------------------------------------------------------------------------
extern "C" int32_t vb_shuffle_create_str_sort_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t val_dtype,
                                                   uint32_t rank, uint32_t world, vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_str_sort_dist: NULL argument");
    *out = nullptr;
    if (val_dtype == VB_BYTES) return set_err(VB_ERR_UNSUPPORTED, "vb_shuffle_create_str_sort_dist: byte-string values do not cross ranks yet");
    if (world < 1 || world > 256 || rank >= world) return set_err(VB_ERR_INVALID, "bad rank %u / world %u (1 <= world <= 256)", rank, world);
    TRY(vb_shuffle_create_str_sort(c, shuffle_id, n_map, n_reduce, val_dtype, out));
    (*out)->rank = rank;
    (*out)->world = world;
    return VB_OK;
}

// Step 3: kcut[1 .. R) = each cut's local key rank (the local keys at or below s_p), over the D local keys koff /
// kbytes and their rows' CSR roff.  A cut's word is w; with w > 0 its interval still has to be narrowed to the word
// agreed at w - 1 (v), which the round's kernel does before it reads word w.  When the intervals of all ranks hold
// one key between them, that key is s_p: the cut is final without reading the rest of its words.
static int str_sort_agree_cuts(vb_shuf *s, const u64 *koff, const unsigned char *kbytes, const u64 *roff, u64 D, u64 N,
                               std::vector<u64> &kcut)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    const u32 W = m->world, R = s->n_reduce, P = R - 1;
    if (!P || !N) return VB_OK;
    enum { MINMAX, BISECT, FINAL, DONE };
    struct Cut { u64 need, lo, hi, v; u32 w; int st; };
    std::vector<Cut> cut(P);
    std::vector<u64> ab(2 * (size_t)P), cmd(2 * (size_t)P), all(3 * (size_t)P * W);
    for (u32 i = 0; i < P; ++i) {
        const u64 need = (u64)(((unsigned __int128)(i + 1) * N) / R);
        cut[i] = Cut{need, 0, 0, 0, 0, need ? MINMAX : DONE};
        ab[2 * i] = 0;
        ab[2 * i + 1] = D;
    }
    DevBuf d_cmd(c), d_ab(c), d_out(c), d_all(c);
    TRY(d_cmd.alloc((size_t)P * 16)); TRY(d_ab.alloc((size_t)P * 16)); TRY(d_out.alloc((size_t)P * 24)); TRY(d_all.alloc((size_t)P * 24 * W));
    CU(cudaMemcpyAsync(d_ab.p, ab.data(), (size_t)P * 16, cudaMemcpyHostToDevice, c->stream));
    // v agreed for cut i at its word: the key ends inside the word (tail < 8) or the search goes on with the next word
    auto resolve = [](Cut &k, u64 v) {
        k.v = v;
        if ((v & 0xFF) < 8) { k.st = FINAL; return; }
        k.st = MINMAX;
        ++k.w;
    };
    for (;;) {
        bool any = false, gather = false;
        for (u32 i = 0; i < P; ++i) {
            Cut &k = cut[i];
            u64 op = SCUT_IDLE, w = k.w, v = 0;
            if (k.st == MINMAX) {
                op = k.w ? SCUT_NARROW : SCUT_MINMAX;
                if (k.w) { w = k.w - 1; v = k.v; }
            } else if (k.st == BISECT) {
                op = SCUT_COUNT;
                v = k.lo + ((k.hi - k.lo) >> 1);
            } else if (k.st == FINAL) {
                op = SCUT_FINAL;
                v = k.v;
                k.st = DONE;
            }
            cmd[2 * i] = op | w << 8;
            cmd[2 * i + 1] = v;
            any |= op != SCUT_IDLE;
            gather |= op == SCUT_MINMAX || op == SCUT_NARROW || op == SCUT_COUNT;
        }
        if (!any) break;
        CU(cudaMemcpyAsync(d_cmd.p, cmd.data(), (size_t)P * 16, cudaMemcpyHostToDevice, c->stream));
        {
            KLaunch kl(s, K_MISC);
            str_cut_round_kernel<<<(P + 127) / 128, 128, 0, c->stream>>>(d_cmd.as<u64>(), P, koff, kbytes, roff, d_ab.as<u64>(), d_out.as<u64>());
            TRY(kl.done("str_cut_round_kernel"));
        }
        if (!gather) continue;
        NC(g_nccl.AllGather(d_out.p, d_all.p, 3 * (size_t)P, ncclUint64, m->comm, c->stream));
        CU(cudaMemcpyAsync(all.data(), d_all.p, (size_t)P * 24 * W, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        for (u32 i = 0; i < P; ++i) {
            Cut &k = cut[i];
            const u64 op = cmd[2 * i] & 0xFF;
            if (op == SCUT_MINMAX || op == SCUT_NARROW) {
                u64 lo = ~0ull, hi = 0, keys = 0;
                for (u32 r = 0; r < W; ++r) {
                    lo = std::min(lo, all[(size_t)r * 3 * P + 3 * i]);
                    hi = std::max(hi, all[(size_t)r * 3 * P + 3 * i + 1]);
                    keys += all[(size_t)r * 3 * P + 3 * i + 2];
                }
                if (!keys) return set_err(VB_ERR_STATE, "string sort: cut %u has no key left on any rank", i + 1);
                if (keys == 1) {                  // FINAL at the key's own word: every rank's cut is its b
                    k.v = hi;
                    k.st = FINAL;
                } else if (lo == hi) {
                    resolve(k, lo);
                } else {
                    k.lo = lo;
                    k.hi = hi;
                    k.st = BISECT;
                }
            } else if (op == SCUT_COUNT) {
                u64 tot = 0;
                for (u32 r = 0; r < W; ++r) tot += all[(size_t)r * 3 * P + 3 * i];
                const u64 mid = cmd[2 * i + 1];
                if (tot >= k.need) k.hi = mid; else k.lo = mid + 1;
                if (k.lo == k.hi) resolve(k, k.lo);
            }
        }
    }
    CU(cudaMemcpyAsync(ab.data(), d_ab.p, (size_t)P * 16, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (u32 i = 0; i < P; ++i) kcut[i + 1] = cut[i].need ? ab[2 * i] : 0;
    return VB_OK;
}

static int exchange_str_sort_locked(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    StrState *t = s->str;
    const u32 W = m->world, me = m->rank, R = s->n_reduce;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->sealed || s->sealing || s->exported || s->freed) return set_err(VB_ERR_STATE, "export after seal/export");
    }
    auto clk = std::chrono::steady_clock::now();
    // 1. rows and fingerprint, before any work: every rank refuses alike
    const std::vector<StrRun> runs = str_map_runs(s);
    u64 n_local = 0;
    for (const StrRun &r : runs) n_local += r.n;
    const u64 row[3] = {n_local, t->sort_vals ? (u64)s->vdt : ~0ull, R};
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, row, 3, &mat));
    u64 N = 0;
    for (u32 r = 0; r < W; ++r) {
        N += mat[3 * r];
        if (mat[3 * r + 1] != mat[1] || mat[3 * r + 2] != mat[2])
            return set_err(VB_ERR_INVALID, "rank %u's string sort differs from rank 0's (val_dtype or n_reduce)", r);
    }
    if (R > 4096) return set_err(VB_ERR_UNSUPPORTED, "sort_by_key across ranks supports up to 4096 output partitions");
    s->xst.counts_wall_ms += lap(clk);
    // 2. local sort; its one-process partition cuts are not used.  It consumes the map side (ids and dictionary), so
    // from here the shuffle counts as exported: after any later error a second exchange or a seal is VB_ERR_STATE
    {
        std::lock_guard<std::mutex> g(s->mu);
        s->exported = true;
    }
    TRY(seal_str_sort(s, runs));
    const u64 D = s->n_keys;
    DevBuf koff(c), kbytes(c), roff(c), pay(c);
    koff.p = t->key_off; kbytes.p = t->key_bytes; roff.p = t->row_off; pay.p = s->res_vals;
    dev_free(c, t->row_boff);
    t->key_off = nullptr; t->key_bytes = nullptr; t->row_off = nullptr; t->row_boff = nullptr;
    s->res_vals = nullptr;
    s->n_keys = 0;
    s->st.rows_out = 0;
    if (!D) {                                     // no local keys: one zero offset for the searches and reads
        TRY(koff.alloc(8)); TRY(roff.alloc(8));
        CU(cudaMemsetAsync(koff.p, 0, 8, c->stream));
        CU(cudaMemsetAsync(roff.p, 0, 8, c->stream));
    }
    s->xst.prepare_wall_ms += lap(clk);
    // 3. the cut keys
    std::vector<u64> kcut((size_t)R + 1, 0);
    kcut[R] = D;
    TRY(str_sort_agree_cuts(s, koff.as<u64>(), kbytes.as<unsigned char>(), roff.as<u64>(), D, N, kcut));
    for (u32 p = 1; p <= R; ++p) kcut[p] = std::max(kcut[p], kcut[p - 1]);
    // 4. the segment table: keys, key bytes and rows of every partition, from every rank (byte-string values: then
    // each partition's value bytes, from the pack of the payload in row order)
    const bool bx = s->bdist;
    const u32 ncol = bx ? 4 : 3;
    std::vector<u64> kb_at, r_at, b_at, seg(ncol * (size_t)R), segall(ncol * (size_t)R * W);
    TRY(str_read_at(s, koff.as<u64>(), kcut, kb_at));
    TRY(str_read_at(s, roff.as<u64>(), kcut, r_at));
    if (bx) TRY(bytes_pack(s, pay.as<u64>(), n_local, r_at, b_at));
    for (u32 p = 0; p < R; ++p) {
        seg[p] = kcut[p + 1] - kcut[p];
        seg[R + p] = kb_at[p + 1] - kb_at[p];
        seg[2 * (size_t)R + p] = r_at[p + 1] - r_at[p];
        if (bx) seg[3 * (size_t)R + p] = b_at[p + 1] - b_at[p];
    }
    {
        DevBuf d_seg(c), d_segall(c);
        TRY(d_seg.alloc(seg.size() * 8)); TRY(d_segall.alloc(segall.size() * 8));
        CU(cudaMemcpyAsync(d_seg.p, seg.data(), seg.size() * 8, cudaMemcpyHostToDevice, c->stream));
        NC(g_nccl.AllGather(d_seg.p, d_segall.p, seg.size(), ncclUint64, m->comm, c->stream));
        CU(cudaMemcpyAsync(segall.data(), d_segall.p, segall.size() * 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    auto at = [&](u32 r, u32 col, u32 p) { return segall[(size_t)r * ncol * R + (size_t)col * R + p]; };
    for (u32 d = 0; d < W; ++d) {
        u64 nk = 0, nv = 0;
        for (u32 p = d; p < R; p += W)
            for (u32 r = 0; r < W; ++r) { nk += at(r, 0, p); nv += at(r, 2, p); }
        TRY(str_import_limits(s, nk, nv));
    }
    s->xst.counts_wall_ms += lap(clk);
    // 5. one grouped send/recv of the wire columns, cut by partition
    DevBuf lens(c), cnts(c);
    TRY(lens.alloc(D * 4));
    TRY(cnts.alloc(D * 4));
    for (int col = 0; D && col < 2; ++col) {
        KLaunch kl(s, K_MISC, D);
        str_diff_u32_kernel<<<str_grid(c, D), 256, 0, c->stream>>>(col ? roff.as<u64>() : koff.as<u64>(), D, col ? cnts.as<u32>() : lens.as<u32>());
        TRY(kl.done("str_diff_u32_kernel"));
    }
    s->sort_part_rows.assign(R, 0);
    u64 nk = 0, nkb = 0, nv = 0, nvb = 0;
    for (u32 p = me; p < R; p += W)
        for (u32 r = 0; r < W; ++r) {
            nk += at(r, 0, p); nkb += at(r, 1, p); nv += at(r, 2, p); s->sort_part_rows[p] += at(r, 2, p);
            if (bx) nvb += at(r, 3, p);
        }
    const bool vals = t->sort_vals;
    DevBuf rl(c), rb(c), rn(c), rv(c), rvl(c), rvb(c);
    TRY(rl.alloc(nk * 4)); TRY(rb.alloc(nkb)); TRY(rn.alloc(nk * 4));
    if (bx) { TRY(rvl.alloc(nv * 4)); TRY(rvb.alloc(nvb)); }
    else if (vals) TRY(rv.alloc(nv * 8));
    std::vector<Xfer> xs;
    u64 sent = 0, own = 0;
    for (u32 p = 0; p < R; ++p) {
        const u32 d = p % W;
        xs.push_back(Xfer{true, d, lens.as<u32>() + kcut[p], seg[p], ncclUint32});
        xs.push_back(Xfer{true, d, kbytes.as<unsigned char>() + kb_at[p], seg[R + p], ncclUint8});
        xs.push_back(Xfer{true, d, cnts.as<u32>() + kcut[p], seg[p], ncclUint32});
        if (bx) {
            xs.push_back(Xfer{true, d, s->bx_lens + r_at[p], seg[2 * (size_t)R + p], ncclUint32});
            xs.push_back(Xfer{true, d, s->bx_bytes + b_at[p], seg[3 * (size_t)R + p], ncclUint8});
        } else if (vals) xs.push_back(Xfer{true, d, pay.as<u64>() + r_at[p], seg[2 * (size_t)R + p], ncclUint64});
        (d == me ? own : sent) += seg[2 * (size_t)R + p];
    }
    u64 ok = 0, ob = 0, ov = 0, obv = 0;
    for (u32 p = me; p < R; p += W)
        for (u32 r = 0; r < W; ++r) {
            const u64 k = at(r, 0, p), b = at(r, 1, p), v = at(r, 2, p);
            xs.push_back(Xfer{false, r, rl.as<u32>() + ok, k, ncclUint32});
            xs.push_back(Xfer{false, r, rb.as<unsigned char>() + ob, b, ncclUint8});
            xs.push_back(Xfer{false, r, rn.as<u32>() + ok, k, ncclUint32});
            if (bx) {
                const u64 vb = at(r, 3, p);
                xs.push_back(Xfer{false, r, rvl.as<u32>() + ov, v, ncclUint32});
                xs.push_back(Xfer{false, r, rvb.as<unsigned char>() + obv, vb, ncclUint8});
                obv += vb;
            } else if (vals) xs.push_back(Xfer{false, r, rv.as<u64>() + ov, v, ncclUint64});
            ok += k; ob += b; ov += v;
        }
    TRY(post_group(s, xs));
    if (bx) TRY(bytes_adopt(s, rvl.as<u32>(), nv, rvb, nvb, rv));
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_NCCL, sent, nv - own);
    void **io = t->i_own;
    io[0] = rl.release(); io[1] = rb.release(); io[2] = rn.release(); io[3] = vals ? rv.release() : nullptr;
    str_take_import(s, (const u32 *)io[0], io[1], (const u32 *)io[2], (const u64 *)io[3], nk, nkb, nv);
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// byte-string values across ranks (vb_shuffle_create_*bytes_dist).  References never leave their rank: the export packs
// the values' bytes in the exported rows' order (the gather of bytevals.cuh over the exported references), the wire
// carries u32 value lengths and the bytes, and the receiver makes what it received one more store, bvals[n_map], with
// fresh references into it in receive order.  Seal, cogroup, joins and the gather then run as on one process.
// ---------------------------------------------------------------------------------------------
// The pack: the values of the n device references refs, in their order, into s->bx_lens (u32) and s->bx_bytes, and
// at[i] = the byte offset of row cut[i].  The map stores are freed after it, in stream order: a reference issued at map
// time decodes to an empty store from here on and is refused by the gather.  Caller holds c->mu.
static int bytes_pack(vb_shuf *s, const u64 *refs, u64 n, const std::vector<u64> &cut, std::vector<u64> &at)
{
    vb_ctx *c = s->ctx;
    DevBuf none(c), offs(c), lens(c), bytes(c);
    TRY(offs.alloc((n + 1) * 8));
    u64 total = 0;
    TRY(bytes_offsets(s, refs, n, VB_DEVICE, none, offs.as<u64>(), &total));
    TRY(lens.alloc(n * 4));
    TRY(bytes.alloc(total));
    if (total) TRY(bytes_gather_launch(s, refs, n, offs.as<u64>(), total, bytes.as<unsigned char>()));
    if (n) {
        KLaunch kl(s, K_MISC, n);
        str_diff_u32_kernel<<<str_grid(c, n), 256, 0, c->stream>>>(offs.as<u64>(), n, lens.as<u32>());
        TRY(kl.done("str_diff_u32_kernel"));
    }
    TRY(str_read_at(s, offs.as<u64>(), cut, at));
    for (u32 m = 0; m < s->n_map; ++m) {
        dev_free(c, s->bvals[m].offs);
        dev_free(c, s->bvals[m].bytes);
        s->bvals[m] = ByteSrc{nullptr, nullptr, 0};
    }
    dev_free(c, s->bvals_dev);
    s->bvals_dev = nullptr;
    s->bx_lens = (u32 *)lens.release();
    s->bx_bytes = (unsigned char *)bytes.release();
    return VB_OK;
}

// The receive side: n received value lengths (device) and the received bytes, which the shuffle takes over as its store
// n_map (offsets: the scan of the lengths); refs [n] = ((n_map + 1) << 32) | i in receive order.  Lengths that do not
// add up to n_bytes are VB_ERR_INVALID, and then nothing is kept.  Caller holds c->mu.
static int bytes_adopt(vb_shuf *s, const u32 *lens, u64 n, DevBuf &bytes, u64 n_bytes, DevBuf &refs)
{
    vb_ctx *c = s->ctx;
    DevBuf wide(c), offs(c), r(c);
    TRY(offs.alloc((n + 1) * 8));
    TRY(r.alloc(n * 8));
    if (n) {
        TRY(wide.alloc(n * 8));
        {
            KLaunch kl(s, K_MISC, n);
            str_widen_u32_kernel<<<str_grid(c, n), 256, 0, c->stream>>>(lens, n, wide.as<u64>());
            TRY(kl.done("str_widen_u32_kernel"));
        }
        TRY(exclusive_scan_u64(s, wide.as<u64>(), offs.as<u64>(), n, offs.as<u64>() + n));
        KLaunch kl(s, K_MISC, n);
        bytes_refs_kernel<<<str_grid(c, n), 256, 0, c->stream>>>(((u64)s->n_map + 1) << 32, n, r.as<u64>());
        TRY(kl.done("bytes_refs_kernel"));
    } else {
        CU(cudaMemsetAsync(offs.p, 0, 8, c->stream));
    }
    u64 total = 0;
    TRY(fetch_status_unlocked(c, offs.as<u64>() + n, &total, 8));
    if (total != n_bytes)
        return set_err(VB_ERR_INVALID, "received value lengths add up to %llu bytes, %llu announced", (unsigned long long)total, (unsigned long long)n_bytes);
    s->bvals.resize((size_t)s->n_map + 1, ByteSrc{nullptr, nullptr, 0});
    s->bvals[s->n_map] = ByteSrc{(const u64 *)offs.release(), (const unsigned char *)bytes.release(), n};
    dev_free(c, s->bvals_dev);            // the gather builds the device table again, with the new store
    s->bvals_dev = nullptr;
    refs.reset();
    refs.p = r.release();
    return VB_OK;
}

static int bytes_dist_args(vb_ctx *c, vb_shuf **out, uint32_t rank, uint32_t world, const char *what)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "%s: NULL argument", what);
    *out = nullptr;
    if (world < 1 || world > 256 || rank >= world) return set_err(VB_ERR_INVALID, "%s: bad rank %u / world %u (1 <= world <= 256)", what, rank, world);
    return VB_OK;
}

static int bytes_dist_set(vb_shuf *s, uint32_t rank, uint32_t world)
{
    s->rank = rank;
    s->world = world;
    s->bdist = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_create_bytes_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, int32_t kdt, int32_t agg,
                                                int32_t part, uint32_t rank, uint32_t world, vb_shuf **out)
{
    TRY(bytes_dist_args(c, out, rank, world, "vb_shuffle_create_bytes_dist"));
    TRY(vb_shuffle_create(c, shuffle_id, n_map, n_reduce, kdt, VB_BYTES, agg, part, out));
    return bytes_dist_set(*out, rank, world);
}

extern "C" int32_t vb_shuffle_create_str_bytes_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t rank,
                                                    uint32_t world, vb_shuf **out)
{
    TRY(bytes_dist_args(c, out, rank, world, "vb_shuffle_create_str_bytes_dist"));
    TRY(vb_shuffle_create_str(c, shuffle_id, n_map, n_reduce, VB_BYTES, VB_AGG_GROUP, out));
    return bytes_dist_set(*out, rank, world);
}

extern "C" int32_t vb_shuffle_create_str_sort_bytes_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t rank,
                                                         uint32_t world, vb_shuf **out)
{
    TRY(bytes_dist_args(c, out, rank, world, "vb_shuffle_create_str_sort_bytes_dist"));
    TRY(vb_shuffle_create_str_sort_bytes(c, shuffle_id, n_map, n_reduce, out));
    return bytes_dist_set(*out, rank, world);
}

// the checks every bytes export / import call makes first: the matching create (str: String keys), GROUP or COGROUP,
// world > 1
static int bytes_dist_check(const vb_shuf *s, bool str, const char *what)
{
    if (!s->bdist || (s->str != nullptr) != str)
        return set_err(VB_ERR_INVALID, "%s needs a shuffle from vb_shuffle_create_%sbytes_dist", what, str ? "str_" : "");
    if (s->agg == VB_AGG_SORT) return set_err(VB_ERR_UNSUPPORTED, "%s: sort_by_key across ranks goes through vb_shuffle_exchange", what);
    if (s->world < 2) return set_err(VB_ERR_STATE, "%s needs a shuffle of world > 1", what);
    return VB_OK;
}

// the state an import needs: exported, not imported yet, not sealed
static int bytes_import_state(vb_shuf *s, const char *what)
{
    std::lock_guard<std::mutex> g(s->mu);
    if (!s->exported || s->imported || s->sealed || s->sealing || s->freed)
        return set_err(VB_ERR_STATE, "%s needs the export first, once, and no seal yet", what);
    return VB_OK;
}

// The received bytes copied into a buffer of the library, then bytes_adopt.  Caller holds c->mu.
static int bytes_import_values(vb_shuf *s, const u32 *lens, u64 n, const void *val_bytes, u64 n_bytes, DevBuf &refs)
{
    vb_ctx *c = s->ctx;
    DevBuf b(c);
    TRY(b.alloc(n_bytes));
    if (n_bytes) CU(cudaMemcpyAsync(b.p, val_bytes, n_bytes, cudaMemcpyDeviceToDevice, c->stream));
    return bytes_adopt(s, lens, n, b, n_bytes, refs);
}

extern "C" int32_t vb_shuffle_export_bytes_prepare(vb_shuf *s, uint64_t *counts, uint64_t *n_val_bytes)
{
    if (!s || !counts || !n_val_bytes) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(bytes_dist_check(s, false, "vb_shuffle_export_bytes_prepare"));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    TRY(export_bytes_locked(s, counts, n_val_bytes));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_bytes_buffers(vb_shuf *s, void **keys, uint32_t **val_lens, void **val_bytes)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    TRY(bytes_dist_check(s, false, "vb_shuffle_export_bytes_buffers"));
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (!s->exported || s->sealed || s->freed) return set_err(VB_ERR_STATE, "vb_shuffle_export_bytes_buffers needs vb_shuffle_export_bytes_prepare first and no seal yet");
    }
    if (keys) *keys = s->exp_keys;
    if (val_lens) *val_lens = s->bx_lens;
    if (val_bytes) *val_bytes = s->bx_bytes;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_import_bytes(vb_shuf *s, const void *keys, const uint32_t *val_lens, const void *val_bytes,
                                           const uint64_t *counts, const uint64_t *n_val_bytes)
{
    if (!s || !counts || !n_val_bytes) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(bytes_dist_check(s, false, "vb_shuffle_import_bytes"));
    TRY(bytes_import_state(s, "vb_shuffle_import_bytes"));
    u64 n = 0, nb = 0;
    for (u32 r = 0; r < s->world; ++r) { n += counts[r]; nb += n_val_bytes[r]; }
    if (n >= 0xFFFFFFFEull) return set_err(VB_ERR_TOO_LARGE, "import of %llu rows (fewer than 2^32 - 2 are supported)", (unsigned long long)n);
    if ((n && (!keys || !val_lens)) || (nb && !val_bytes)) return set_err(VB_ERR_INVALID, "NULL column with a non-zero count");
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    DevBuf refs(c);
    TRY(bytes_import_values(s, val_lens, n, val_bytes, nb, refs));
    std::lock_guard<std::mutex> g(s->mu);
    s->imp_own_v = (u64 *)refs.release();
    s->imp_keys = (const u64 *)keys;
    s->imp_vals = s->imp_own_v;
    s->imp_n = n;
    s->imported = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_str_bytes_prepare(vb_shuf *s, uint64_t *n_keys, uint64_t *n_key_bytes, uint64_t *n_vals, uint64_t *n_val_bytes)
{
    if (!s || !n_keys || !n_key_bytes || !n_vals || !n_val_bytes) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(bytes_dist_check(s, true, "vb_shuffle_export_str_bytes_prepare"));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    TRY(export_str_locked(s, n_keys, n_key_bytes, n_vals, n_val_bytes));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_str_bytes_buffers(vb_shuf *s, uint32_t **key_lens, void **key_bytes, uint32_t **val_counts,
                                                       uint32_t **val_lens, void **val_bytes)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    TRY(bytes_dist_check(s, true, "vb_shuffle_export_str_bytes_buffers"));
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (!s->exported || s->sealed || s->freed) return set_err(VB_ERR_STATE, "vb_shuffle_export_str_bytes_buffers needs vb_shuffle_export_str_bytes_prepare first and no seal yet");
    }
    const StrState *t = s->str;
    if (key_lens) *key_lens = t->x_lens;
    if (key_bytes) *key_bytes = t->x_bytes;
    if (val_counts) *val_counts = t->x_cnts;
    if (val_lens) *val_lens = s->bx_lens;
    if (val_bytes) *val_bytes = s->bx_bytes;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_import_str_bytes(vb_shuf *s, const uint32_t *key_lens, const void *key_bytes, const uint32_t *val_counts,
                                               const uint32_t *val_lens, const void *val_bytes, const uint64_t *n_keys,
                                               const uint64_t *n_key_bytes, const uint64_t *n_vals, const uint64_t *n_val_bytes)
{
    if (!s || !n_keys || !n_key_bytes || !n_vals || !n_val_bytes) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(bytes_dist_check(s, true, "vb_shuffle_import_str_bytes"));
    TRY(bytes_import_state(s, "vb_shuffle_import_str_bytes"));
    u64 nk = 0, nkb = 0, nv = 0, nvb = 0;
    for (u32 r = 0; r < s->world; ++r) { nk += n_keys[r]; nkb += n_key_bytes[r]; nv += n_vals[r]; nvb += n_val_bytes[r]; }
    if ((nk && (!key_lens || !val_counts)) || (nkb && !key_bytes) || (nv && !val_lens) || (nvb && !val_bytes))
        return set_err(VB_ERR_INVALID, "NULL column with a non-zero count");
    TRY(str_import_limits(s, nk, nv));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    DevBuf refs(c);
    TRY(bytes_import_values(s, val_lens, nv, val_bytes, nvb, refs));
    StrState *t = s->str;
    t->i_own[3] = refs.release();
    str_take_import(s, key_lens, key_bytes, val_counts, (const u64 *)t->i_own[3], nk, nkb, nv);
    return VB_OK;
}

extern "C" int32_t vb_shuffle_reduce_str_size(vb_shuf *s, uint32_t r, uint64_t *n_keys, uint64_t *n_key_bytes, uint64_t *n_vals)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->str) return set_err(VB_ERR_INVALID, "vb_shuffle_reduce_str_size needs a shuffle from vb_shuffle_create_str");
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    TRY(wait_sealed(s));
    if (n_keys) *n_keys = s->bucket_off[r + 1] - s->bucket_off[r];
    if (n_key_bytes) *n_key_bytes = s->str->kb_off[r + 1] - s->str->kb_off[r];
    if (n_vals) *n_vals = is_group_op(s->agg) ? s->val_off[r + 1] - s->val_off[r] : s->multi ? s->bucket_off[r + 1] - s->bucket_off[r] : 0;
    return VB_OK;
}

// out[0 .. nk] = src[0 .. nk] - base (partition-relative CSR offsets starting at 0)
static int copy_out_rebased(vb_shuf *s, u64 *dst, const u64 *src, u64 nk, u64 base, int dst_loc)
{
    vb_ctx *c = s->ctx;
    if (!dst) return VB_OK;
    if (nk == 0) {
        static const u64 zero = 0;
        CU(cudaMemcpyAsync(dst, &zero, 8, dst_loc == VB_HOST ? cudaMemcpyHostToHost : cudaMemcpyHostToDevice, c->stream));
        return VB_OK;
    }
    DevBuf tmp(c);
    TRY(tmp.alloc((nk + 1) * 8));
    KLaunch kl(s, K_MISC);
    rebase_kernel<<<(unsigned)((nk + 1 + 255) / 256), 256, 0, c->stream>>>(src, nk + 1, base, tmp.as<u64>());
    TRY(kl.done("rebase_kernel"));
    return copy_out(s, dst, tmp.p, (nk + 1) * 8, dst_loc);
}

// vb_shuffle_reduce_str and vb_shuffle_reduce_str_cols after their argument checks: partition r's keys, then its GROUP
// value lists (out_offsets, out_vals) or its first n_cols result columns (out_cols[o]; a NULL entry is skipped).
static int str_reduce_out(vb_shuf *s, uint32_t r, uint64_t *out_key_offsets, void *out_key_bytes, void *const *out_cols, u32 n_cols,
                          uint64_t *out_offsets, void *out_vals, int32_t dst_loc)
{
    TRY(wait_sealed(s));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    StrState *t = s->str;
    const u64 b0 = s->bucket_off[r], nk = s->bucket_off[r + 1] - b0;
    const u64 kb0 = t->kb_off[r], nkb = t->kb_off[r + 1] - kb0;
    TRY(copy_out_rebased(s, out_key_offsets, t->key_off ? t->key_off + b0 : nullptr, nk, kb0, dst_loc));
    TRY(copy_out(s, out_key_bytes, t->key_bytes ? t->key_bytes + kb0 : nullptr, nkb, dst_loc));
    if (is_group_op(s->agg)) {
        const u64 v0 = s->val_off[r], nv = s->val_off[r + 1] - v0;
        TRY(copy_out_rebased(s, out_offsets, s->res_offs ? s->res_offs + b0 : nullptr, nk, v0, dst_loc));
        TRY(copy_out(s, out_vals, s->res_vals ? s->res_vals + v0 : nullptr, nv * 8, dst_loc));
    } else {
        for (u32 o = 0; out_cols && o < n_cols; ++o)
            TRY(copy_out(s, out_cols[o], s->res_cols ? s->res_cols + (u64)o * s->n_keys + b0 : nullptr, nk * 8, dst_loc));
    }
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_reduce_str(vb_shuf *s, uint32_t r, uint64_t *out_key_offsets, void *out_key_bytes, void *out_combined,
                                         uint64_t *out_offsets, void *out_vals, int32_t dst_loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->str) return set_err(VB_ERR_INVALID, "vb_shuffle_reduce_str needs a shuffle from vb_shuffle_create_str");
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    if (s->multi && (out_combined || out_offsets || out_vals))
        return set_err(VB_ERR_INVALID, "shuffle %llu has several aggregates per key: read them with vb_shuffle_reduce_str_cols", (unsigned long long)s->id);
    if (s->str->sort) {
        if (out_offsets || out_vals) return set_err(VB_ERR_INVALID, "shuffle %llu sorts rows: it has no value lists (out_offsets / out_vals)", (unsigned long long)s->id);
        if (out_combined && !s->str->sort_vals) return set_err(VB_ERR_INVALID, "key-only sort has no payload");
        return str_sort_out(s, r, out_key_offsets, out_key_bytes, out_combined, dst_loc);
    }
    void *const combined[1] = {out_combined};
    return str_reduce_out(s, r, out_key_offsets, out_key_bytes, combined, 1, out_offsets, out_vals, dst_loc);
}

// ---------------------------------------------------------------------------------------------
// combine_by_key over string keys (vb_shuffle_create_str_multi): the string map and seal steps (dictionary encode,
// dense ids by partition) with the accumulators of vb_shuffle_create_multi folded over dense ids
// (str_reduce_multi_kernel) and finalized by the integer combine's rules.  Across ranks the string wire columns carry
// the accumulators [n_acc][keys] in the plain value form of vb_shuffle_export_cols_buffers.
// ---------------------------------------------------------------------------------------------
extern "C" int32_t vb_shuffle_create_str_multi(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t n_val_cols,
                                               const int32_t *val_dtypes, uint32_t n_aggs, const vb_agg_col *aggs, vb_shuf **out)
{
    if (!c || !out || !val_dtypes || !aggs) return set_err(VB_ERR_INVALID, "vb_shuffle_create_str_multi: NULL argument");
    *out = nullptr;
    MultiSpec ms;
    TRY(multi_spec(n_val_cols, val_dtypes, n_aggs, aggs, &ms));
    TRY(vb_shuffle_create_str(c, shuffle_id, n_map, n_reduce, VB_U64, VB_AGG_SUM, out));
    set_spec(*out, ms);
    (*out)->multi = true;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_create_str_multi_dist(vb_ctx *c, uint64_t shuffle_id, uint32_t n_map, uint32_t n_reduce, uint32_t n_val_cols,
                                                    const int32_t *val_dtypes, uint32_t n_aggs, const vb_agg_col *aggs, uint32_t rank,
                                                    uint32_t world, vb_shuf **out)
{
    if (!c || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_str_multi_dist: NULL argument");
    *out = nullptr;
    if (world < 1 || world > 256 || rank >= world) return set_err(VB_ERR_INVALID, "bad rank %u / world %u (1 <= world <= 256)", rank, world);
    TRY(vb_shuffle_create_str_multi(c, shuffle_id, n_map, n_reduce, n_val_cols, val_dtypes, n_aggs, aggs, out));
    (*out)->rank = rank;
    (*out)->world = world;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_reduce_str_cols(vb_shuf *s, uint32_t r, uint64_t *out_key_offsets, void *out_key_bytes, void *const *out_aggs,
                                              int32_t dst_loc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    if (!s->str || !s->multi) return set_err(VB_ERR_INVALID, "vb_shuffle_reduce_str_cols needs a shuffle from vb_shuffle_create_str_multi");
    if (r >= s->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", r, s->n_reduce);
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    return str_reduce_out(s, r, out_key_offsets, out_key_bytes, out_aggs, s->outs.n, nullptr, nullptr, dst_loc);
}

// the checks every string _cols export / import call makes first
static int str_multi_dist_check(const vb_shuf *s, const char *what)
{
    if (s->str && s->str->sort && s->world > 1)
        return set_err(VB_ERR_UNSUPPORTED, "%s: sort_by_key over string keys across ranks goes through vb_shuffle_exchange (vb_ctx_comm_init)", what);
    if (!s->str || !s->multi) return set_err(VB_ERR_INVALID, "%s needs a shuffle from vb_shuffle_create_str_multi_dist", what);
    if (s->world < 2) return set_err(VB_ERR_STATE, "%s needs a string-key combine shuffle of world > 1 (vb_shuffle_create_str_multi_dist)", what);
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_str_cols_prepare(vb_shuf *s, uint64_t *n_keys, uint64_t *n_key_bytes)
{
    if (!s || !n_keys || !n_key_bytes) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(str_multi_dist_check(s, "vb_shuffle_export_str_cols_prepare"));
    vb_ctx *c = s->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    std::vector<u64> n_vals(s->world);
    TRY(export_str_locked(s, n_keys, n_key_bytes, n_vals.data()));
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

extern "C" int32_t vb_shuffle_export_str_cols_buffers(vb_shuf *s, uint32_t **key_lens, void **key_bytes, uint64_t **accs, uint32_t *n_acc)
{
    if (!s) return set_err(VB_ERR_INVALID, "NULL shuffle");
    TRY(str_multi_dist_check(s, "vb_shuffle_export_str_cols_buffers"));
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (!s->exported || s->sealed || s->freed)
            return set_err(VB_ERR_STATE, "vb_shuffle_export_str_cols_buffers needs vb_shuffle_export_str_cols_prepare first and no seal yet");
    }
    const StrState *t = s->str;
    if (key_lens) *key_lens = t->x_lens;
    if (key_bytes) *key_bytes = t->x_bytes;
    if (accs) *accs = t->x_vals;
    if (n_acc) *n_acc = s->acc_map.n;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_import_str_cols(vb_shuf *s, const uint32_t *key_lens, const void *key_bytes, const uint64_t *accs, uint32_t n_acc,
                                              const uint64_t *n_keys, const uint64_t *n_key_bytes)
{
    if (!s || !n_keys || !n_key_bytes) return set_err(VB_ERR_INVALID, "NULL argument");
    TRY(str_multi_dist_check(s, "vb_shuffle_import_str_cols"));
    if (n_acc != s->acc_map.n) return set_err(VB_ERR_INVALID, "%u accumulator columns imported, the shuffle has %u", n_acc, s->acc_map.n);
    u64 nk = 0, nkb = 0;
    for (u32 r = 0; r < s->world; ++r) { nk += n_keys[r]; nkb += n_key_bytes[r]; }
    return str_import(s, "vb_shuffle_import_str_cols", "vb_shuffle_export_str_cols_prepare", key_lens, key_bytes, nullptr, accs, nk, nkb, nk);
}

// vb_shuffle_exchange of a string-key reduce op or combine: export, then the exchange of 2 + n_acc columns: u32 key
// lengths and the n_acc u64 accumulator columns split by the key counts, key bytes by the byte counts.  The gathered
// row is the key and byte counts to every destination, then exchange_multi_locked's spec fingerprint (no key width:
// keys are strings; the key kind of vb_shuffle_set_str_key in its place), so a rank whose op, spec or key kind differs
// is refused on every rank before any send.
static int exchange_str_accs_locked(vb_shuf *s)
{
    vb_ctx *c = s->ctx;
    Comm *m = c->comm;
    StrState *t = s->str;
    const u32 W = m->world, me = m->rank, NA = s->acc_map.n;
    const size_t len = 2 * (size_t)W + 3;        // n_keys[W], n_key_bytes[W], the fingerprint
    std::vector<u64> row(len, 0), n_vals(W);
    auto clk = std::chrono::steady_clock::now();
    TRY(export_str_locked(s, row.data(), row.data() + W, n_vals.data()));
    s->xst.prepare_wall_ms += lap(clk);
    row[2 * W] = s->acc_map.op;
    row[2 * W + 1] = s->acc_map.tx;
    row[2 * W + 2] = (u64)NA | (u64)t->kind << 8 | (u64)s->n_reduce << 32;
    const u64 *mat = nullptr;
    TRY(comm_all_gather(c, row.data(), len, &mat));
    s->xst.counts_wall_ms += lap(clk);
    for (u32 p = 1; p < W; ++p)
        for (u32 i = 0; i < 3; ++i)
            if (mat[p * len + 2 * W + i] != mat[2 * W + i])
                return set_err(VB_ERR_INVALID, "rank %u's reduce op or combine spec differs from rank 0's (accumulators, ops, transforms, key kind or n_reduce)", p);
    for (u32 d = 0; d < W; ++d) {
        const u64 nd = xsplit(mat, len, W, d, 0).roff[W];
        TRY(str_import_limits(s, nd, nd));
    }
    const std::vector<XSplit> sp{xsplit(mat, len, W, me, 0), xsplit(mat, len, W, me, 1)};
    const u64 n_sent = sp[0].soff[W], nk = sp[0].roff[W], nkb = sp[1].roff[W];
    DevBuf lens(c), bytes(c), accs(c);
    TRY(lens.alloc(nk * 4));
    TRY(bytes.alloc(nkb));
    TRY(accs.alloc(nk * 8 * NA));
    std::vector<XCol> cols{{ncclUint32, t->x_lens, lens.p, 0}, {ncclUint8, t->x_bytes, bytes.p, 1}};
    for (u32 a = 0; a < NA; ++a) cols.push_back({ncclUint64, t->x_vals + (u64)a * n_sent, accs.as<u64>() + (u64)a * nk, 0});
    TRY(post_group(s, xfers(sp, cols, W)));
    s->xst.post_wall_ms += lap(clk);
    xchg_done(s, VB_XCHG_NCCL, n_sent - sp[0].send[me], nk - sp[0].recv[me]);
    void **own = t->i_own;
    own[0] = lens.release(); own[1] = bytes.release(); own[3] = accs.release();
    str_take_import(s, (const u32 *)own[0], own[1], nullptr, (const u64 *)own[3], nk, nkb, nk);
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// cogroup and join of string keys (CoGroupedRdd::compute over `String` keys, co_grouped_rdd.rs:75-135, 206-249)
// The N-way plan of the integer sides (cogroup_n_plan) runs on the match matrix of per-side key indices; for string
// sides only the lookup (cogroup_n_str_probe_kernel over each side's key index) and the output keys differ.  An output
// key's bytes come from the first side of its match row that has it.  Every join goes through the outer-join plan
// with its `required` mask (all bits: the inner join) and writes each key with rows once, with its row offsets.
// ---------------------------------------------------------------------------------------------

// The key index of a sealed string shuffle's result keys, built on first use with the context locked and kept until
// vb_shuffle_free.  Sized like the dictionary index (load <= 0.5, 12 bytes per slot).
static int str_key_index(vb_shuf *s)
{
    StrState *t = s->str;
    vb_ctx *c = s->ctx;
    if (t->ix_fp || !s->n_keys) return VB_OK;
    const u64 D = s->n_keys;
    const u32 log_cap = choose_log_cap(D, D, false, STR_MAX_LOG_CAP, c->l2_bytes, 12);
    const u64 cap = 1ull << log_cap;
    DevBuf fp(c), id(c), h(c);
    TRY(fp.alloc(cap * 8));
    TRY(id.alloc(cap * 4));
    TRY(h.alloc(D * 8));
    CU(cudaMemsetAsync(fp.p, 0, cap * 8, c->stream));
    {
        KLaunch kl(s, K_DICT, D);
        const u64 blocks = std::min<u64>((D + 255) / 256, (u64)c->sm_count * 8);
        if (t->kind == STRKEY_BYTES)
            str_key_index_kernel<STRKEY_BYTES><<<(unsigned)blocks, 256, 0, c->stream>>>(t->key_off, t->key_bytes, (u32)D, fp.as<u64>(), id.as<u32>(),
                                                                                        log_cap, str_fp_mask(), h.as<u64>());
        else
            str_key_index_kernel<STRKEY_STR><<<(unsigned)blocks, 256, 0, c->stream>>>(t->key_off, t->key_bytes, (u32)D, fp.as<u64>(), id.as<u32>(),
                                                                                      log_cap, str_fp_mask(), h.as<u64>());
        TRY(kl.done("str_key_index_kernel"));
    }
    CU(cudaStreamSynchronize(c->stream));
    t->ix_fp = (u64 *)fp.release();
    t->ix_id = (u32 *)id.release();
    t->res_hash = (u64 *)h.release();
    t->ix_log_cap = log_cap;
    return VB_OK;
}

// A string reduce or combine result as a cogroup / join side without a second shuffle (vb_shuffle_create_narrow's string
// form).  Partition r of the parent holds exactly the keys with vb_hash_str(key) % n_reduce == r, each once, so the view
// is a sealed string GROUP shuffle over the same placement: copies of the key offsets, the key bytes and one result
// column, and offsets 0..n (one value per key).  No dictionary is built here: the key index the joins probe comes from
// str_key_index at the first cogroup or join, as for every GROUP side, and its kernel already inserts distinct keys
// without comparing their bytes.
static int narrow_str_build(vb_shuf *v, const vb_shuf *p, const u64 *col)
{
    vb_ctx *c = v->ctx;
    const StrState *pt = p->str;
    StrState *t = v->str;
    const u64 n = p->n_keys, nb = pt->kb_off[p->n_reduce];
    if (n == 0) return VB_OK;                         // an empty side: no arrays (as seal_str_runs leaves it)
    DevBuf koff(c), kbytes(c), vals(c), offs(c);
    TRY(koff.alloc((n + 1) * 8)); TRY(kbytes.alloc(nb)); TRY(vals.alloc(n * 8)); TRY(offs.alloc((n + 1) * 8));
    CU(cudaMemcpyAsync(koff.p, pt->key_off, (n + 1) * 8, cudaMemcpyDeviceToDevice, c->stream));
    if (nb) CU(cudaMemcpyAsync(kbytes.p, pt->key_bytes, nb, cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaMemcpyAsync(vals.p, col, n * 8, cudaMemcpyDeviceToDevice, c->stream));
    {
        KLaunch kl(v, K_MISC, n + 1);
        range_kernel<<<str_grid(c, n + 1), 256, 0, c->stream>>>(offs.as<u64>(), 0, 1, n + 1);
        TRY(kl.done("range_kernel"));
    }
    t->key_off = (u64 *)koff.release();
    t->key_bytes = (unsigned char *)kbytes.release();
    v->res_vals = (u64 *)vals.release();
    v->res_offs = (u64 *)offs.release();
    return VB_OK;
}

extern "C" int32_t vb_shuffle_create_narrow_str(vb_shuf *p, uint32_t out_col, vb_shuf **out)
{
    if (!p || !out) return set_err(VB_ERR_INVALID, "vb_shuffle_create_narrow_str: NULL argument");
    *out = nullptr;
    if (!p->str) return set_err(VB_ERR_INVALID, "vb_shuffle_create_narrow_str: shuffle %llu has integer keys (use vb_shuffle_create_narrow)",
                                (unsigned long long)p->id);
    if (p->str->sort || !is_reduce_op(p->agg))
        return set_err(VB_ERR_INVALID, "vb_shuffle_create_narrow_str: shuffle %llu is not a string reduce-op or combine_by_key shuffle",
                       (unsigned long long)p->id);
    if (out_col >= p->outs.n) return set_err(VB_ERR_INVALID, "vb_shuffle_create_narrow_str: output column %u of %u", out_col, p->outs.n);
    TRY(wait_sealed(p));
    vb_ctx *c = p->ctx;
    vb_shuf *v = make_internal_like(p);
    v->agg = VB_AGG_GROUP;
    v->vdt = p->out_dt[out_col];
    v->rank = p->rank; v->world = p->world;
    v->bucket_off = p->bucket_off; v->val_off = p->bucket_off;
    v->n_keys = v->n_vals = v->st.rows_out = p->n_keys;
    StrState *vt = str_attach(v);
    vt->kb_off = p->str->kb_off;
    vt->kind = p->str->kind;
    int rc;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        rc = [&]() -> int {
            CU(cudaSetDevice(c->device));
            TRY(narrow_str_build(v, p, p->res_cols ? p->res_cols + (u64)out_col * p->n_keys : nullptr));
            CU(cudaStreamSynchronize(c->stream));
            return VB_OK;
        }();
    }
    if (rc != VB_OK) { vb_shuffle_free(v); return rc; }
    *out = v;
    return VB_OK;
}

// describe the indexed string sides for the kernels
static int str_n_sides(vb_shuf *const *sides, u32 n, u32 rid, StrNSides *a)
{
    *a = StrNSides{};
    a->n = n;
    a->fp_mask = str_fp_mask();
    for (u32 j = 0; j < n; ++j) {
        const vb_shuf *s = sides[j];
        const StrState *t = s->str;
        if (s->n_keys && !t->ix_fp) return set_err(VB_ERR_STATE, "string cogroup side without a key index");
        a->fp[j] = t->ix_fp; a->id[j] = t->ix_id; a->log_cap[j] = t->ix_log_cap;
        a->hash[j] = t->res_hash; a->key_off[j] = t->key_off; a->bytes[j] = t->key_bytes;
        a->kb[j] = (u32)s->bucket_off[rid];
    }
    return VB_OK;
}

// The keys a call over the plan writes (all of a cogroup's; a join's with rows, taken in order by the stable
// compaction with their first rows), their byte offsets and total bytes.  Done once per plan.
static int str_plan_keys(vb_shuf *const *sides, u32 n, u32 rid, i64 kind, CogroupNPlan *p)
{
    if (p->str_done) return VB_OK;
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    const bool join = kind != NP_COGROUP;
    StrNSides sa;
    TRY(str_n_sides(sides, n, rid, &sa));
    DevBuf sel(c), koff(c), roff(c), len(c), ov(c);
    u64 nk = p->n_keys, nkb = 0;
    if (join) {
        if (nk) {
            DevBuf flag(c), idx(c);
            TRY(flag.alloc(nk));
            TRY(idx.alloc(nk * 8));
            {
                KLaunch kl(s0, K_JOIN);
                str_join_keep_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, c->stream>>>(p->pos, nk, p->total, flag.as<unsigned char>(),
                                                                                          idx.as<u64>());
                TRY(kl.done("str_join_keep_kernel"));
            }
            u64 m = 0;
            TRY(compact_rows(s0, idx.as<u64>(), p->pos, nk, flag.as<unsigned char>(), sel, ov, &m));
            nk = m;
        }
        TRY(roff.alloc((nk + 1) * 8));
        if (nk) CU(cudaMemcpyAsync(roff.p, ov.p, nk * 8, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(roff.as<u64>() + nk, &p->total, 8, cudaMemcpyHostToDevice, c->stream));
    }
    TRY(koff.alloc((nk + 1) * 8));
    if (nk) {
        TRY(len.alloc(nk * 8));
        {
            KLaunch kl(s0, K_JOIN);
            str_n_key_len_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, c->stream>>>(sa, p->match, sel.as<u64>(), nk, len.as<u64>());
            TRY(kl.done("str_n_key_len_kernel"));
        }
        TRY(exclusive_scan_u64(s0, len.as<u64>(), koff.as<u64>(), nk, koff.as<u64>() + nk));
        CU(cudaMemcpyAsync(c->h_scratch, koff.as<u64>() + nk, 8, cudaMemcpyDeviceToHost, c->stream));
    } else {
        CU(cudaMemsetAsync(koff.p, 0, 8, c->stream));
    }
    CU(cudaStreamSynchronize(c->stream));
    if (nk) nkb = *(u64 *)c->h_scratch;
    p->str_sel = (u64 *)sel.release();
    p->str_koff = (u64 *)koff.release();
    p->str_roff = (u64 *)roff.release();
    p->str_nk = nk;
    p->str_nkb = nkb;
    p->str_done = true;
    return VB_OK;
}

// out_key_offsets [str_nk + 1] and out_key_bytes [str_nkb] of the plan's keys (NULL outputs skipped)
static int str_write_keys(vb_shuf *const *sides, u32 n, u32 rid, i64 kind, CogroupNPlan *p, u64 *out_key_offsets,
                          void *out_key_bytes, int dst_loc)
{
    TRY(str_plan_keys(sides, n, rid, kind, p));
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    TRY(copy_out(s0, out_key_offsets, p->str_koff, (p->str_nk + 1) * 8, dst_loc));
    if (!out_key_bytes || !p->str_nkb) return VB_OK;
    StrNSides sa;
    TRY(str_n_sides(sides, n, rid, &sa));
    DevBuf tmp(c);
    unsigned char *d = (unsigned char *)out_key_bytes;
    if (dst_loc == VB_HOST) { TRY(tmp.alloc(p->str_nkb)); d = tmp.as<unsigned char>(); }
    {
        KLaunch kl(s0, K_JOIN);
        str_n_key_bytes_kernel<<<(unsigned)((p->str_nk * 32 + 255) / 256), 256, 0, c->stream>>>(sa, p->match, p->str_sel, p->str_nk,
                                                                                               p->str_koff, d);
        TRY(kl.done("str_n_key_bytes_kernel"));
    }
    if (dst_loc == VB_HOST) TRY(copy_out(s0, out_key_bytes, d, p->str_nkb, VB_HOST));
    return VB_OK;
}

// vb_cogroup_n's argument rules over string GROUP shuffles; waits until every side is sealed
static int cogroup_n_str_check(vb_shuf *const *sides, u32 n, u32 rid)
{
    if (!sides) return set_err(VB_ERR_INVALID, "sides is NULL");
    if (n < 1 || n > VB_MAX_COGROUP_SIDES) return set_err(VB_ERR_INVALID, "n_sides %u is not in [1, %d]", n, VB_MAX_COGROUP_SIDES);
    for (u32 j = 0; j < n; ++j) {
        const vb_shuf *s = sides[j];
        if (!s) return set_err(VB_ERR_INVALID, "side %u is NULL", j);
        if (!s->str) return set_err(VB_ERR_INVALID, "side %u is not a string-key shuffle (use vb_cogroup_n / vb_join_n_outer)", j);
        if (s->agg != VB_AGG_GROUP) return set_err(VB_ERR_INVALID, "side %u is not a GROUP shuffle", j);
        if (s->n_reduce != sides[0]->n_reduce) return set_err(VB_ERR_INVALID, "side %u uses a different partitioner than side 0", j);
        if (s->str->kind != sides[0]->str->kind)     // equal bytes sit in different partitions under the two hashes
            return set_err(VB_ERR_INVALID, "side %u hashes its keys as %s, side 0 as %s", j, s->str->kind == STRKEY_BYTES ? "bytes" : "String",
                           sides[0]->str->kind == STRKEY_BYTES ? "bytes" : "String");
        if (s->ctx != sides[0]->ctx) return set_err(VB_ERR_INVALID, "side %u lives on a different context than side 0", j);
    }
    if (rid >= sides[0]->n_reduce) return set_err(VB_ERR_INVALID, "reduce_id %u >= n_reduce %u", rid, sides[0]->n_reduce);
    for (u32 j = 0; j < n; ++j) TRY(wait_sealed(sides[j]));
    return VB_OK;
}

static int join_n_str_check(vb_shuf *const *sides, u32 n, u32 rid, u32 required)
{
    TRY(cogroup_n_str_check(sides, n, rid));
    if (required >> n) return set_err(VB_ERR_INVALID, "required mask %#x names a side >= n_sides %u", required, n);
    return VB_OK;
}

// the plan of (sides, rid, kind) with its string keys, every side indexed; the context is locked
static int str_plan(vb_shuf *const *sides, u32 n, u32 rid, i64 kind, CogroupNPlan **p)
{
    for (u32 j = 0; j < n; ++j) TRY(str_key_index(sides[j]));
    CogroupNSides a;
    TRY(cogroup_n_sides(sides, n, rid, &a));
    TRY(cogroup_n_plan(sides, n, rid, kind, a, p));
    return str_plan_keys(sides, n, rid, kind, *p);
}

extern "C" int32_t vb_cogroup_n_str_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint64_t *n_keys,
                                         uint64_t *n_key_bytes, uint64_t *n_vals)
{
    TRY(cogroup_n_str_check(sides, n_sides, rid));
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    CogroupNPlan *p = nullptr;
    TRY(str_plan(sides, n_sides, rid, NP_COGROUP, &p));
    if (n_keys) *n_keys = p->str_nk;
    if (n_key_bytes) *n_key_bytes = p->str_nkb;
    for (u32 j = 0; n_vals && j < n_sides; ++j) n_vals[j] = sides[j]->val_off[rid + 1] - sides[j]->val_off[rid];
    return VB_OK;
}

extern "C" int32_t vb_cogroup_n_str(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint64_t *out_key_offsets,
                                    void *out_key_bytes, uint64_t *const *out_offsets, void *const *out_vals, int32_t dst_loc)
{
    TRY(cogroup_n_str_check(sides, n_sides, rid));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(str_key_index(sides[j]));
    return cogroup_n_write(sides, n_sides, rid, out_key_bytes, out_offsets, out_vals, dst_loc, out_key_offsets);
}

extern "C" int32_t vb_join_n_str_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required,
                                      uint64_t *n_rows, uint64_t *n_keys, uint64_t *n_key_bytes)
{
    TRY(join_n_str_check(sides, n_sides, rid, required));
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    CogroupNPlan *p = nullptr;
    TRY(str_plan(sides, n_sides, rid, required, &p));
    if (n_rows) *n_rows = p->total;
    if (n_keys) *n_keys = p->str_nk;
    if (n_key_bytes) *n_key_bytes = p->str_nkb;
    return VB_OK;
}

extern "C" int32_t vb_join_n_str(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required, uint64_t *out_key_offsets,
                                 void *out_key_bytes, uint64_t *out_row_offsets, void *const *out_vals, uint8_t *const *out_valid,
                                 int32_t dst_loc)
{
    TRY(join_n_str_check(sides, n_sides, rid, required));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(str_key_index(sides[j]));
    return join_n_outer_write(sides, n_sides, rid, required, out_key_bytes, out_vals, out_valid, dst_loc, out_key_offsets,
                              out_row_offsets);
}

// vb_semi_join_n over string sides: side 0's keys of the partition probed against each filter side's key index (by the
// full hash, then the bytes); the kept keys written once, from side 0, with their row offsets, and side 0's lists as rows
extern "C" int32_t vb_semi_join_n_str_size(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required,
                                           uint32_t excluded, uint64_t *n_rows, uint64_t *n_keys, uint64_t *n_key_bytes)
{
    TRY(cogroup_n_str_check(sides, n_sides, rid));
    TRY(semi_masks_check(n_sides, required, excluded));
    vb_ctx *c = sides[0]->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(str_key_index(sides[j]));
    CogroupNPlan *p = nullptr;
    vb_shuf *g = nullptr;
    TRY(semi_plan(sides, n_sides, rid, required, excluded, &p, &g));
    TRY(str_plan_keys(sides, 1, rid, semi_kind(required, excluded), p));
    if (n_rows) *n_rows = p->total;
    if (n_keys) *n_keys = p->str_nk;
    if (n_key_bytes) *n_key_bytes = p->str_nkb;
    return VB_OK;
}

extern "C" int32_t vb_semi_join_n_str(vb_shuf *const *sides, uint32_t n_sides, uint32_t rid, uint32_t required, uint32_t excluded,
                                      uint64_t *out_key_offsets, void *out_key_bytes, uint64_t *out_row_offsets, void *out_vals,
                                      int32_t dst_loc)
{
    TRY(cogroup_n_str_check(sides, n_sides, rid));
    TRY(semi_masks_check(n_sides, required, excluded));
    if (dst_loc != VB_HOST && dst_loc != VB_DEVICE) return set_err(VB_ERR_INVALID, "bad dst_loc");
    vb_shuf *s0 = sides[0];
    vb_ctx *c = s0->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    for (u32 j = 0; j < n_sides; ++j) TRY(str_key_index(sides[j]));
    const i64 kind = semi_kind(required, excluded);
    CogroupNPlan *p = nullptr;
    vb_shuf *g = nullptr;
    TRY(semi_plan(sides, n_sides, rid, required, excluded, &p, &g));
    int rc = [&]() -> int {
        TRY(str_plan_keys(sides, 1, rid, kind, p));      // one-side plan: every key's bytes come from side 0
        const u64 total = p->total;
        if (total && (!out_vals || !out_key_offsets || !out_row_offsets || (p->str_nkb && !out_key_bytes)))
            return set_err(VB_ERR_INVALID, "NULL output with %llu rows to write", (unsigned long long)total);
        if (total) {
            DevBuf tmp(c);
            u64 *d = (u64 *)out_vals;
            if (dst_loc == VB_HOST) { TRY(tmp.alloc(total * 8)); d = tmp.as<u64>(); }
            {
                KLaunch kl(s0, K_JOIN, total);
                const u64 blocks = std::min<u64>((total + 255) / 256, (u64)c->sm_count * 8);
                cogroup_n_gather_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(p->pos, (u32)p->n_keys, p->match, 1, 0, g->res_offs,
                                                                                g->res_vals, d);
                TRY(kl.done("cogroup_n_gather_kernel"));
            }
            if (dst_loc == VB_HOST) TRY(copy_out(s0, out_vals, d, total * 8, VB_HOST));
        }
        TRY(str_write_keys(sides, 1, rid, kind, p, out_key_offsets, out_key_bytes, dst_loc));
        return copy_out(s0, out_row_offsets, p->str_roff, (p->str_nk + 1) * 8, dst_loc);
    }();
    cudaStreamSynchronize(c->stream);
    drop_cogroup_n_plan(sides, n_sides, rid, kind);
    return rc;
}

extern "C" uint64_t vb_hash_str(const void *bytes, uint64_t len) { return metro64_1_str((const unsigned char *)bytes, len); }

extern "C" uint32_t vb_get_partition_str(const void *bytes, uint64_t len, uint32_t n_reduce)
{
    if (n_reduce == 0) return 0;
    return (uint32_t)(metro64_1_str((const unsigned char *)bytes, len) % (uint64_t)n_reduce);
}

extern "C" uint64_t vb_hash_bytes(const void *bytes, uint64_t len) { return metro64_1_bytes((const unsigned char *)bytes, len); }

extern "C" uint32_t vb_get_partition_bytes(const void *bytes, uint64_t len, uint32_t n_reduce)
{
    if (n_reduce == 0) return 0;
    return (uint32_t)(metro64_1_bytes((const unsigned char *)bytes, len) % (uint64_t)n_reduce);
}

// ---------------------------------------------------------------------------------------------
// free / stats
// ---------------------------------------------------------------------------------------------
extern "C" int32_t vb_shuffle_free(vb_shuf *s)
{
    if (!s) return VB_OK;
    vb_ctx *c = s->ctx;
    {
        std::unique_lock<std::mutex> g(s->mu);
        s->freed = true;
        s->cv.notify_all();
        s->cv.wait(g, [&] { return s->waiters == 0 && !s->sealing; });   // blocked reduce/join/seal callers leave first
    }
    {
        std::lock_guard<std::mutex> lk(c->mu);
        cudaSetDevice(c->device);
        resolve_timers(s);
        for (auto &m : s->maps) free_map(s, m);
        release_inputs(s);
        dev_free(c, s->res_keys); dev_free(c, s->res_comb); dev_free(c, s->res_offs); dev_free(c, s->res_vals); dev_free(c, s->res_cols);
        dev_free(c, s->dict); dev_free(c, s->dense_of_slot);
        for (auto &kv : s->join_plans) { dev_free(c, kv.second.pos); dev_free(c, kv.second.match); }
        for (auto &kv : s->n_plans) free_cogroup_n_plan(c, kv.second);
        for (auto &kv : s->semi) { dev_free(c, kv.second.tab); dev_free(c, kv.second.mask); }
        free_lazy_rows(s);
        free_str(s);
        free_rep(s);
        for (ByteSrc &b : s->bvals) { dev_free(c, b.offs); dev_free(c, b.bytes); }
        dev_free(c, s->bvals_dev);
        cudaStreamSynchronize(c->stream);
    }
    for (auto &kv : s->filtered) { vb_shuffle_free(kv.second.first); vb_shuffle_free(kv.second.second); }
    for (vb_shuf *t : s->trash) vb_shuffle_free(t);
    for (auto &kv : s->semi) vb_shuffle_free(kv.second.kept);
    delete s;
    return VB_OK;
}

extern "C" int32_t vb_shuffle_stats(vb_shuf *s, vb_stats *out)
{
    if (!s || !out) return set_err(VB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    cudaSetDevice(s->ctx->device);
    resolve_timers(s);
    *out = s->st;
    return VB_OK;
}

// per-kernel-class device time (profiling on): klass 0 hash_agg, 1 dict, 2 merge, 3 rp_hist,
// 4 rp_scan, 5 rp_scatter, 6 misc, 7 join, 8 str_order
extern "C" int32_t vb_shuffle_kernel_time(vb_shuf *s, int32_t klass, double *ms, uint64_t *launches)
{
    if (!s || klass < 0 || klass >= K_N) return set_err(VB_ERR_INVALID, "bad argument");
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    cudaSetDevice(s->ctx->device);
    resolve_timers(s);
    if (ms) *ms = s->kms[klass];
    if (launches) *launches = s->klaunch[klass];
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// host-side pieces of the path
// ---------------------------------------------------------------------------------------------
extern "C" uint64_t vb_hash_key(uint64_t key, uint32_t key_width) { return hash_key(key, key_width); }

extern "C" uint32_t vb_get_partition(uint64_t key, uint32_t key_width, uint32_t n_reduce)
{
    if (n_reduce == 0) return 0;
    return (uint32_t)(hash_key(key, key_width) % (uint64_t)n_reduce);
}

// ParallelCollection::slice (src/rdd/parallel_collection_rdd.rs:116-145).  The reference walks the
// elements and cuts at most once per element; in closed form that is
//   n >= num_slices : exactly num_slices slices, slice s = [floor(s*n/num_slices), floor((s+1)*n/num_slices))
//   n <  num_slices : every element triggers a cut (the running `end` never gets ahead of the element
//                     index), giving an empty leading slice followed by n singletons (n+1 slices)
// (tests/test_abi_cpu.py checks this against the literal loop of the oracle).
extern "C" uint64_t vb_slice(uint64_t n, uint64_t num_slices, uint64_t *starts)
{
    if (num_slices < 1 || !starts) return 0;
    if (n >= num_slices) {
        for (uint64_t s = 0; s < num_slices; ++s) starts[s] = (uint64_t)(((unsigned __int128)s * n) / num_slices);
        starts[num_slices] = n;
        return num_slices;
    }
    starts[0] = 0;
    for (uint64_t i = 0; i < n; ++i) starts[i + 1] = i;
    starts[n + 1] = n;
    return n + 1;
}

// ---------------------------------------------------------------------------------------------
// device-resident sources
// ---------------------------------------------------------------------------------------------
__global__ void range_kernel(u64 *__restrict__ out, u64 start, u64 step, u64 n)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 st = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += st) out[i] = start + i * step;
}

// Context::range (src/context.rs:419-431): the elements of (start..=end).step_by(step), written on the device.
extern "C" uint64_t vb_range_len(uint64_t start, uint64_t end, uint64_t step)
{
    if (step == 0 || end < start) return 0;
    return (end - start) / step + 1;
}

extern "C" int32_t vb_range(vb_ctx *c, void *out_dev, uint64_t start, uint64_t end, uint64_t step)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    if (step == 0) return set_err(VB_ERR_INVALID, "step must be >= 1 (Rust's step_by panics on 0)");
    const u64 n = vb_range_len(start, end, step);
    if (n == 0) return VB_OK;
    if (!out_dev) return set_err(VB_ERR_INVALID, "out_dev is NULL");
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    const u64 blocks = std::min<u64>((n + 255) / 256, (u64)c->sm_count * 16);
    range_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>((u64 *)out_dev, start, step, n);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------
// synthetic input
// ---------------------------------------------------------------------------------------------
extern "C" int32_t vb_gen_pairs(vb_ctx *c, void *rows_dev, void *keys_dev, void *vals_dev, uint64_t first, uint64_t n,
                                int32_t mode, uint64_t n_distinct, uint64_t rank_base, uint64_t seed_k, uint64_t seed_v,
                                double zipf_s)
{
    if (!c) return set_err(VB_ERR_INVALID, "ctx is NULL");
    if (!rows_dev && !keys_dev) return set_err(VB_ERR_INVALID, "no output buffer");
    if (mode < GEN_UNIFORM || mode > GEN_UNIQUE) return set_err(VB_ERR_INVALID, "bad generator mode");
    if (mode != GEN_UNIQUE && n_distinct == 0) return set_err(VB_ERR_INVALID, "n_distinct must be > 0");
    if (n == 0) return VB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    if (mode == GEN_ZIPF && (c->zipf_n != n_distinct || c->zipf_s != zipf_s)) {
        std::vector<double> cdf(n_distinct);
        long double h = 0;
        for (u64 k = 0; k < n_distinct; ++k) { h += 1.0L / powl((long double)(k + 1), (long double)zipf_s); cdf[k] = (double)h; }
        for (u64 k = 0; k < n_distinct; ++k) cdf[k] = (double)(cdf[k] / (double)h);
        cdf[n_distinct - 1] = 1.0;
        if (c->zipf_cdf) cudaFreeAsync(c->zipf_cdf, c->stream);
        c->zipf_cdf = nullptr;
        CU(cudaMallocAsync((void **)&c->zipf_cdf, n_distinct * 8, c->pool, c->stream));
        CU(cudaMemcpyAsync(c->zipf_cdf, cdf.data(), n_distinct * 8, cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        c->zipf_n = n_distinct;
        c->zipf_s = zipf_s;
    }
    u64 blocks = std::min<u64>((n + 255) / 256, (u64)c->sm_count * 16);
    gen_pairs_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>((u64 *)rows_dev, (u64 *)keys_dev, (u64 *)vals_dev, first, n, mode,
                                                              n_distinct, rank_base, seed_k, seed_v, c->zipf_cdf);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    return VB_OK;
}
