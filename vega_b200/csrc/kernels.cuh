// kernels.cuh — hand-written sm_90a kernels of the shuffle + aggregation path.
//
//   hash_agg_kernel   map-side combine (dependency.rs:191-210) and reduce-side merge
//                     (shuffled_rdd.rs:154-164) as one streaming pass into an L2-resident
//                     open-addressing table: 128-bit evict-first loads, one probe + one RED per row.
//                     OPK_DICT variant builds the key dictionary for group_by_key / cogroup.
//   rp_hist / rp_scatter   one stable radix pass (multisplit by hash(K) % nparts, LSD sort digits):
//                     warp match-any ranking, shared-memory staged tiles, coalesced run writes.
//   scan kernels, CSR boundary, join probe/expand, generators.
//
// Integer / indexing work: HBM- and L2-bound, no tensor cores by design.
#pragma once
#include "common.cuh"

namespace vb {

// ---------------------------------------------------------------------------------------------
// Hash table: open addressing over 4-key buckets, keys and accumulators in separate arrays.
//
// A *dependent* linear-probing loop (30-46 % of rows need a second probe at load 0.48) serialises
// L2 latencies inside divergent warps.  So a bucket is the 4 keys of one 32-byte sector, fetched
// by one pair of 128-bit loads: at load <= 0.6 almost every row resolves in its first probe and the
// kernel issues all probes of a tile before consuming any.  L1::no_allocate on the probes keeps
// the REDs that follow from invalidating L1 lines.
// ---------------------------------------------------------------------------------------------
struct Table {
    u64 *keys;      // [cap + 4]: keys[cap] is the marker of the special slot (1 = EMPTY_KEY present)
    u64 *accs;      // [cap + 4]: combiner per slot (reduce ops); unused by the dictionary
    u32 log_cap;    // cap = 1 << log_cap slots = cap / 4 buckets; log_cap >= 2
    u32 keep_l2;    // 1: bucket probes ask L2 to evict the table last (set by the host when the table fits L2)
    u32 max_probe;  // probe rounds an insert may take before it raises the abort flag (chain_limit, set by the host)
};
constexpr u64 EMPTY_KEY = ~0ull;
constexpr u32 BUCKET = 4;
constexpr u32 HA_MAX_PROBE = 256;   // buckets

// Probe-round limit of the inserts into a table.  A round either moves on to the next bucket or, after a CAS lost to a
// concurrent insert, re-reads the same bucket.  A table that can grow gives up after HA_MAX_PROBE rounds, and the host
// rebuilds it larger.  A table that cannot grow is one the host sized to at least twice the keys that can enter it, and
// its inserts have no round limit: at load <= 0.5 fewer than nb / 2 buckets are full, so a walk passes fewer than nb / 2
// full buckets, and every lost CAS is a slot another key took, of which there are fewer than 2 nb.  So every insert ends
// within 2.5 nb < 2^32 rounds, however many keys share a home bucket and however the inserts interleave (crafted keys
// cost time in the chain length, never a failure).
VB_HD u32 chain_limit(bool can_grow) { return can_grow ? HA_MAX_PROBE : ~0u; }
VB_HD size_t table_bytes(u32 log_cap) { return (((size_t)1 << log_cap) + BUCKET) * 16; }
VB_HD Table table_at(void *base, u32 log_cap)
{
    Table t;
    t.keys = (u64 *)base;
    t.accs = (u64 *)base + (((size_t)1 << log_cap) + BUCKET);
    t.log_cap = log_cap;
    t.keep_l2 = 0;
    t.max_probe = HA_MAX_PROBE;
    return t;
}

struct TableCtl {
    u32 abort;        // set by the kernel: table too full / probe sequence too long → host restarts
    u32 pad;
    unsigned long long n_inserted;
};

enum : int { IN_AOS = 0, IN_SOA = 1, IN_TABLE = 2, IN_ACCS = 3 };   // IN_ACCS: received partials (hash_agg_multi_kernel)
enum : int { OPK_ADD_U64 = 0, OPK_ADD_F64 = 1, OPK_MIN_U64 = 2, OPK_MAX_U64 = 3, OPK_COUNT = 4, OPK_DICT = 5 };

// f64 ADD starts from -0.0, the IEEE additive identity (-0.0 + x == x for every x, +0.0 included): a key whose values
// are all -0.0 sums to -0.0, as vega's fold from the first value does, and any other zero sum to +0.0, in every order.
VB_HD u64 op_identity(int opk) { return opk == OPK_MIN_U64 ? ~0ull : opk == OPK_ADD_F64 ? 0x8000000000000000ull : 0ull; }

template <int OPK>
VB_D void op_red(u64 *acc, u64 v)
{
    if (OPK == OPK_ADD_U64) atomicAdd((unsigned long long *)acc, (unsigned long long)v);
    else if (OPK == OPK_COUNT) atomicAdd((unsigned long long *)acc, 1ull);
    else if (OPK == OPK_ADD_F64) atomicAdd((double *)acc, __longlong_as_double((long long)v));
    else if (OPK == OPK_MIN_U64) atomicMin((unsigned long long *)acc, (unsigned long long)v);
    else if (OPK == OPK_MAX_U64) atomicMax((unsigned long long *)acc, (unsigned long long)v);
}

__global__ void table_init_kernel(Table t, u64 identity)
{
    const u64 cap = 1ull << t.log_cap;
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i < cap + BUCKET; i += stride) {
        t.keys[i] = (i >= cap) ? 0ull : EMPTY_KEY;
        t.accs[i] = identity;
    }
}

struct Bucket4 { u64 k0, k1, k2, k3; };

// one 32-byte sector: 4 candidate keys.  sm_90 loads at most 128 bits per thread, so the sector is read
// by two independent 128-bit loads issued back to back (both in flight together: one L2 latency, not two).
// t.keep_l2: the loads carry an L2 evict_last policy (else evict_normal, the default), so that the streamed input (evict_first) never pushes a table
// that fits L2 out of it (H100: 11 % off the headline step, DESIGN §5).  Not for larger tables, where it made
// the kernel slower.
VB_D Bucket4 ld_bucket(const Table &t, u64 b)
{
    const u64 *p = &t.keys[4 * b];
    Bucket4 r;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%4], %5;\n\t"
                 "ld.global.L1::no_allocate.L2::cache_hint.v2.u64 {%2, %3}, [%4+16], %5;"
                 : "=l"(r.k0), "=l"(r.k1), "=l"(r.k2), "=l"(r.k3)
                 : "l"(p), "l"(t.keep_l2 ? policy_evict_last() : policy_evict_normal()));
    return r;
}
VB_D int bucket_find(const Bucket4 &b, u64 key)
{
    return b.k0 == key ? 0 : b.k1 == key ? 1 : b.k2 == key ? 2 : b.k3 == key ? 3 : -1;
}

constexpr int HA_THREADS = 256;
constexpr int HA_ROWS = 4;
constexpr int HA_TILE = HA_THREADS * HA_ROWS;

VB_D u64 home_bucket(u64 key, u32 log_cap) { return slot_hash(key) >> (64 - (log_cap - 2)); }

// Resolve `key` starting from bucket `b` whose content `bk` is already loaded: find it, or claim the
// first empty slot with a CAS, or move on to the next bucket.  Slots only ever go EMPTY → key and are
// claimed first-empty-first, so a key can never end up in two slots (a stale view is an older view).
// on_hit(slot) combines into the slot's accumulator(s).
template <class OnHit>
VB_D bool table_resolve_with(const Table &t, u64 b, Bucket4 bk, u64 key, u32 &inserted, OnHit &&on_hit)
{
    const u64 nb_mask = (1ull << (t.log_cap - 2)) - 1;
#pragma unroll 1
    for (u32 probe = 0; probe < t.max_probe; ++probe) {
        int hit = bucket_find(bk, key);
        if (hit < 0) {
            const int e = bucket_find(bk, EMPTY_KEY);
            if (e < 0) {
                b = (b + 1) & nb_mask;
            } else {
                const u64 old = atomicCAS((unsigned long long *)&t.keys[4 * b + e], (unsigned long long)EMPTY_KEY, (unsigned long long)key);
                if (old == EMPTY_KEY) { ++inserted; hit = e; }
                else if (old == key) hit = e;
            }
        }
        if (hit >= 0) {
            on_hit(4 * b + (u64)hit);
            return true;
        }
        bk = ld_bucket(t, b);
    }
    return false;
}
template <int OPK>
VB_D bool table_resolve(const Table &t, u64 b, Bucket4 bk, u64 key, u64 v, u32 &slot_idx, u32 &inserted)
{
    return table_resolve_with(t, b, bk, key, inserted, [&](u64 s) { op_red<OPK>(&t.accs[s], v); slot_idx = (u32)s; });
}

// ---- per-CTA hot-key cache (skewed keys) -------------------------------------------------------
// With Zipf(1.1) keys the hottest key owns 12 % of the rows: 1.2e8 REDs to ONE L2 address serialise
// (an order of magnitude slower than uniform keys).  Each CTA therefore keeps a small 2-choice cache
// of (key, partial combiner) in shared memory: rows whose key is cached are combined with a
// shared-memory atomic and never reach L2; the cache is flushed into the table once, at CTA exit.
// Keys are cached first-come (hot keys come first with high probability).  For uniformly distributed
// keys nothing hits, so every CTA measures its hit rate over its first 16 tiles and switches the
// cache off below 1/16.
constexpr int HC_SLOTS = 1024;

template <int OPK>
VB_D void op_shared(u64 *acc, u64 v)
{
    if (OPK == OPK_ADD_U64) atomicAdd((unsigned long long *)acc, (unsigned long long)v);
    else if (OPK == OPK_COUNT) atomicAdd((unsigned long long *)acc, 1ull);
    else if (OPK == OPK_ADD_F64) atomicAdd((double *)acc, __longlong_as_double((long long)v));
    else if (OPK == OPK_MIN_U64) atomicMin((unsigned long long *)acc, (unsigned long long)v);
    else if (OPK == OPK_MAX_U64) atomicMax((unsigned long long *)acc, (unsigned long long)v);
}

// 0: not absorbed (row goes to the table); 1: hit an already cached key; 2: claimed an empty cache slot.
// on_hit(i) combines the row into cache slot i.
template <u32 SLOTS, class OnHit>
VB_D int cache_combine_with(u64 *hc_keys, u64 h, u64 key, OnHit &&on_hit)
{
    const u32 i1 = (u32)h & (SLOTS - 1), i2 = (u32)(h >> 10) & (SLOTS - 1);
    const u64 c1 = hc_keys[i1];
    if (c1 == key) { on_hit(i1); return 1; }
    const u64 c2 = hc_keys[i2];
    if (c2 == key) { on_hit(i2); return 1; }
    u32 slot;
    if (c1 == EMPTY_KEY) slot = i1;
    else if (c2 == EMPTY_KEY) slot = i2;
    else return 0;
    const u64 old = atomicCAS((unsigned long long *)&hc_keys[slot], (unsigned long long)EMPTY_KEY, (unsigned long long)key);
    if (old == EMPTY_KEY) { on_hit(slot); return 2; }
    if (old == key) { on_hit(slot); return 1; }
    return 0;
}
template <int OPK>
VB_D int cache_combine(u64 *hc_keys, u64 *hc_acc, u64 h, u64 key, u64 v)
{
    return cache_combine_with<HC_SLOTS>(hc_keys, h, key, [&](u32 i) { op_shared<OPK>(&hc_acc[i], v); });
}

template <int ROWS, class OnHit>
VB_D void ha_probe_rows(const Table &t, TableCtl *ctl, const u64 (&k)[ROWS], bool (&ok)[ROWS], const u64 (&h)[ROWS], u32 &my_inserts,
                        OnHit &&on_hit);

// The per-tile work shared by the register-staged and the bulk-staged kernels: thread-private rows
// k/v/ok (HA_ROWS of them, row j of the thread is input row row0 + j * HA_THREADS) → special key,
// hot-key cache, then lockstep probe rounds with one RED per resolved row.
template <int OPK, int TX, bool CACHE, int ROWS>
VB_D void ha_process_rows(const Table &t, TableCtl *ctl, u64 (&k)[ROWS], u64 (&v)[ROWS], bool (&ok)[ROWS], u64 row0,
                          u32 *__restrict__ slot_out, u64 *hc_keys, u64 *hc_acc, bool use_cache, u32 &my_inserts, u32 &my_hits)
{
    const u64 cap = 1ull << t.log_cap;
    // f64 MIN/MAX fold like Rust's f64::min / f64::max: a NaN value is ignored (it becomes the op's identity, so the
    // key is still inserted), and a key whose values are all NaN finalises to tx_inv(identity), which is a NaN.
    constexpr bool NAN_IS_IDENTITY = (TX == TX_F64) && (OPK == OPK_MIN_U64 || OPK == OPK_MAX_U64);
    u64 h[ROWS];
#pragma unroll
    for (int j = 0; j < ROWS; ++j) {
        h[j] = slot_hash(k[j]);
        if (NAN_IS_IDENTITY && (v[j] & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull) v[j] = op_identity(OPK);
        else if (TX != TX_NONE) v[j] = tx_fwd(v[j], TX);
        if (ok[j] && k[j] == EMPTY_KEY) {           // a real key equal to the empty marker: special slot
            t.keys[cap] = 1ull;
            op_red<OPK>(&t.accs[cap], v[j]);
            if (OPK == OPK_DICT) st_stream_u32(slot_out + row0 + (u64)j * HA_THREADS, (u32)cap);
            ok[j] = false;
        }
    }
    if (CACHE && use_cache) {
#pragma unroll
        for (int j = 0; j < ROWS; ++j) {
            if (!ok[j]) continue;
            const int c = cache_combine<OPK>(hc_keys, hc_acc, h[j], k[j], v[j]);
            if (c) { ok[j] = false; my_hits += (c == 1); }
        }
    }
    ha_probe_rows(t, ctl, k, ok, h, my_inserts, [&](u64 sl, int j) {
        op_red<OPK>(&t.accs[sl], v[j]);
        if (OPK == OPK_DICT) st_stream_u32(slot_out + row0 + (u64)j * HA_THREADS, (u32)sl);
    });
}

// Lockstep probe/insert of the pending rows (ok[j]) of one thread, with hashes h[j]; on_hit(slot, j) once per
// resolved row.  A row still pending after t.max_probe probe rounds raises the table's abort flag.
template <int ROWS, class OnHit>
VB_D void ha_probe_rows(const Table &t, TableCtl *ctl, const u64 (&k)[ROWS], bool (&ok)[ROWS], const u64 (&h)[ROWS], u32 &my_inserts,
                        OnHit &&on_hit)
{
    const u32 hshift = 64 - (t.log_cap - 2);
    // Probe rounds run in lockstep over the ROWS rows of a thread: every round first consumes the
    // buckets loaded by the previous one, then issues the next probes of all unresolved rows together,
    // so a tile costs max-over-rows (not sum-over-rows) dependent L2 latencies.
    Bucket4 bk[ROWS];
    u64 bidx[ROWS];
    const u64 nb_mask = (1ull << (t.log_cap - 2)) - 1;
#pragma unroll
    for (int j = 0; j < ROWS; ++j) {
        bidx[j] = h[j] >> hshift;
        if (ok[j]) bk[j] = ld_bucket(t, bidx[j]);
    }
    bool pending = true;
#pragma unroll 1
    for (u32 probe = 0; pending && probe < t.max_probe; ++probe) {
        pending = false;
#pragma unroll
        for (int j = 0; j < ROWS; ++j) {
            if (!ok[j]) continue;
            int hit = bucket_find(bk[j], k[j]);
            if (hit < 0) {
                const int e = bucket_find(bk[j], EMPTY_KEY);
                if (e < 0) {
                    bidx[j] = (bidx[j] + 1) & nb_mask;                    // bucket full: next bucket
                } else {
                    const u64 old = atomicCAS((unsigned long long *)&t.keys[4 * bidx[j] + e], (unsigned long long)EMPTY_KEY,
                                              (unsigned long long)k[j]);
                    if (old == EMPTY_KEY) { ++my_inserts; hit = e; }
                    else if (old == k[j]) hit = e;                        // else: lost the slot, re-read this bucket
                }
            }
            if (hit >= 0) {
                on_hit(4 * bidx[j] + (u64)hit, j);
                ok[j] = false;
            } else {
                pending = true;
            }
        }
        if (pending) {
#pragma unroll
            for (int j = 0; j < ROWS; ++j)
                if (ok[j]) bk[j] = ld_bucket(t, bidx[j]);
        }
    }
    if (pending) atomicExch(&ctl->abort, 1u);   // a row took more than t.max_probe probe rounds
}

// One pass over n rows.  IN_AOS: a = rows (16 B each).  IN_SOA: a = keys, b = vals (b may be
// NULL for COUNT/DICT).  IN_TABLE: a/b = keys/accs of a source table of n-1 slots + the special slot.
// TX: order-preserving value transform applied on load (MIN/MAX over i64/f64).
template <int IN, int OPK, int TX>
__global__ void __launch_bounds__(HA_THREADS, 3)   // 3 CTAs/SM: the A/B winner against 2 and 4
hash_agg_kernel(const u64 *__restrict__ a, const u64 *__restrict__ b, u64 n, Table t, TableCtl *ctl, u64 max_inserts,
                u32 *__restrict__ slot_out)
{
    constexpr bool CACHE = (OPK != OPK_DICT) && (IN != IN_TABLE);
    constexpr int OPK_FLUSH = (OPK == OPK_COUNT) ? OPK_ADD_U64 : OPK;      // partial counts are summed
    __shared__ u32 s_inserts;
    __shared__ u32 s_abort;
    __shared__ u32 s_hits;
    __shared__ u64 hc_keys[CACHE ? HC_SLOTS : 1];
    __shared__ u64 hc_acc[CACHE ? HC_SLOTS : 1];
    const u32 tid = threadIdx.x;
    if (tid == 0) { s_inserts = 0; s_abort = 0; s_hits = 0; }
    if (CACHE)
        for (u32 i = tid; i < HC_SLOTS; i += HA_THREADS) { hc_keys[i] = EMPTY_KEY; hc_acc[i] = op_identity(OPK); }
    __syncthreads();
    const u64 pol = policy_evict_first();
    const u64 n_tiles = (n + HA_TILE - 1) / HA_TILE;
    u32 my_inserts = 0, my_hits = 0;
    u32 iter = 0;
    bool use_cache = CACHE;
    for (u64 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++iter) {
        const u64 base = tile * HA_TILE;
        u64 k[HA_ROWS], v[HA_ROWS];
        bool ok[HA_ROWS];
#pragma unroll
        for (int j = 0; j < HA_ROWS; ++j) {
            const u64 idx = base + (u64)j * HA_THREADS + tid;
            ok[j] = idx < n;
            k[j] = 0; v[j] = 0;
            if (ok[j]) {
                if (IN == IN_AOS) {
                    ulonglong2 r = ld_stream_u64x2(a + 2 * idx, pol);
                    k[j] = r.x; v[j] = r.y;
                } else if (IN == IN_SOA) {
                    k[j] = ld_stream_u64(a + idx, pol);
                    if (OPK != OPK_COUNT && OPK != OPK_DICT) v[j] = ld_stream_u64(b + idx, pol);
                } else {
                    k[j] = ld_stream_u64(a + idx, pol);
                    v[j] = ld_stream_u64(b + idx, pol);
                    if (idx == n - 1) { ok[j] = (k[j] == 1ull); k[j] = EMPTY_KEY; }   // special slot
                    else if (k[j] == EMPTY_KEY) ok[j] = false;                       // unoccupied
                }
            }
        }
        ha_process_rows<OPK, TX, CACHE, HA_ROWS>(t, ctl, k, v, ok, base + tid, slot_out, hc_keys, hc_acc, use_cache, my_inserts, my_hits);
        if ((iter & 15u) == 15u) {   // periodic load-factor check (+ cache verdict); iter is CTA-uniform
            u32 w = __reduce_add_sync(0xffffffffu, my_inserts);
            my_inserts = 0;
            if ((tid & 31u) == 0 && w) atomicAdd(&s_inserts, w);
            if (CACHE && iter == 15u) {
                u32 hw = __reduce_add_sync(0xffffffffu, my_hits);
                if ((tid & 31u) == 0 && hw) atomicAdd(&s_hits, hw);
            }
            __syncthreads();
            if (tid == 0) {
                u32 c = s_inserts;
                s_inserts = 0;
                u64 tot = atomicAdd(&ctl->n_inserted, (unsigned long long)c) + c;
                u32 ab = ld_volatile_u32(&ctl->abort);
                if (tot > max_inserts) { ab = 1; atomicExch(&ctl->abort, 1u); }
                s_abort = ab;
            }
            __syncthreads();
            if (s_abort) return;
            if (CACHE && iter == 15u && s_hits * 16u < 16u * HA_TILE) use_cache = false;   // < 1/16 of the first 16 tiles
        }
    }
    if (CACHE) {   // flush the cache into the table (merge op)
        __syncthreads();
        for (u32 i = tid; i < HC_SLOTS; i += HA_THREADS) {
            const u64 key = hc_keys[i];
            if (key == EMPTY_KEY) continue;
            const u64 hb = home_bucket(key, t.log_cap);
            u32 slot = 0;
            if (!table_resolve<OPK_FLUSH>(t, hb, ld_bucket(t, hb), key, hc_acc[i], slot, my_inserts)) atomicExch(&ctl->abort, 1u);
        }
    }
    u32 w = __reduce_add_sync(0xffffffffu, my_inserts);
    if ((tid & 31u) == 0 && w) atomicAdd(&s_inserts, w);
    __syncthreads();
    if (tid == 0 && s_inserts) atomicAdd(&ctl->n_inserted, (unsigned long long)s_inserts);
}

// ---- bulk-staged variant (TMA engine) ---------------------------------------------------------------
// Same aggregation, different input path.  ncu on the register-staged kernel above shows the SM's
// L1TEX→XBAR request port as the busiest unit (l1tex__m_l1tex2xbar_req_cycles_active 81 %; one request
// per cycle per SM, and a random probe, a RED and every 128 B of the stream each cost one), with the
// port idle whenever all resident CTAs sit in the DRAM-latency phase of their tile.  Here a producer
// warp keeps HB_STAGES input tiles in flight per CTA with cp.async.bulk + mbarrier (no registers, no
// LSU instructions for the stream); the 8 consumer warps only ever wait on L2-latency probes, so the
// request port stays busy.  Full tiles only (16-byte aligned, 16 KB each); the host sends inputs with
// unaligned bases to the register-staged kernel, and the sub-tile tail is read with plain loads.
#ifndef VB_HB_STAGES
#define VB_HB_STAGES 3
#endif
// 4 rows per thread x 2 CTAs per SM: the H100 A/B winner (reduce_by_key 1e9 rows, 1e6 keys: 5 % ahead of 2 x 4;
// 2 x 4 with 4 stages and 1 x 7 were far slower; 4 x 3 spills)
#ifndef VB_HB_ROWS
#define VB_HB_ROWS 4
#endif
#ifndef VB_HB_CTAS
#define VB_HB_CTAS 2
#endif
constexpr int HB_STAGES = VB_HB_STAGES;
constexpr int HB_ROWS = VB_HB_ROWS;             // rows per consumer thread per tile
constexpr int HB_TILE = HA_THREADS * HB_ROWS;
constexpr int HB_THREADS = HA_THREADS + 32;     // 8 consumer warps + 1 producer warp
constexpr size_t hb_smem_bytes(bool has_vals) { return (size_t)HB_STAGES * HB_TILE * (has_vals ? 16 : 8); }

template <int IN, int OPK, int TX>
__global__ void __launch_bounds__(HB_THREADS, VB_HB_CTAS)
hash_agg_bulk_kernel(const u64 *__restrict__ a, const u64 *__restrict__ b, u64 n, Table t, TableCtl *ctl, u64 max_inserts,
                     u32 *__restrict__ slot_out)
{
    static_assert(IN == IN_AOS || IN == IN_SOA, "table merges use hash_agg_kernel");
    constexpr bool CACHE = (OPK != OPK_DICT);
    constexpr int OPK_FLUSH = (OPK == OPK_COUNT) ? OPK_ADD_U64 : OPK;
    constexpr bool HAS_V = (IN == IN_AOS) || (OPK != OPK_COUNT && OPK != OPK_DICT);
    constexpr u32 STAGE_BYTES = HB_TILE * (HAS_V ? 16 : 8);
    extern __shared__ __align__(128) unsigned char hb_stage[];      // [HB_STAGES][STAGE_BYTES]
    __shared__ __align__(8) u64 full_bar[HB_STAGES];
    __shared__ __align__(8) u64 empty_bar[HB_STAGES];
    __shared__ u32 s_inserts;
    __shared__ u32 s_abort;
    __shared__ u32 s_hits;
    __shared__ u64 hc_keys[CACHE ? HC_SLOTS : 1];
    __shared__ u64 hc_acc[CACHE ? HC_SLOTS : 1];
    const u32 tid = threadIdx.x;
    if (tid == 0) {
        s_inserts = 0; s_abort = 0; s_hits = 0;
#pragma unroll
        for (int s = 0; s < HB_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], HA_THREADS / 32); }
        mbar_fence_init();
    }
    if (CACHE)
        for (u32 i = tid; i < HC_SLOTS; i += HB_THREADS) { hc_keys[i] = EMPTY_KEY; hc_acc[i] = op_identity(OPK); }
    __syncthreads();
    const u64 n_full = n / HB_TILE;                         // tiles that go through the copy engine

    if (tid >= HA_THREADS) {                                // ===== producer warp =====
        if (tid == HA_THREADS) {
            const u64 pol = policy_evict_first();
            u32 i = 0;
            for (u64 tile = blockIdx.x; tile < n_full; tile += gridDim.x, ++i) {
                const u32 s = i % HB_STAGES;
                if (i >= HB_STAGES) mbar_wait(&empty_bar[s], ((i / HB_STAGES) & 1u) ^ 1u);   // consumers released the slot
                unsigned char *dst = hb_stage + (size_t)s * STAGE_BYTES;
                mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
                if (IN == IN_AOS) {
                    bulk_g2s(dst, a + 2 * tile * HB_TILE, STAGE_BYTES, &full_bar[s], pol);
                } else {
                    bulk_g2s(dst, a + tile * HB_TILE, HB_TILE * 8, &full_bar[s], pol);
                    if (HAS_V) bulk_g2s(dst + HB_TILE * 8, b + tile * HB_TILE, HB_TILE * 8, &full_bar[s], pol);
                }
            }
        }
        return;                                             // every copy it issued is awaited by the consumers below
    }

    // ===== consumer warps =====
    u32 my_inserts = 0, my_hits = 0;
    u32 iter = 0;
    bool use_cache = CACHE;
    bool drain = false;        // after an abort: keep the pipeline moving (copies in flight target this CTA's smem), skip the work
    for (u64 tile = blockIdx.x; tile < n_full; tile += gridDim.x, ++iter) {
        const u32 s = iter % HB_STAGES;
        mbar_wait(&full_bar[s], (iter / HB_STAGES) & 1u);
        const unsigned char *src = hb_stage + (size_t)s * STAGE_BYTES;
        u64 k[HB_ROWS], v[HB_ROWS];
        bool ok[HB_ROWS];
#pragma unroll
        for (int j = 0; j < HB_ROWS; ++j) {
            const u32 r = (u32)j * HA_THREADS + tid;
            ok[j] = !drain;
            if (IN == IN_AOS) {
                const ulonglong2 row = reinterpret_cast<const ulonglong2 *>(src)[r];
                k[j] = row.x; v[j] = row.y;
            } else {
                k[j] = reinterpret_cast<const u64 *>(src)[r];
                v[j] = HAS_V ? reinterpret_cast<const u64 *>(src + HB_TILE * 8)[r] : 0ull;
            }
        }
        // The slot is refilled by the copy engine (async proxy) while these reads went through the generic
        // proxy: a proxy fence orders them before the release (without it ~1e-7 of the rows were read torn).
        fence_proxy_async();
        __syncwarp();
        if ((tid & 31u) == 0) mbar_arrive(&empty_bar[s]);   // this warp's rows are in registers: slot may be refilled
        if (!drain) ha_process_rows<OPK, TX, CACHE, HB_ROWS>(t, ctl, k, v, ok, tile * HB_TILE + tid, slot_out, hc_keys, hc_acc, use_cache, my_inserts, my_hits);
        if ((iter & 15u) == 15u) {   // periodic load-factor check (+ cache verdict); iter is CTA-uniform
            u32 w = __reduce_add_sync(0xffffffffu, my_inserts);
            my_inserts = 0;
            if ((tid & 31u) == 0 && w) atomicAdd(&s_inserts, w);
            if (CACHE && iter == 15u) {
                u32 hw = __reduce_add_sync(0xffffffffu, my_hits);
                if ((tid & 31u) == 0 && hw) atomicAdd(&s_hits, hw);
            }
            named_bar_sync(1, HA_THREADS);
            if (tid == 0) {
                u32 c = s_inserts;
                s_inserts = 0;
                u64 tot = atomicAdd(&ctl->n_inserted, (unsigned long long)c) + c;
                u32 ab = ld_volatile_u32(&ctl->abort);
                if (tot > max_inserts) { ab = 1; atomicExch(&ctl->abort, 1u); }
                s_abort = ab;
            }
            named_bar_sync(1, HA_THREADS);
            if (s_abort) drain = true;
            if (CACHE && iter == 15u && s_hits * 16u < 16u * HB_TILE) use_cache = false;
        }
    }
    // tail (< HB_TILE rows): plain loads, by the CTA whose turn it would have been
    if (!drain && (n % HB_TILE) && blockIdx.x == (u32)(n_full % gridDim.x)) {
        const u64 pol = policy_evict_first();
        const u64 base = n_full * HB_TILE;
        u64 k[HB_ROWS], v[HB_ROWS];
        bool ok[HB_ROWS];
#pragma unroll
        for (int j = 0; j < HB_ROWS; ++j) {
            const u64 idx = base + (u64)j * HA_THREADS + tid;
            ok[j] = idx < n;
            k[j] = 0; v[j] = 0;
            if (ok[j]) {
                if (IN == IN_AOS) { ulonglong2 r = ld_stream_u64x2(a + 2 * idx, pol); k[j] = r.x; v[j] = r.y; }
                else { k[j] = ld_stream_u64(a + idx, pol); if (HAS_V) v[j] = ld_stream_u64(b + idx, pol); }
            }
        }
        ha_process_rows<OPK, TX, CACHE, HB_ROWS>(t, ctl, k, v, ok, base + tid, slot_out, hc_keys, hc_acc, use_cache, my_inserts, my_hits);
    }
    if (CACHE) {   // flush the cache into the table (merge op)
        named_bar_sync(1, HA_THREADS);
        if (!drain)
            for (u32 i = tid; i < HC_SLOTS; i += HA_THREADS) {
                const u64 key = hc_keys[i];
                if (key == EMPTY_KEY) continue;
                const u64 hb = home_bucket(key, t.log_cap);
                u32 slot = 0;
                if (!table_resolve<OPK_FLUSH>(t, hb, ld_bucket(t, hb), key, hc_acc[i], slot, my_inserts)) atomicExch(&ctl->abort, 1u);
            }
    }
    u32 w = __reduce_add_sync(0xffffffffu, my_inserts);
    if ((tid & 31u) == 0 && w) atomicAdd(&s_inserts, w);
    named_bar_sync(1, HA_THREADS);
    if (tid == 0 && s_inserts) atomicAdd(&ctl->n_inserted, (unsigned long long)s_inserts);
}

// ---- several aggregates per key (combine_by_key) -------------------------------------------------------
// Table: keys[cap + 4], then n accumulator columns accs[a][cap + 4] (column a at t.accs + a * (cap + 4)), each
// kept apart from the keys and from each other for the same reason the single-column table is not interleaved.
// A row costs one probe/insert (ha_probe_rows, shared with the kernels above) and then one RED per accumulator.
// Up to MA_MAX_COLS input value columns; the column count is a template parameter (register arrays are only
// indexed by compile-time indices: an accumulator picks its column with an unrolled compare chain), the
// accumulator list (op, order transform, input column) is a kernel argument read from parameter space.
constexpr int MA_MAX_COLS = 4;
constexpr int MA_MAX_ACCS = 8;
// One byte per accumulator, packed into a u64 so a run-time accumulator index is a shift, not a local-memory array.
struct AccSpec {
    u32 n;      // accumulators
    u64 op;     // OPK_ADD_U64 / OPK_ADD_F64 / OPK_MIN_U64 / OPK_MAX_U64 / OPK_COUNT
    u64 tx;     // order transform on load (MIN/MAX over i64 / f64; NaN -> identity for f64)
    u64 src;    // input value column (table merges: accumulator a reads source column a)
};
VB_HD int spec_at(u64 packed, int a) { return (int)(packed >> (8 * a)) & 0xFF; }
VB_HD void spec_set(u64 &packed, int a, int v) { packed = (packed & ~(0xFFull << (8 * a))) | ((u64)(v & 0xFF) << (8 * a)); }
struct MaCols {
    const u64 *c[MA_MAX_COLS];           // value columns (IN_TABLE / IN_ACCS: c[0] = the source's first accumulator column)
    u64 stride;                          // IN_TABLE / IN_ACCS: distance between the source's accumulator columns
};
VB_HD size_t table_bytes_multi(u32 log_cap, u32 n_acc) { return (((size_t)1 << log_cap) + BUCKET) * 8 * (1 + n_acc); }
VB_HD u64 acc_stride(u32 log_cap) { return (1ull << log_cap) + BUCKET; }

// Hot-key cache of the multi kernels: 512 slots x (key + n partials) in dynamic shared memory (36 KB at 8
// accumulators), so that stage + cache of the bulk variant still fit two CTAs per SM at 4 value columns.
constexpr u32 MA_HC_SLOTS = 512;
VB_HD size_t ma_cache_bytes(u32 n_acc) { return (size_t)MA_HC_SLOTS * 8 * (1 + n_acc); }
// Rows per thread: 4 with one value column, 2 with more (the tile's values live in registers until the REDs; the
// bulk kernel spilled at 2 columns x 4 rows under its 2-CTA register budget).
template <int NV> constexpr int ma_rows() { return NV == 1 ? 4 : 2; }
#ifndef VB_MA_STAGES
#define VB_MA_STAGES 3
#endif
constexpr int MA_STAGES = VB_MA_STAGES;
template <int NV> constexpr size_t ma_stage_bytes() { return (size_t)HA_THREADS * ma_rows<NV>() * 8 * (1 + NV); }
template <int NV> constexpr size_t ma_bulk_smem(u32 n_acc) { return MA_STAGES * ma_stage_bytes<NV>() + ma_cache_bytes(n_acc); }

// one RED with a run-time op (warp-uniform: every lane runs the same accumulator list); global or shared memory
VB_D void op_red_rt(u64 *acc, int opk, u64 v)
{
    switch (opk) {
    case OPK_ADD_U64: atomicAdd((unsigned long long *)acc, (unsigned long long)v); break;
    case OPK_ADD_F64: atomicAdd((double *)acc, __longlong_as_double((long long)v)); break;
    case OPK_MIN_U64: atomicMin((unsigned long long *)acc, (unsigned long long)v); break;
    case OPK_MAX_U64: atomicMax((unsigned long long *)acc, (unsigned long long)v); break;
    default: atomicAdd((unsigned long long *)acc, 1ull); break;       // OPK_COUNT
    }
}
VB_HD int merge_op(int opk) { return opk == OPK_COUNT ? OPK_ADD_U64 : opk; }   // partial counts are summed

template <int NV, int ROWS>
VB_D u64 ma_pick(const u64 (&v)[NV][ROWS], int src, int j)
{
    u64 x = v[0][j];
#pragma unroll
    for (int c = 1; c < NV; ++c)
        if (src == c) x = v[c][j];
    return x;
}
// the value accumulator `a` folds: order transform, and a NaN becomes the identity of f64 MIN/MAX (tx is set only for MIN/MAX)
VB_D u64 ma_prep(u64 x, int opk, int tx)
{
    if (tx == TX_F64 && (x & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull) return op_identity(opk);
    return tx_fwd(x, tx);
}

__global__ void table_init_multi_kernel(Table t, AccSpec sp)
{
    const u64 cap = 1ull << t.log_cap, stride = acc_stride(t.log_cap);
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 step = (u64)gridDim.x * blockDim.x;
    for (; i < stride; i += step) {
        t.keys[i] = (i >= cap) ? 0ull : EMPTY_KEY;
        for (int a = 0; a < (int)sp.n; ++a) t.accs[(u64)a * stride + i] = op_identity(spec_at(sp.op, a));
    }
}

// Special key, hot-key cache, probe + one RED per accumulator for ROWS rows of a thread.  IN_SOA: v[c][j] is the
// value of column c; IN_TABLE (merge): v[0][j] is the source slot, whose accumulators are read at the RED; IN_ACCS
// (import merge): v[0][j] is the received row, whose plain-value partials are read at the RED and order-transformed.
template <int IN, int NV, int ROWS, bool CACHE>
VB_D void ma_process_rows(const Table &t, TableCtl *ctl, const AccSpec &sp, const MaCols &src, u64 (&k)[ROWS], u64 (&v)[NV][ROWS],
                          bool (&ok)[ROWS], u64 *hc_keys, u64 *hc_acc, bool use_cache, u32 &my_inserts, u32 &my_hits)
{
    const u64 cap = 1ull << t.log_cap, stride = acc_stride(t.log_cap);
    const u64 ops = sp.op, txs = sp.tx, srcs = sp.src;
    const int n_acc = (int)sp.n;
    // not unrolled: 8 accumulators x ROWS rows x 3 call sites of an unrolled RED chain spilled
    auto red_all = [&](u64 *base, u64 col_stride, int j) {
#pragma unroll 1
        for (int a = 0; a < n_acc; ++a) {
            const int op = spec_at(ops, a);
            u64 x;
            if constexpr (IN == IN_TABLE) x = ld_cg_u64(src.c[0] + (u64)a * src.stride + v[0][j]);
            else if constexpr (IN == IN_ACCS) x = ma_prep(ld_cg_u64(src.c[0] + (u64)a * src.stride + v[0][j]), op, spec_at(txs, a));
            else x = ma_prep(ma_pick<NV, ROWS>(v, spec_at(srcs, a), j), op, spec_at(txs, a));
            op_red_rt(base + (u64)a * col_stride, op, x);
        }
    };
    u64 h[ROWS];
#pragma unroll
    for (int j = 0; j < ROWS; ++j) {
        h[j] = slot_hash(k[j]);
        if (ok[j] && k[j] == EMPTY_KEY) {           // a real key equal to the empty marker: special slot
            t.keys[cap] = 1ull;
            red_all(t.accs + cap, stride, j);
            ok[j] = false;
        }
    }
    if (CACHE && use_cache) {
#pragma unroll
        for (int j = 0; j < ROWS; ++j) {
            if (!ok[j]) continue;
            const int c = cache_combine_with<MA_HC_SLOTS>(hc_keys, h[j], k[j], [&](u32 i) { red_all(hc_acc + i, MA_HC_SLOTS, j); });
            if (c) { ok[j] = false; my_hits += (c == 1); }
        }
    }
    ha_probe_rows(t, ctl, k, ok, h, my_inserts, [&](u64 sl, int j) { red_all(t.accs + sl, stride, j); });
}

template <u32 NT>
VB_D void ma_cache_init(u64 *hc_keys, u64 *hc_acc, const AccSpec &sp, u32 tid)
{
    for (u32 i = tid; i < MA_HC_SLOTS; i += NT) {
        hc_keys[i] = EMPTY_KEY;
        for (int a = 0; a < (int)sp.n; ++a) hc_acc[a * MA_HC_SLOTS + i] = op_identity(spec_at(sp.op, a));
    }
}
// flush the CTA's cached partials into the table, combined with each accumulator's merge op
VB_D void ma_cache_flush(const Table &t, TableCtl *ctl, const AccSpec &sp, const u64 *hc_keys, const u64 *hc_acc, u32 tid, u32 &my_inserts)
{
    const u64 stride = acc_stride(t.log_cap);
    for (u32 i = tid; i < MA_HC_SLOTS; i += HA_THREADS) {
        const u64 key = hc_keys[i];
        if (key == EMPTY_KEY) continue;
        const u64 hb = home_bucket(key, t.log_cap);
        if (!table_resolve_with(t, hb, ld_bucket(t, hb), key, my_inserts, [&](u64 s) {
                for (int a = 0; a < (int)sp.n; ++a) op_red_rt(t.accs + (u64)a * stride + s, merge_op(spec_at(sp.op, a)), hc_acc[a * MA_HC_SLOTS + i]);
            }))
            atomicExch(&ctl->abort, 1u);
    }
}

// Periodic load-factor check of the multi kernels (+ the cache verdict after the first 16 tiles), over the
// HA_THREADS consumer threads (named barrier 1).  Returns true when the table overflowed (host restarts larger).
template <bool CACHE>
VB_D bool ma_check(TableCtl *ctl, u64 max_inserts, u32 iter, u32 tile_rows, u32 &my_inserts, u32 my_hits, bool &use_cache, u32 *s_inserts,
                   u32 *s_hits, u32 *s_abort)
{
    const u32 tid = threadIdx.x;
    u32 w = __reduce_add_sync(0xffffffffu, my_inserts);
    my_inserts = 0;
    if ((tid & 31u) == 0 && w) atomicAdd(s_inserts, w);
    if (CACHE && iter == 15u) {
        u32 hw = __reduce_add_sync(0xffffffffu, my_hits);
        if ((tid & 31u) == 0 && hw) atomicAdd(s_hits, hw);
    }
    named_bar_sync(1, HA_THREADS);
    if (tid == 0) {
        u32 c = *s_inserts;
        *s_inserts = 0;
        u64 tot = atomicAdd(&ctl->n_inserted, (unsigned long long)c) + c;
        u32 ab = ld_volatile_u32(&ctl->abort);
        if (tot > max_inserts) { ab = 1; atomicExch(&ctl->abort, 1u); }
        *s_abort = ab;
    }
    named_bar_sync(1, HA_THREADS);
    if (CACHE && iter == 15u && *s_hits * 16u < 16u * tile_rows) use_cache = false;   // < 1/16 of the first 16 tiles
    return *s_abort != 0;
}

// Register-staged multi-aggregate combine: IN_SOA (keys + NV value columns), IN_TABLE (merge of a per-map
// table of the same spec: NV = 1, sp = the merge spec) or IN_ACCS (merge of partials received from other ranks:
// keys[n] + accumulator a of row i at cols.c[0][a * n + i] in plain value form, NV = 1, sp = the merge ops with the
// map spec's order transforms; every row is a real key, and a key arrives at most once per rank, so no hot-key
// cache).  Dynamic shared memory: the hot-key cache (IN_SOA).
template <int IN, int NV>
__global__ void __launch_bounds__(HA_THREADS, 2)
hash_agg_multi_kernel(const u64 *__restrict__ keys, MaCols cols, u64 n, Table t, AccSpec sp, TableCtl *ctl, u64 max_inserts)
{
    static_assert(IN == IN_SOA || ((IN == IN_TABLE || IN == IN_ACCS) && NV == 1), "SoA rows, a table merge or received partials");
    constexpr bool CACHE = (IN == IN_SOA);
    constexpr int ROWS = ma_rows<NV>();
    constexpr int TILE = HA_THREADS * ROWS;
    extern __shared__ __align__(16) u64 ma_cache[];          // hc_keys[MA_HC_SLOTS], hc_acc[n][MA_HC_SLOTS]
    __shared__ u32 s_inserts, s_abort, s_hits;
    u64 *hc_keys = ma_cache, *hc_acc = ma_cache + MA_HC_SLOTS;
    const u32 tid = threadIdx.x;
    if (tid == 0) { s_inserts = 0; s_abort = 0; s_hits = 0; }
    if (CACHE) ma_cache_init<HA_THREADS>(hc_keys, hc_acc, sp, tid);
    __syncthreads();
    const u64 pol = policy_evict_first();
    const u64 n_tiles = (n + TILE - 1) / TILE;
    u32 my_inserts = 0, my_hits = 0, iter = 0;
    bool use_cache = CACHE;
    for (u64 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++iter) {
        const u64 base = tile * TILE;
        u64 k[ROWS], v[NV][ROWS];
        bool ok[ROWS];
#pragma unroll
        for (int j = 0; j < ROWS; ++j) {
            const u64 idx = base + (u64)j * HA_THREADS + tid;
            ok[j] = idx < n;
            k[j] = 0;
#pragma unroll
            for (int c = 0; c < NV; ++c) v[c][j] = 0;
            if (ok[j]) {
                k[j] = ld_stream_u64(keys + idx, pol);
                if (IN == IN_SOA) {
#pragma unroll
                    for (int c = 0; c < NV; ++c)
                        if (cols.c[c]) v[c][j] = ld_stream_u64(cols.c[c] + idx, pol);
                } else if (IN == IN_ACCS) {
                    v[0][j] = idx;
                } else {
                    v[0][j] = idx;
                    if (idx == n - 1) { ok[j] = (k[j] == 1ull); k[j] = EMPTY_KEY; }   // special slot
                    else if (k[j] == EMPTY_KEY) ok[j] = false;                       // unoccupied
                }
            }
        }
        ma_process_rows<IN, NV, ROWS, CACHE>(t, ctl, sp, cols, k, v, ok, hc_keys, hc_acc, use_cache, my_inserts, my_hits);
        if ((iter & 15u) == 15u && ma_check<CACHE>(ctl, max_inserts, iter, TILE, my_inserts, my_hits, use_cache, &s_inserts, &s_hits, &s_abort))
            return;
    }
    if (CACHE) {
        __syncthreads();
        ma_cache_flush(t, ctl, sp, hc_keys, hc_acc, tid, my_inserts);
    }
    u32 w = __reduce_add_sync(0xffffffffu, my_inserts);
    if ((tid & 31u) == 0 && w) atomicAdd(&s_inserts, w);
    __syncthreads();
    if (tid == 0 && s_inserts) atomicAdd(&ctl->n_inserted, (unsigned long long)s_inserts);
}

// Bulk-staged (copy engine) multi-aggregate combine over SoA keys + NV value columns: the producer warp stages
// the keys and every value column of a tile with cp.async.bulk (MA_STAGES tiles in flight), the 8 consumer warps
// probe and RED, as hash_agg_bulk_kernel.  Dynamic shared memory: [MA_STAGES][keys | col 0 | ... | col NV-1], then
// the hot-key cache.  Full 16-byte aligned tiles only; the sub-tile tail is read with plain loads.
template <int NV>
__global__ void __launch_bounds__(HB_THREADS, 2)
hash_agg_multi_bulk_kernel(const u64 *__restrict__ keys, MaCols cols, u64 n, Table t, AccSpec sp, TableCtl *ctl, u64 max_inserts)
{
    constexpr bool CACHE = true;
    constexpr int ROWS = ma_rows<NV>();
    constexpr int TILE = HA_THREADS * ROWS;
    constexpr u32 STAGE_BYTES = (u32)ma_stage_bytes<NV>();
    extern __shared__ __align__(128) unsigned char ma_stage[];
    __shared__ __align__(8) u64 full_bar[MA_STAGES];
    __shared__ __align__(8) u64 empty_bar[MA_STAGES];
    __shared__ u32 s_inserts, s_abort, s_hits;
    u64 *hc_keys = (u64 *)(ma_stage + (size_t)MA_STAGES * STAGE_BYTES), *hc_acc = hc_keys + MA_HC_SLOTS;
    const u32 tid = threadIdx.x;
    if (tid == 0) {
        s_inserts = 0; s_abort = 0; s_hits = 0;
#pragma unroll
        for (int s = 0; s < MA_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], HA_THREADS / 32); }
        mbar_fence_init();
    }
    if (CACHE) ma_cache_init<HB_THREADS>(hc_keys, hc_acc, sp, tid);
    __syncthreads();
    const u64 n_full = n / TILE;

    if (tid >= HA_THREADS) {                                // ===== producer warp =====
        if (tid == HA_THREADS) {
            const u64 pol = policy_evict_first();
            u32 i = 0;
            for (u64 tile = blockIdx.x; tile < n_full; tile += gridDim.x, ++i) {
                const u32 s = i % MA_STAGES;
                if (i >= MA_STAGES) mbar_wait(&empty_bar[s], ((i / MA_STAGES) & 1u) ^ 1u);
                unsigned char *dst = ma_stage + (size_t)s * STAGE_BYTES;
                u32 bytes = TILE * 8;
#pragma unroll
                for (int c = 0; c < NV; ++c) bytes += cols.c[c] ? TILE * 8 : 0;
                mbar_arrive_expect_tx(&full_bar[s], bytes);
                bulk_g2s(dst, keys + tile * TILE, TILE * 8, &full_bar[s], pol);
#pragma unroll
                for (int c = 0; c < NV; ++c)
                    if (cols.c[c]) bulk_g2s(dst + (size_t)(1 + c) * TILE * 8, cols.c[c] + tile * TILE, TILE * 8, &full_bar[s], pol);
            }
        }
        return;
    }

    // ===== consumer warps =====
    u32 my_inserts = 0, my_hits = 0, iter = 0;
    bool use_cache = CACHE;
    bool drain = false;        // after an abort: keep the pipeline moving (copies in flight target this CTA's smem), skip the work
    for (u64 tile = blockIdx.x; tile < n_full; tile += gridDim.x, ++iter) {
        const u32 s = iter % MA_STAGES;
        mbar_wait(&full_bar[s], (iter / MA_STAGES) & 1u);
        const u64 *src = reinterpret_cast<const u64 *>(ma_stage + (size_t)s * STAGE_BYTES);
        u64 k[ROWS], v[NV][ROWS];
        bool ok[ROWS];
#pragma unroll
        for (int j = 0; j < ROWS; ++j) {
            const u32 r = (u32)j * HA_THREADS + tid;
            ok[j] = !drain;
            k[j] = src[r];
#pragma unroll
            for (int c = 0; c < NV; ++c) v[c][j] = cols.c[c] ? src[(1 + c) * TILE + r] : 0ull;
        }
        fence_proxy_async();        // generic-proxy reads ordered before the slot is refilled by the async proxy
        __syncwarp();
        if ((tid & 31u) == 0) mbar_arrive(&empty_bar[s]);
        if (!drain) ma_process_rows<IN_SOA, NV, ROWS, CACHE>(t, ctl, sp, cols, k, v, ok, hc_keys, hc_acc, use_cache, my_inserts, my_hits);
        if ((iter & 15u) == 15u && ma_check<CACHE>(ctl, max_inserts, iter, TILE, my_inserts, my_hits, use_cache, &s_inserts, &s_hits, &s_abort))
            drain = true;
    }
    if (!drain && (n % TILE) && blockIdx.x == (u32)(n_full % gridDim.x)) {   // tail: plain loads
        const u64 pol = policy_evict_first();
        const u64 base = n_full * TILE;
        u64 k[ROWS], v[NV][ROWS];
        bool ok[ROWS];
#pragma unroll
        for (int j = 0; j < ROWS; ++j) {
            const u64 idx = base + (u64)j * HA_THREADS + tid;
            ok[j] = idx < n;
            k[j] = 0;
#pragma unroll
            for (int c = 0; c < NV; ++c) v[c][j] = 0;
            if (ok[j]) {
                k[j] = ld_stream_u64(keys + idx, pol);
#pragma unroll
                for (int c = 0; c < NV; ++c)
                    if (cols.c[c]) v[c][j] = ld_stream_u64(cols.c[c] + idx, pol);
            }
        }
        ma_process_rows<IN_SOA, NV, ROWS, CACHE>(t, ctl, sp, cols, k, v, ok, hc_keys, hc_acc, use_cache, my_inserts, my_hits);
    }
    if (CACHE) {
        named_bar_sync(1, HA_THREADS);
        if (!drain) ma_cache_flush(t, ctl, sp, hc_keys, hc_acc, tid, my_inserts);
    }
    u32 w = __reduce_add_sync(0xffffffffu, my_inserts);
    if ((tid & 31u) == 0 && w) atomicAdd(&s_inserts, w);
    named_bar_sync(1, HA_THREADS);
    if (tid == 0 && s_inserts) atomicAdd(&ctl->n_inserted, (unsigned long long)s_inserts);
}

// Finalize: output column o of row i (key slot slots[i]) from the table.  kind 0: the accumulator with the inverse
// order transform; MEAN: sum / count as f64, the sum read as u64 (1), i64 (2) or f64 (3).
enum : int { MO_COPY = 0, MO_MEAN_U64 = 1, MO_MEAN_I64 = 2, MO_MEAN_F64 = 3 };
struct OutSpec {
    u32 n;
    unsigned char acc[MA_MAX_ACCS], cnt[MA_MAX_ACCS], kind[MA_MAX_ACCS], tx[MA_MAX_ACCS];
};
__global__ void multi_finalize_kernel(const u64 *__restrict__ accs, u64 stride, const u64 *__restrict__ slots, u64 d, OutSpec os,
                                      u64 *__restrict__ out)
{
    const u64 step = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < d; i += step) {
        const u64 sl = slots[i];
#pragma unroll
        for (int o = 0; o < MA_MAX_ACCS; ++o) {
            if (o >= (int)os.n) break;
            const u64 x = accs[(u64)os.acc[o] * stride + sl];
            u64 r;
            if (os.kind[o] == MO_COPY) {
                r = tx_inv(x, os.tx[o]);
            } else {
                const double cnt = (double)accs[(u64)os.cnt[o] * stride + sl];
                const double sum = os.kind[o] == MO_MEAN_U64 ? (double)x
                                 : os.kind[o] == MO_MEAN_I64 ? (double)(long long)x : __longlong_as_double((long long)x);
                r = (u64)__double_as_longlong(sum / cnt);
            }
            out[(u64)o * d + i] = r;
        }
    }
}

// Strided key sample for the distinct-count estimate that sizes the first table.
template <int IN>
__global__ void sample_keys_kernel(const u64 *__restrict__ a, u64 n, u64 stride, u64 *__restrict__ out, u32 m)
{
    u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    u64 i = (u64)j * stride;
    if (i >= n) i = n - 1;
    out[j] = (IN == IN_AOS) ? a[2 * i] : a[i];
}

// Read-only lookup used by the join: slot index of `key`, or 0xFFFFFFFF.  Slots never go back to EMPTY_KEY, so the
// first bucket with an empty slot ends the key's chain; a chain can run up to half the table (chain_limit).
VB_D u32 table_find(const Table &t, u64 key)
{
    const u64 cap = 1ull << t.log_cap, nb_mask = (cap >> 2) - 1;
    if (key == EMPTY_KEY) return t.keys[cap] == 1ull ? (u32)cap : 0xFFFFFFFFu;
    u64 b = home_bucket(key, t.log_cap);
    for (u64 probe = 0; probe <= nb_mask; ++probe) {
        const Bucket4 bk = ld_bucket(t, b);
        const int hit = bucket_find(bk, key);
        if (hit >= 0) return (u32)(4 * b + hit);
        if (bucket_find(bk, EMPTY_KEY) >= 0) return 0xFFFFFFFFu;
        b = (b + 1) & nb_mask;
    }
    return 0xFFFFFFFFu;
}

// ---------------------------------------------------------------------------------------------
// Radix pass (stable multisplit / one LSD digit)
// ---------------------------------------------------------------------------------------------
#ifndef VB_RP_TILE
#define VB_RP_TILE 4096
#endif
#ifndef VB_RPS_THREADS
#define VB_RPS_THREADS 512
#endif
constexpr int RP_THREADS = 256;
constexpr int RP_WARPS = RP_THREADS / 32;
constexpr int RP_TILE = VB_RP_TILE;              // rows per tile
constexpr int RP_ITEMS = RP_TILE / RP_THREADS;   // histogram kernel: items per thread per tile
constexpr int RP_NB = 256;                       // bins of a pass: 8-bit digits; bin RP_NB = "invalid, drop"
constexpr int RPS_THREADS = VB_RPS_THREADS;      // scatter kernel: 16 warps x 8 items cover the same 4096-row tile with
constexpr int RPS_WARPS = RPS_THREADS / 32;      // <= 64 registers/thread, so 2 CTAs = 32 warps stay resident per SM
constexpr int RPS_ITEMS = RP_TILE / RPS_THREADS; // (256 x 16 needed 128 registers: 16 warps/SM, issue slots 32 % busy)
// Every pass, the LSD sort passes included, uses 8-bit digits: a 10-bit variant of the sort was slower per pass
// (per-tile scan over 1025 bins + 4-row write runs).

enum : int { LD_SOA64 = 0, LD_AOS64 = 1, LD_KEY32_VAL_SOA = 2, LD_KEY32_VAL_AOS = 3, LD_TABLE_KV = 4, LD_TABLE_KI = 5, LD_POS = 6 };

// Where a pass reads its rows from.  One struct, run-time mode (CTA-uniform branch).
struct Loader {
    int mode;
    const void *keys;   // u64* / u32* / rows (AoS) / table keys
    const void *vals;   // u64* (table modes: the accs array) or AoS rows for LD_KEY32_VAL_AOS
    u64 cap;            // table modes: number of regular slots (row `cap` is the special slot)
};

// LD_POS rows (repartition, vb_shuffle_map_repartition): the maps' rows in map-id order, row i of map m at position
// start + 1 + i (mod 2^64).  The loader's key is that position, computed from the row index: no key column exists.
// Loader.keys = RepMap[cap + 1] over the cap maps; entry cap holds the total row count.
struct RepMap {
    u64 row_off;        // the map's first row in the concatenation of the maps
    u64 start;          // first_position of the map
    const u64 *col;     // the one item column, moved as the value; NULL: the value is the row reference ((m + 1) << 32 | i)
};

// the map holding row i (the last m with row_off <= i; empty maps share their successor's offset) and the row in it
VB_D u64 rep_locate(const RepMap *__restrict__ t, u32 n_map, u64 i, u32 &m)
{
    u32 lo = 0, hi = n_map;
    while (hi - lo > 1) {
        const u32 mid = (lo + hi) >> 1;
        if (__ldg(&t[mid].row_off) <= i) lo = mid;
        else hi = mid;
    }
    m = lo;
    return i - __ldg(&t[lo].row_off);
}

// Loader / digit modes are compile-time (LDM, DGM): a run-time switch per item left ptxas with a
// branch per load and no memory-level parallelism.
template <typename KeyT, int LDM>
VB_D bool rp_load(const Loader &ld, u64 i, KeyT &key, u64 &val, u64 pol)
{
    if constexpr (LDM == LD_SOA64) {
        key = (KeyT)ld_stream_u64((const u64 *)ld.keys + i, pol);
        val = ld.vals ? ld_stream_u64((const u64 *)ld.vals + i, pol) : 0ull;
        return true;
    } else if constexpr (LDM == LD_AOS64) {
        ulonglong2 r = ld_stream_u64x2((const u64 *)ld.keys + 2 * i, pol);
        key = (KeyT)r.x; val = r.y;
        return true;
    } else if constexpr (LDM == LD_KEY32_VAL_SOA) {
        key = (KeyT)ld_stream_u32((const u32 *)ld.keys + i, pol);
        val = ld.vals ? ld_stream_u64((const u64 *)ld.vals + i, pol) : 0ull;
        return true;
    } else if constexpr (LDM == LD_KEY32_VAL_AOS) {
        key = (KeyT)ld_stream_u32((const u32 *)ld.keys + i, pol);
        val = ld_stream_u64((const u64 *)ld.vals + 2 * i + 1, pol);
        return true;
    } else if constexpr (LDM == LD_POS) {
        const RepMap *t = (const RepMap *)ld.keys;
        u32 m;
        const u64 r = rep_locate(t, (u32)ld.cap, i, m);
        key = (KeyT)(__ldg(&t[m].start) + 1 + r);
        const u64 *col = (const u64 *)__ldg((const unsigned long long *)&t[m].col);
        val = col ? ld_stream_u64(col + r, pol) : ((u64)(m + 1) << 32 | r);
        return true;
    } else {
        const u64 k = ld_stream_u64((const u64 *)ld.keys + i, pol);
        val = (LDM == LD_TABLE_KI) ? i : ld_stream_u64((const u64 *)ld.vals + i, pol);
        if (i == ld.cap) { key = (KeyT)EMPTY_KEY; return k == 1ull; }
        key = (KeyT)k;
        return k != EMPTY_KEY;
    }
}

// key only (histogram pass)
template <typename KeyT, int LDM>
VB_D bool rp_load_key(const Loader &ld, u64 i, KeyT &key, u64 pol)
{
    if constexpr (LDM == LD_SOA64) { key = (KeyT)ld_stream_u64((const u64 *)ld.keys + i, pol); return true; }
    else if constexpr (LDM == LD_AOS64) { key = (KeyT)ld_stream_u64((const u64 *)ld.keys + 2 * i, pol); return true; }
    else if constexpr (LDM == LD_KEY32_VAL_SOA || LDM == LD_KEY32_VAL_AOS) { key = (KeyT)ld_stream_u32((const u32 *)ld.keys + i, pol); return true; }
    else if constexpr (LDM == LD_POS) {
        const RepMap *t = (const RepMap *)ld.keys;
        u32 m;
        const u64 r = rep_locate(t, (u32)ld.cap, i, m);
        key = (KeyT)(__ldg(&t[m].start) + 1 + r);
        return true;
    }
    else {
        const u64 k = ld_stream_u64((const u64 *)ld.keys + i, pol);
        if (i == ld.cap) { key = (KeyT)EMPTY_KEY; return k == 1ull; }
        key = (KeyT)k;
        return k != EMPTY_KEY;
    }
}

enum : int { DG_BITS = 0, DG_BUCKET = 1, DG_DEST = 2, DG_HASHTOP = 3 };

// Which bin a key goes to.  DG_BITS: radix digit of the (order-transformed) key.  DG_BUCKET:
// digit of HashPartitioner::get_partition(key).  DG_DEST: owning rank = partition % world.
// DG_HASHTOP: top bits of slot_hash(key) — pre-partitions rows so a table larger than L2 is visited region by region.
struct Digit {
    int mode;
    u32 shift, mask;
    int tx;
    u32 key_width;
    FastMod fm;        // % n_reduce
    FastMod fm_world;  // % world
};

template <typename KeyT, int DGM>
VB_D u32 rp_digit(const Digit &dg, KeyT key)
{
    if constexpr (DGM == DG_BITS) {
        u64 k = (sizeof(KeyT) == 8) ? tx_fwd((u64)key, dg.tx) : (u64)key;
        return (u32)(k >> dg.shift) & dg.mask;
    } else if constexpr (DGM == DG_HASHTOP) {
        // top bits of the table's slot hash: rows of one digit probe one contiguous region of the table
        return (u32)(slot_hash((u64)key) >> dg.shift) & dg.mask;
    } else {
        u32 b = get_partition((u64)key, dg.key_width, dg.fm);
        if constexpr (DGM == DG_DEST) return fastmod(b, dg.fm_world);
        return (b >> dg.shift) & dg.mask;
    }
}

// Lanes of the warp whose 9-bit digit (8 digit bits + the "invalid" bit RP_NB) equals mine.  Built from 9 ballots
// instead of MATCH.ANY: the hardware match iterates over the distinct values in the warp (~30 for random
// digits) and dominated both radix kernels (short_scoreboard stalls).
VB_D u32 warp_match_digit(u32 d)
{
    u32 peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b <= 8; ++b) {
        const bool bit = (d >> b) & 1u;
        const u32 m = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? m : ~m;
    }
    return peers;
}

// part p covers rows [p*rows_per_part, min(n, (p+1)*rows_per_part)); hist[d*num_parts + p].
// Each part is histogrammed by `split` CTAs (blockIdx.x = part*split + sub) that add their counts
// with global atomics, so the grid fills the machine even though there are only ~2 parts per SM.
// hist must be zeroed before the launch.
// Counting needs no ranking, so instead of a ballot match per item (78 instructions per item,
// math_pipe_throttle) every LANE keeps private byte counters
// pc[warp][digit][lane] in shared memory: an item is one LDS.U8 / IADD / STS.U8, no atomics, no votes.
// A thread adds at most RP_ITEMS per tile, so the bytes are folded into the CTA's u32 histogram
// every 255 / RP_ITEMS tiles (15 * 16 = 240 <= 255).
constexpr size_t rp_hist_smem() { return (size_t)RP_WARPS * RP_NB * 32; }

template <typename KeyT, int LDM, int DGM>
__global__ void __launch_bounds__(RP_THREADS)
rp_hist_kernel(Loader ld, Digit dg, u64 n, u64 rows_per_part, u32 *__restrict__ hist, u32 num_parts, u32 split)
{
    constexpr int NB = RP_NB;
    extern __shared__ __align__(16) unsigned char pc_raw[];        // [RP_WARPS][NB][32] byte counters
    __shared__ u32 cta_hist[NB];
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
    unsigned char *pc = pc_raw + (size_t)warp * NB * 32;
    u32 *pcw = (u32 *)pc;
    for (u32 i = lane; i < NB * 8; i += 32) pcw[i] = 0;
    for (u32 d = tid; d < NB; d += RP_THREADS) cta_hist[d] = 0;
    __syncthreads();
    const u64 pol = policy_evict_first();
    const u32 part = blockIdx.x / split, sub = blockIdx.x % split;
    const u64 begin = (u64)part * rows_per_part;
    const u64 end = min(n, begin + rows_per_part);
    auto fold = [&]() {      // warp-local: sum the 32 lane counters of each digit into cta_hist, clear them
        __syncwarp();
        for (u32 b = lane; b < NB; b += 32) {
            u32 s = 0;
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                const u32 x = pcw[b * 8 + w];
                pcw[b * 8 + w] = 0;
                s += (x & 0xFF) + ((x >> 8) & 0xFF) + ((x >> 16) & 0xFF) + (x >> 24);
            }
            if (s) atomicAdd(&cta_hist[b], s);
        }
        __syncwarp();
    };
    constexpr int HB = 8;   // items per batch: keeps the u64 instantiation at <= 64 registers
    u32 tiles_since_fold = 0;
    constexpr bool STREAM = (LDM == LD_SOA64 || LDM == LD_AOS64 || LDM == LD_KEY32_VAL_SOA || LDM == LD_KEY32_VAL_AOS || LDM == LD_POS);   // every row valid
    for (u64 t0 = begin + (u64)sub * RP_TILE; t0 < end; t0 += (u64)split * RP_TILE) {
        if (STREAM && t0 + RP_TILE <= end) {      // whole tile in range: no bounds checks, no branch around the counter update
#pragma unroll 1
            for (int h = 0; h < RP_ITEMS; h += HB) {
                KeyT key[HB];
#pragma unroll
                for (int i = 0; i < HB; ++i) {
                    const u64 idx = t0 + (u64)warp * (32 * RP_ITEMS) + (u64)(h + i) * 32 + lane;
                    rp_load_key<KeyT, LDM>(ld, idx, key[i], pol);
                }
#pragma unroll
                for (int i = 0; i < HB; ++i) pc[rp_digit<KeyT, DGM>(dg, key[i]) * 32 + lane] += 1;
            }
            if (++tiles_since_fold == 255 / RP_ITEMS) { fold(); tiles_since_fold = 0; }
            continue;
        }
#pragma unroll 1
        for (int h = 0; h < RP_ITEMS; h += HB) {
            KeyT key[HB];
            bool ok[HB];
#pragma unroll
            for (int i = 0; i < HB; ++i) {
                const u64 idx = t0 + (u64)warp * (32 * RP_ITEMS) + (u64)(h + i) * 32 + lane;
                key[i] = 0;
                ok[i] = (idx < end) && rp_load_key<KeyT, LDM>(ld, idx, key[i], pol);
            }
#pragma unroll
            for (int i = 0; i < HB; ++i) {
                if (ok[i]) {
                    const u32 d = rp_digit<KeyT, DGM>(dg, key[i]);
                    pc[d * 32 + lane] += 1;      // private to this lane: plain read-modify-write
                }
            }
        }
        if (++tiles_since_fold == 255 / RP_ITEMS) { fold(); tiles_since_fold = 0; }
    }
    fold();
    __syncthreads();
    for (u32 d = tid; d < NB; d += RP_THREADS) {
        const u32 s = cta_hist[d];
        if (s) atomicAdd(&hist[(u64)d * num_parts + part], s);
    }
}

// Exclusive scan of hist[0 .. len) in place (single CTA); total written to hist[len].
__global__ void __launch_bounds__(1024) rp_scan_kernel(u32 *hist, u32 len)
{
    __shared__ u32 warp_sums[32];
    __shared__ u32 s_total;
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const u32 per = (len + 1023u) / 1024u;
    const u32 lo = min(len, tid * per), hi = min(len, lo + per);
    u32 s = 0;
    for (u32 i = lo; i < hi; ++i) s += hist[i];
    u32 incl = s;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= (u32)off) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        u32 ws = warp_sums[lane];
        u32 wi = ws;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            u32 t = __shfl_up_sync(0xffffffffu, wi, off);
            if (lane >= (u32)off) wi += t;
        }
        warp_sums[lane] = wi - ws;
        if (lane == 31) s_total = wi;
    }
    __syncthreads();
    u32 run = warp_sums[warp] + (incl - s);
    for (u32 i = lo; i < hi; ++i) {
        u32 c = hist[i];
        hist[i] = run;
        run += c;
    }
    if (tid == 0) hist[len] = s_total;
}

// One stable scatter pass.  Per 4096-row tile: rank every row inside its warp by digit (ballots), scan
// the warp counts across the CTA, stage the tile in shared memory in output order together with each
// row's GLOBAL output index, then write it out with consecutive threads touching consecutive staged
// rows (runs of ~16 rows per digit → coalesced 64-128 B segments).  5 barriers per tile; the counters
// for the next tile are cleared and its loads are in flight while the current tile is written out.
// Destination tables of a REMOTE scatter: digit d (= destination rank) is written to the peer's
// receive arena mapped into this process (CUDA IPC over NVLink), at row adj[d] + flat_index.
struct RemoteDst {
    u64 *const *keys;   // [world] device array of peer key bases
    u64 *const *vals;   // [world]
    const u32 *adj;     // [world] (my row offset inside the peer's arena) - (start of digit d in the flat order)
    u32 world;
};

// REMOTE = the shuffle's exchange fused into the partition pass: instead of packing rows by
// destination rank locally and handing the buffers to an all-to-all, the staged runs are stored straight
// into the destination GPUs' HBM (st.global on peer-mapped addresses), so the NVLink transfer overlaps
// ranking/staging of the following tiles.
template <typename KeyT, bool HAS_VAL, int LDM, int DGM, bool REMOTE = false>
__global__ void __launch_bounds__(RPS_THREADS, (RPS_THREADS > 512 ? 1 : RPS_THREADS > 256 ? 2 : 4))
rp_scatter_kernel(Loader ld, Digit dg, u64 n, u64 rows_per_part, const u32 *__restrict__ part_off, u32 num_parts,
                  KeyT *__restrict__ out_keys, u64 *__restrict__ out_vals, RemoteDst rd)
{
    constexpr int NB = RP_NB;
    static_assert(NB <= RPS_THREADS, "one thread per digit in the tile scan");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64 *stage_vals = (u64 *)smem_raw;                                       // [RP_TILE] if HAS_VAL
    KeyT *stage_keys = (KeyT *)(smem_raw + (HAS_VAL ? RP_TILE * 8 : 0));     // [RP_TILE]
    // the widest rows (u64 key + u64 value) stage the 1-byte digit and look the offset up at write-out
    // instead of staging a 4-byte output index: faster for them, slightly slower for the others (A/B)
    constexpr bool STAGE_IDX = !(sizeof(KeyT) == 8 && HAS_VAL);
    u32 *stage_out = (u32 *)(stage_keys + RP_TILE);                          // [RP_TILE] global output index (STAGE_IDX)
    unsigned char *stage_dig = (unsigned char *)(stage_keys + RP_TILE);      // [RP_TILE] digit (!STAGE_IDX)
    __shared__ u32 cnt[RPS_WARPS][NB + 1];   // per warp: count, then exclusive prefix over warps
    __shared__ u32 dbase[NB + 1];            // tile-local start of digit d; dbase[NB] = #valid rows of the tile
    __shared__ u32 gbase[NB + 1];            // run_off[d] - dbase[d]: staged position p of digit d goes to gbase[d] + p
    __shared__ u32 run_off[NB];              // global output offset of the next row of digit d for this part
    __shared__ u32 wtot[RPS_WARPS];
    __shared__ u64 *s_dk[REMOTE ? NB : 1];
    __shared__ u64 *s_dv[REMOTE ? NB : 1];
    __shared__ u32 s_adj[REMOTE ? NB : 1];
    static_assert(!REMOTE || (sizeof(KeyT) == 8 && HAS_VAL), "remote scatter moves (u64 key, u64 value) rows");
    if (REMOTE)
        for (u32 d = threadIdx.x; d < rd.world && d < (u32)NB; d += RPS_THREADS) { s_dk[d] = rd.keys[d]; s_dv[d] = rd.vals[d]; s_adj[d] = rd.adj[d]; }

    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
    const u32 lt = lanemask_lt();
    const u64 pol = policy_evict_first();
    const u32 part = blockIdx.x;
    const u64 begin = (u64)part * rows_per_part;
    const u64 end = min(n, begin + rows_per_part);
    for (u32 d = tid; d < NB; d += RPS_THREADS) run_off[d] = part_off[(u64)d * num_parts + part];
    for (u32 d = tid; d < RPS_WARPS * (NB + 1); d += RPS_THREADS) (&cnt[0][0])[d] = 0;

    KeyT key[RPS_ITEMS];
    u64 val[RPS_ITEMS];
    bool ok[RPS_ITEMS];
    auto load_tile = [&](u64 t0) {
#pragma unroll
        for (int i = 0; i < RPS_ITEMS; ++i) {   // every load of the tile is issued before any is used
            const u64 idx = t0 + (u64)warp * (32 * RPS_ITEMS) + (u64)i * 32 + lane;
            key[i] = 0; val[i] = 0;
            ok[i] = (idx < end) && rp_load<KeyT, LDM>(ld, idx, key[i], val[i], pol);
        }
    };
    // (u64 key + u64 value needs 32 registers for the tile alone: prefetching spilled under the 64-register cap)
    constexpr bool PREFETCH = !(sizeof(KeyT) == 8 && HAS_VAL);
    if (PREFETCH && begin < end) load_tile(begin);
    __syncthreads();

    for (u64 t0 = begin; t0 < end; t0 += RP_TILE) {
        if (!PREFETCH) load_tile(t0);
        unsigned short dig[RPS_ITEMS], rank[RPS_ITEMS];
#pragma unroll
        for (int i = 0; i < RPS_ITEMS; ++i) dig[i] = (unsigned short)(ok[i] ? rp_digit<KeyT, DGM>(dg, key[i]) : (u32)NB);
#pragma unroll
        for (int i = 0; i < RPS_ITEMS; ++i) {
            const u32 d = dig[i];
            const u32 peers = warp_match_digit(d);
            const u32 leader = (u32)(__ffs(peers) - 1);
            u32 base = 0;
            if (lane == leader) { base = cnt[warp][d]; cnt[warp][d] = base + __popc(peers); }   // only the group leader touches smem
            base = __shfl_sync(0xffffffffu, base, leader);
            rank[i] = (unsigned short)(base + __popc(peers & lt));
            __syncwarp();                                                       // orders this round's store before the next round's load
        }
        __syncthreads();                                                        // B1: warp counts complete
        // thread d < NB: exclusive scan of digit d over the warps, then a block-wide exclusive scan over the digits;
        // the "invalid" bin NB sits after all valid rows and is handled by one extra thread below
        u32 total = 0;
        if (tid < NB) {
#pragma unroll
            for (int w = 0; w < RPS_WARPS; ++w) { const u32 c = cnt[w][tid]; cnt[w][tid] = total; total += c; }
        }
        u32 incl = total;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const u32 t = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= (u32)off) incl += t;
        }
        if (lane == 31) wtot[warp] = incl;
        __syncthreads();                                                        // B2: warp totals visible
        if (tid < NB) {
            u32 excl = incl - total;
            for (u32 w = 0; w < warp; ++w) excl += wtot[w];
            dbase[tid] = excl;
#pragma unroll
            for (int w = 0; w < RPS_WARPS; ++w) cnt[w][tid] += excl;            // cnt[w][d] = tile position of warp w's first row of digit d
            const u32 ro = run_off[tid];
            gbase[tid] = ro - excl;
            run_off[tid] = ro + total;
            if (tid == NB - 1) {                                                // rows of the invalid bin follow the valid ones
                u32 nv = excl + total;
                dbase[NB] = nv;
                for (int w = 0; w < RPS_WARPS; ++w) { const u32 c = cnt[w][NB]; cnt[w][NB] = nv; nv += c; }
            }
        }
        __syncthreads();                                                        // B3: positions / gbase visible
#pragma unroll
        for (int i = 0; i < RPS_ITEMS; ++i) {
            const u32 d = dig[i];
            const u32 pos = cnt[warp][d] + rank[i];
            stage_keys[pos] = key[i];
            if (HAS_VAL) stage_vals[pos] = val[i];
            if (d < NB) {                                   // rows with d == NB (invalid) sit past n_valid
                if (STAGE_IDX) stage_out[pos] = gbase[d] + pos;
                else stage_dig[pos] = (unsigned char)d;
            }
        }
        if (PREFETCH && t0 + RP_TILE < end) load_tile(t0 + RP_TILE);             // in flight during the write-out below
        __syncthreads();                                                        // B4: tile staged, cnt free
        for (u32 d = tid; d < RPS_WARPS * (NB + 1); d += RPS_THREADS) (&cnt[0][0])[d] = 0;
        const u32 n_valid = dbase[NB];
        for (u32 p = tid; p < n_valid; p += RPS_THREADS) {
            if (REMOTE) {
                const u32 d = stage_dig[p];
                const u32 o = gbase[d] + p + s_adj[d];
                s_dk[d][o] = (u64)stage_keys[p];
                s_dv[d][o] = stage_vals[p];
            } else {
                // (writing the same bytes to sequential destinations instead is only 0-5 % faster: the
                //  scattered DRAM writes are not what bounds this kernel — barriers and latency are)
                const u32 o = STAGE_IDX ? stage_out[p] : gbase[stage_dig[p]] + p;
                out_keys[o] = stage_keys[p];
                if (HAS_VAL) out_vals[o] = stage_vals[p];
            }
        }
        __syncthreads();                                                        // B5: staging buffers and cnt reusable
    }
}

template <typename KeyT, bool HAS_VAL>
constexpr size_t rp_scatter_smem() { return (size_t)RP_TILE * ((HAS_VAL ? 8 : 0) + sizeof(KeyT) + ((sizeof(KeyT) == 8 && HAS_VAL) ? 1 : 4)); }

// ---------------------------------------------------------------------------------------------
// Unordered multisplit of the occupied slots of a combined table (reduce ops): (key, combiner) rows by reduce
// partition or by owner rank.  The reference's order inside a reduce partition is HashMap order (unspecified), so
// no stability is needed here: two small kernels (count, scatter with one global cursor claim per tile and bin)
// replace the histogram + single-CTA scan + stable scatter of the general pass, whose fixed cost (~150 us) is
// most of a step's seal/exchange time once the map-side combine has shrunk 1e9 rows to 1e6.
// ---------------------------------------------------------------------------------------------
constexpr int TS_THREADS = 256, TS_ITEMS = 8, TS_TILE = TS_THREADS * TS_ITEMS, TS_MAX_BINS = 256;

template <int DGM>
VB_D bool ts_load(const u64 *__restrict__ keys, u64 cap, u64 i, const Digit &dg, u64 &key, u32 &bin)
{
    if (i > cap) return false;
    const u64 k = keys[i];
    if (i == cap) { if (k != 1ull) return false; key = EMPTY_KEY; }      // special slot: a real key equal to the empty marker
    else { if (k == EMPTY_KEY) return false; key = k; }
    bin = rp_digit<u64, DGM>(dg, key);
    return true;
}

template <int DGM>
__global__ void __launch_bounds__(TS_THREADS) table_bin_count_kernel(const u64 *__restrict__ keys, u64 cap, Digit dg, u32 *__restrict__ counts)
{
    __shared__ u32 h[TS_MAX_BINS];
    for (u32 d = threadIdx.x; d < TS_MAX_BINS; d += TS_THREADS) h[d] = 0;
    __syncthreads();
    const u64 stride = (u64)gridDim.x * TS_THREADS;
    for (u64 i = (u64)blockIdx.x * TS_THREADS + threadIdx.x; i <= cap; i += stride) {
        u64 key; u32 bin;
        if (ts_load<DGM>(keys, cap, i, dg, key, bin)) atomicAdd(&h[bin], 1u);
    }
    __syncthreads();
    for (u32 d = threadIdx.x; d < TS_MAX_BINS; d += TS_THREADS) if (h[d]) atomicAdd(&counts[d], h[d]);
}

template <int DGM>
__global__ void __launch_bounds__(TS_THREADS)
table_bin_scatter_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ accs, u64 cap, Digit dg, const u32 *__restrict__ counts,
                         u32 *__restrict__ cursors, u64 *__restrict__ out_keys, u64 *__restrict__ out_vals)
{
    __shared__ u32 base[TS_MAX_BINS], tile_cnt[TS_MAX_BINS], tile_base[TS_MAX_BINS], ws[TS_THREADS / 32];
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    {   // exclusive scan of the global counts (every CTA redoes these 256 adds instead of a separate scan kernel)
        const u32 c = counts[tid];
        u32 incl = c;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const u32 t = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= (u32)off) incl += t; }
        if (lane == 31) ws[warp] = incl;
        __syncthreads();
        u32 b = 0;
        for (u32 w = 0; w < warp; ++w) b += ws[w];
        base[tid] = b + incl - c;
        tile_cnt[tid] = 0;
    }
    __syncthreads();
    const u64 n_tiles = (cap + 1 + TS_TILE - 1) / TS_TILE;
    for (u64 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        u64 key[TS_ITEMS], val[TS_ITEMS];
        u32 br[TS_ITEMS];                         // bin | local rank << 8 ; 0xFFFFFFFF = no row
#pragma unroll
        for (int j = 0; j < TS_ITEMS; ++j) {
            const u64 i = tile * TS_TILE + (u64)j * TS_THREADS + tid;
            u32 bin;
            br[j] = 0xFFFFFFFFu;
            if (ts_load<DGM>(keys, cap, i, dg, key[j], bin)) {
                val[j] = accs[i];
                br[j] = bin | (atomicAdd(&tile_cnt[bin], 1u) << 8);
            }
        }
        __syncthreads();
        { const u32 c = tile_cnt[tid]; if (c) tile_base[tid] = base[tid] + atomicAdd(&cursors[tid], c); }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < TS_ITEMS; ++j) {
            if (br[j] == 0xFFFFFFFFu) continue;
            const u32 o = tile_base[br[j] & 0xFFu] + (br[j] >> 8);
            out_keys[o] = key[j];
            out_vals[o] = val[j];
        }
        tile_cnt[tid] = 0;
        __syncthreads();
    }
}

// The same split of a multi-aggregate table by owner rank (combine_by_key export): the key and every accumulator
// column, destination-major.  Accumulator a of output row o goes to out_accs[a * total + o] in plain value form
// (tx_inv with its own order transform; total = the exported rows, from table_bin_count_kernel's counts); stride is
// the distance between the table's accumulator columns.
__global__ void __launch_bounds__(TS_THREADS)
table_bin_scatter_multi_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ accs, u64 stride, u64 cap, Digit dg, AccSpec sp,
                               const u32 *__restrict__ counts, u32 *__restrict__ cursors, u64 total, u64 *__restrict__ out_keys,
                               u64 *__restrict__ out_accs)
{
    __shared__ u32 base[TS_MAX_BINS], tile_cnt[TS_MAX_BINS], tile_base[TS_MAX_BINS], ws[TS_THREADS / 32];
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    {
        const u32 c = counts[tid];
        u32 incl = c;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const u32 t = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= (u32)off) incl += t; }
        if (lane == 31) ws[warp] = incl;
        __syncthreads();
        u32 b = 0;
        for (u32 w = 0; w < warp; ++w) b += ws[w];
        base[tid] = b + incl - c;
        tile_cnt[tid] = 0;
    }
    __syncthreads();
    const u64 n_tiles = (cap + 1 + TS_TILE - 1) / TS_TILE;
    for (u64 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        u64 key[TS_ITEMS], slot[TS_ITEMS];
        u32 br[TS_ITEMS];
#pragma unroll
        for (int j = 0; j < TS_ITEMS; ++j) {
            const u64 i = tile * TS_TILE + (u64)j * TS_THREADS + tid;
            u32 bin;
            br[j] = 0xFFFFFFFFu;
            if (ts_load<DG_DEST>(keys, cap, i, dg, key[j], bin)) {
                slot[j] = i;
                br[j] = bin | (atomicAdd(&tile_cnt[bin], 1u) << 8);
            }
        }
        __syncthreads();
        { const u32 c = tile_cnt[tid]; if (c) tile_base[tid] = base[tid] + atomicAdd(&cursors[tid], c); }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < TS_ITEMS; ++j) {
            if (br[j] == 0xFFFFFFFFu) continue;
            const u64 o = tile_base[br[j] & 0xFFu] + (br[j] >> 8);
            out_keys[o] = key[j];
#pragma unroll 1
            for (int a = 0; a < (int)sp.n; ++a) out_accs[(u64)a * total + o] = tx_inv(accs[(u64)a * stride + slot[j]], spec_at(sp.tx, a));
        }
        tile_cnt[tid] = 0;
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// Generic multi-block exclusive scan (u64), chunk = 4096 elements per CTA
// ---------------------------------------------------------------------------------------------
constexpr int SC_THREADS = 256;
constexpr int SC_ITEMS = 16;
constexpr int SC_CHUNK = SC_THREADS * SC_ITEMS;

VB_D u64 block_exclusive_scan_u64(u64 v, u64 *total, u64 *warp_sums /*[8]*/)
{
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    u64 incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        u64 t = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= (u32)off) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    u64 wbase = 0, tsum = 0;
#pragma unroll
    for (int w = 0; w < SC_THREADS / 32; ++w) {
        u64 x = warp_sums[w];
        if ((u32)w < warp) wbase += x;
        tsum += x;
    }
    *total = tsum;
    __syncthreads();
    return wbase + incl - v;
}

__global__ void __launch_bounds__(SC_THREADS) scan_reduce_kernel(const u64 *__restrict__ in, u64 n, u64 *__restrict__ sums)
{
    __shared__ u64 ws[SC_THREADS / 32];
    const u64 base = (u64)blockIdx.x * SC_CHUNK;
    u64 s = 0;
    for (int i = 0; i < SC_ITEMS; ++i) {
        u64 idx = base + (u64)i * SC_THREADS + threadIdx.x;
        if (idx < n) s += in[idx];
    }
    u64 tot;
    block_exclusive_scan_u64(s, &tot, ws);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

// out[i] = offsets[block] + exclusive prefix within the chunk.  offsets may be NULL (single chunk).
// If total_out != NULL the last block writes the grand total there.
__global__ void __launch_bounds__(SC_THREADS)
scan_apply_kernel(const u64 *__restrict__ in, u64 *__restrict__ out, u64 n, const u64 *__restrict__ offsets, u64 *total_out)
{
    __shared__ u64 ws[SC_THREADS / 32];
    const u64 base = (u64)blockIdx.x * SC_CHUNK + (u64)threadIdx.x * SC_ITEMS;
    u64 v[SC_ITEMS];
    u64 s = 0;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        v[i] = (base + i < n) ? in[base + i] : 0ull;
        s += v[i];
    }
    u64 tot;
    u64 run = block_exclusive_scan_u64(s, &tot, ws) + (offsets ? offsets[blockIdx.x] : 0ull);
    const u64 carry_in = offsets ? offsets[blockIdx.x] : 0ull;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        if (base + i < n) out[base + i] = run;
        run += v[i];
    }
    if (total_out && blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *total_out = carry_in + tot;
}

// ---------------------------------------------------------------------------------------------
// group_by_key helpers
// ---------------------------------------------------------------------------------------------
// dense_of_slot[cslot[j]] = j   (cslot holds slot indices as u64 payloads of the bucket multisplit)
__global__ void scatter_dense_kernel(const u64 *__restrict__ cslot, u32 n, u32 *__restrict__ dense_of_slot)
{
    u32 j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) dense_of_slot[cslot[j]] = j;
}

// ids[i] = dense_of_slot[ids[i]] in place (dense_of_slot, 4 B per table slot, is read through L2)
__global__ void translate_ids_kernel(u32 *__restrict__ ids, u64 n, const u32 *__restrict__ dense_of_slot)
{
    // One look-up per thread and iteration, 2048 threads per SM: close to the floor of one L2 request per id.  Tried and slower:
    // fusing the look-up into the first sort pass's histogram kernel (24 warps per SM cannot cover two dependent L2 round trips
    // per batch), and four ids per thread with evict-first look-ups (the hint ages the table out of L2).
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) ids[i] = dense_of_slot[ids[i]];
}

// Key dictionary of n keys known to be distinct (a reduce result taken as a cogroup side), one thread per key: insert key i
// into the table (keys[] pre-set to EMPTY_KEY, keys[cap..cap+4) to 0), dense_of_slot[its slot] = i, and offs[i] = i (one
// value per key), offs[n] = n.  A key equal to EMPTY_KEY takes the special slot cap.  A probe chain longer than
// t.max_probe probe rounds raises ctl->abort and the host rebuilds the table larger.
__global__ void narrow_dict_kernel(const u64 *__restrict__ keys, u64 n, Table t, u32 *__restrict__ dense_of_slot,
                                   u64 *__restrict__ offs, TableCtl *ctl)
{
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    offs[i] = i;
    if (i == n) return;
    const u64 key = keys[i];
    const u64 cap = 1ull << t.log_cap;
    if (key == EMPTY_KEY) {
        t.keys[cap] = 1ull;
        dense_of_slot[cap] = (u32)i;
        return;
    }
    const u64 b = home_bucket(key, t.log_cap);
    u32 inserted = 0;
    if (!table_resolve_with(t, b, ld_bucket(t, b), key, inserted, [&](u64 slot) { dense_of_slot[slot] = (u32)i; }))
        atomicExch(&ctl->abort, 1u);
}

// CSR offsets from sorted dense ids: offsets[id] = first row of id; offsets[n_ids] = n.
__global__ void csr_bounds_kernel(const u32 *__restrict__ ids, u64 n, u64 *__restrict__ offsets, u64 n_ids)
{
    // four ids per thread (one 128-bit load + the id just before them): 2.5x fewer load instructions than one id per thread
    const u64 n4 = n / 4;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) offsets[n_ids] = n;
    for (u64 j = t; j < n4; j += stride) {
        const uint4 v = reinterpret_cast<const uint4 *>(ids)[j];
        const u64 i = 4 * j;
        const u32 prev = j ? ids[i - 1] : ~v.x;          // j == 0: anything different from v.x
        if (prev != v.x) offsets[v.x] = i;
        if (v.x != v.y) offsets[v.y] = i + 1;
        if (v.y != v.z) offsets[v.z] = i + 2;
        if (v.z != v.w) offsets[v.w] = i + 3;
    }
    for (u64 i = 4 * n4 + t; i < n; i += stride) {       // the last n % 4 ids
        const u32 id = ids[i];
        if (i == 0 || ids[i - 1] != id) offsets[id] = i;
    }
}

// out[i] = tx_inv(in[i])
__global__ void tx_inv_kernel(u64 *__restrict__ v, u64 n, int tx)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = tx_inv(v[i], tx);
}

// de-interleave AoS rows into SoA (gather of map partitions that are not contiguous)
__global__ void aos_to_soa_kernel(const u64 *__restrict__ rows, u64 n, u64 *__restrict__ keys, u64 *__restrict__ vals)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 pol = policy_evict_first();
    for (; i < n; i += stride) {
        ulonglong2 r = ld_stream_u64x2(rows + 2 * i, pol);
        keys[i] = r.x;
        vals[i] = r.y;
    }
}

// ---------------------------------------------------------------------------------------------
// join (CoGroupedRdd::compute + cross product)
// ---------------------------------------------------------------------------------------------
// Join kinds: the inner join (the N-way join below; here only the kind of a filtered pair), and the outer joins with the
// values of vb_join_kind (include/vega_b200.h).
enum : int { JK_INNER = 0, JK_LEFT = 1, JK_RIGHT = 2, JK_FULL = 3 };
template <int KIND> constexpr bool jk_keeps_left() { return KIND == JK_LEFT || KIND == JK_FULL; }

// Outer join, left keys [lb, le): find the key in the right shuffle's dictionary; cnt = lenL * lenR.  An unmatched key
// counts lenL rows (k, v, None) when the kind keeps the left side.  rtab.keys is NULL when the right side has no rows.
template <int KIND>
__global__ void join_probe_kernel(const u64 *__restrict__ lkeys, const u64 *__restrict__ loffs, u32 lb, u32 le,
                                  Table rtab, const u32 *__restrict__ r_dense,
                                  const u64 *__restrict__ roffs, u64 *__restrict__ cnt, u32 *__restrict__ match)
{
    u32 j = lb + blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= le) return;
    u64 key = lkeys[j];
    u32 s = rtab.keys ? table_find(rtab, key) : 0xFFFFFFFFu;
    u64 c = 0;
    u32 m = 0xFFFFFFFFu;
    if (s != 0xFFFFFFFFu) {
        m = r_dense[s];
        c = (loffs[j + 1] - loffs[j]) * (roffs[m + 1] - roffs[m]);
    } else if (jk_keeps_left<KIND>()) {
        c = loffs[j + 1] - loffs[j];
    }
    cnt[j - lb] = c;
    match[j - lb] = m;
}

// For right keys [rb, re) of a RIGHT / FULL join: cnt = lenR for a key the left side lacks (rows (k, None, w)), else 0
// (its rows come from the left-driven part).  ltab.keys is NULL when the left side has no rows.
__global__ void join_probe_right_kernel(const u64 *__restrict__ rkeys, const u64 *__restrict__ roffs, u32 rb, u32 re,
                                        Table ltab, u64 *__restrict__ cnt)
{
    const u32 j = rb + blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= re) return;
    const bool in_left = ltab.keys && table_find(ltab, rkeys[j]) != 0xFFFFFFFFu;
    cnt[j - rb] = in_left ? 0 : roffs[j + 1] - roffs[j];
}

// Outer join, one thread per output row: binary-search the owning left key, then (v, w) = divmod.  LEFT / FULL also
// write the rows of unmatched left keys as (k, v, 0); every kind writes the validity bytes when out_vv / out_wv are given.
template <int KIND>
__global__ void join_expand_kernel(const u64 *__restrict__ pos /*[nl] exclusive*/, u32 nl, u64 total,
                                   const u64 *__restrict__ lkeys, const u64 *__restrict__ loffs, const u64 *__restrict__ lvals,
                                   u32 lb, const u32 *__restrict__ match, const u64 *__restrict__ roffs,
                                   const u64 *__restrict__ rvals, u64 *__restrict__ out_k, u64 *__restrict__ out_v,
                                   u64 *__restrict__ out_w, unsigned char *__restrict__ out_vv, unsigned char *__restrict__ out_wv)
{
    u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (; o < total; o += stride) {
        u32 lo = 0, hi = nl;   // largest j with pos[j] <= o  (keys with cnt 0 share pos with the next)
        while (hi - lo > 1) {
            u32 mid = (lo + hi) >> 1;
            if (pos[mid] <= o) lo = mid; else hi = mid;
        }
        const u32 j = lo;
        const u32 m = match[j];
        const u64 local = o - pos[j];
        if (jk_keeps_left<KIND>() && m == 0xFFFFFFFFu) {
            out_k[o] = lkeys[lb + j];
            out_v[o] = lvals[loffs[lb + j] + local];
            out_w[o] = 0;
            if (out_vv) out_vv[o] = 1;
            if (out_wv) out_wv[o] = 0;
            continue;
        }
        const u64 lenr = roffs[m + 1] - roffs[m];
        const u64 vi = local / lenr, wi = local - vi * lenr;
        out_k[o] = lkeys[lb + j];
        out_v[o] = lvals[loffs[lb + j] + vi];
        out_w[o] = rvals[roffs[m] + wi];
        if (out_vv) out_vv[o] = 1;
        if (out_wv) out_wv[o] = 1;
    }
}

// Rows [pos[0], total) of a RIGHT / FULL join: the right-only keys, (k, 0, w) with validity (0, 1).  pos[nr] holds the
// exclusive positions of the partition's right keys, continuing after the left-driven rows.
__global__ void join_expand_right_kernel(const u64 *__restrict__ pos, u32 nr, u64 total, const u64 *__restrict__ rkeys,
                                         const u64 *__restrict__ roffs, const u64 *__restrict__ rvals, u32 rb,
                                         u64 *__restrict__ out_k, u64 *__restrict__ out_v, u64 *__restrict__ out_w,
                                         unsigned char *__restrict__ out_vv, unsigned char *__restrict__ out_wv)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 o = pos[0] + (u64)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += stride) {
        u32 lo = 0, hi = nr;
        while (hi - lo > 1) {
            u32 mid = (lo + hi) >> 1;
            if (pos[mid] <= o) lo = mid; else hi = mid;
        }
        const u32 j = rb + lo;
        out_k[o] = rkeys[j];
        out_v[o] = 0;
        out_w[o] = rvals[roffs[j] + (o - pos[lo])];
        if (out_vv) out_vv[o] = 0;
        if (out_wv) out_wv[o] = 1;
    }
}

// ---------------------------------------------------------------------------------------------
// N-way cogroup and inner join (CoGroupedRdd::compute with n parents).  The output keys are side 0's keys, then each
// later side's new keys (those no earlier side has).  match is key-major: row o holds output key o's index on every
// side (a global key index of that side's CSR), 0xFFFFFFFF where the side lacks the key.
// ---------------------------------------------------------------------------------------------
constexpr u32 CGN_MAX_SIDES = 16;
struct CogroupNSides {
    Table tab[CGN_MAX_SIDES];            // key dictionaries; keys NULL: the side has no rows
    const u32 *dense[CGN_MAX_SIDES];     // dictionary slot -> key index
    const u64 *keys[CGN_MAX_SIDES];      // CSR keys, offsets and values (res_*)
    const u64 *offs[CGN_MAX_SIDES];
    const u64 *vals[CGN_MAX_SIDES];
    u32 kb[CGN_MAX_SIDES];               // the partition's first key on each side
    u32 n;
};
struct JoinNOut {
    u64 *k;
    u64 *v[CGN_MAX_SIDES];
};

// Keys [kb_i, kb_i + nk) of side i: row t = the key's index on every side (its own: kb_i + t).  Side i > 0 sets
// flag[t] = 1 and lidx[t] = t for a key no side j < i has, and writes only the entries j > i of its row (the others
// are known: 0xFFFFFFFF before i, kb_i + t at i); the rows of other keys are left unfinished and never used.
__global__ void cogroup_n_probe_kernel(const __grid_constant__ CogroupNSides a, u32 i, u32 nk, u32 *__restrict__ rows,
                                       unsigned char *__restrict__ flag, u64 *__restrict__ lidx)
{
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nk) return;
    const u64 key = a.keys[i][a.kb[i] + t];
    for (u32 j = 0; j < a.n; ++j) {
        u32 m = a.kb[i] + t;
        if (j != i) {
            const u32 s = a.tab[j].keys ? table_find(a.tab[j], key) : 0xFFFFFFFFu;
            m = s != 0xFFFFFFFFu ? a.dense[j][s] : 0xFFFFFFFFu;
        }
        if (j < i && m != 0xFFFFFFFFu) { flag[t] = 0; return; }     // an earlier side already gave this key
        if (i == 0 || j > i) rows[(u64)t * a.n + j] = m;
    }
    if (i) { flag[t] = 1; lidx[t] = t; }
}

// out[o] = the match row of side i's new key lidx[o] (n entries per row), for its m new keys in output order: 0xFFFFFFFF
// for the sides before i, its own index kb_i + lidx[o] for side i, and the probe's entries of rows after i
__global__ void cogroup_n_take_rows_kernel(const u32 *__restrict__ rows, u32 n, u32 i, u32 kb_i, const u64 *__restrict__ lidx, u64 m,
                                           u32 *__restrict__ out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < m * n; e += stride) {
        const u64 o = e / n;
        const u32 j = (u32)(e - o * n);
        out[e] = j < i ? 0xFFFFFFFFu : j == i ? kb_i + (u32)lidx[o] : rows[lidx[o] * n + j];
    }
}

// Side 0's list offsets, out[i] for i in [0, n): its CSR offsets of keys [lb, lb + nl) rebased to base, then n_lv (an
// empty list) for the keys after side 0's.
__global__ void cogroup_left_offsets_kernel(const u64 *__restrict__ loffs, u32 lb, u32 nl, u64 n, u64 base, u64 n_lv,
                                            u64 *__restrict__ out)
{
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = i < nl ? loffs[lb + i] - base : n_lv;
}

// cnt[o] = the length of output key o's list on side j (0 where the side lacks the key)
__global__ void cogroup_n_count_kernel(const u32 *__restrict__ match, u32 n, u32 j, u32 nk, const u64 *__restrict__ offs,
                                       u64 *__restrict__ cnt)
{
    const u32 o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nk) return;
    const u32 m = match[(u64)o * n + j];
    cnt[o] = m != 0xFFFFFFFFu ? offs[m + 1] - offs[m] : 0;
}

// Side j's values in output key order, one thread per value: value o belongs to the largest key index k with
// pos[k] <= o (keys with an empty list share pos with the next key), and its source segment is side j's key match[k][j].
// The values written are the ones the scanned lengths cover (pos[nk]), so no thread reads past a segment even if the key
// list missed a key of the side.
__global__ void cogroup_n_gather_kernel(const u64 *__restrict__ pos, u32 nk, const u32 *__restrict__ match, u32 n, u32 j,
                                        const u64 *__restrict__ offs, const u64 *__restrict__ vals, u64 *__restrict__ out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x, total = pos[nk];
    for (u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += stride) {
        u32 lo = 0, hi = nk;
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (pos[mid] <= o) lo = mid; else hi = mid;
        }
        out[o] = vals[offs[match[(u64)lo * n + j]] + (o - pos[lo])];
    }
}

// Inner join, side 0's keys o < nk: cnt[o] = the product of the key's list lengths over all sides, 0 when a side lacks
// the key.  A product of 2^63 or more sets *too_large (cnt 0).  sums[0] / sums[1] accumulate the sum of cnt >> 32 and
// of cnt & 0xFFFFFFFF, so the host can tell an exact partition total of 2^63 or more from a wrapped one.
__global__ void join_n_count_kernel(const __grid_constant__ CogroupNSides a, const u32 *__restrict__ match, u32 nk,
                                    u64 *__restrict__ cnt, unsigned long long *__restrict__ sums, u32 *__restrict__ too_large)
{
    const u32 o = blockIdx.x * blockDim.x + threadIdx.x;
    u64 c = 0;
    if (o < nk) {
        const u32 *row = match + (u64)o * a.n;
        bool all = true;
        for (u32 j = 0; j < a.n; ++j) all = all && row[j] != 0xFFFFFFFFu;
        if (all) {
            c = 1;
            for (u32 j = 0; j < a.n && c; ++j) {
                const u64 len = a.offs[j][row[j] + 1] - a.offs[j][row[j]];
                const u64 p = c * len;
                if (__umul64hi(c, len) || (p >> 63)) { atomicOr(too_large, 1u); c = 0; }
                else c = p;
            }
        }
        cnt[o] = c;
    }
    u64 hi = c >> 32, lo = c & 0xFFFFFFFFull;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        hi += __shfl_down_sync(0xffffffffu, hi, off);
        lo += __shfl_down_sync(0xffffffffu, lo, off);
    }
    if ((threadIdx.x & 31) == 0 && (hi | lo)) {
        atomicAdd(&sums[0], (unsigned long long)hi);
        atomicAdd(&sums[1], (unsigned long long)lo);
    }
}

// One thread per output row: the owning key k is the largest with pos[k] <= row; the row's position within the key is
// split into one digit per side, the last side varying fastest (for v0 in l0 { for v1 in l1 { ... } }).
__global__ void join_n_expand_kernel(const __grid_constant__ CogroupNSides a, const u64 *__restrict__ pos, u32 nk, u64 total,
                                     const u32 *__restrict__ match, const __grid_constant__ JoinNOut out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += stride) {
        u32 lo = 0, hi = nk;
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (pos[mid] <= o) lo = mid; else hi = mid;
        }
        const u32 *row = match + (u64)lo * a.n;
        u64 local = o - pos[lo];
        for (u32 j = a.n; j-- > 0;) {
            const u64 b = a.offs[j][row[j]];
            u64 d = local;
            if (j) {
                const u64 len = a.offs[j][row[j] + 1] - b;
                local = d / len;
                d -= local * len;
            }
            out.v[j][o] = a.vals[j][b + d];
        }
        out.k[o] = a.keys[0][a.kb[0] + lo];
    }
}

// N-way outer join over the keys of a cogroup plan (side 0's nk0 keys, then new_keys).  A side is required when its bit
// of `required` is set; an optional side that lacks the key takes one None slot (value 0, validity 0).  The expand
// needs no mask: a key that lacks a required side has no rows, so every 0xFFFFFFFF it meets is an optional side.
struct JoinNOuterOut {
    u64 *k;
    u64 *v[CGN_MAX_SIDES];
    unsigned char *valid[CGN_MAX_SIDES];   // NULL entries are not written
    const u64 *new_keys;                   // output keys nk0 .. of the plan
    u32 nk0;
};

// Output keys o < nk: cnt[o] = 0 if a required side lacks the key, else the product over all sides of max(len, 1).
// Overflow and the hi / lo sums as join_n_count_kernel.
__global__ void join_n_outer_count_kernel(const __grid_constant__ CogroupNSides a, const u32 *__restrict__ match, u32 nk,
                                          u32 required, u64 *__restrict__ cnt, unsigned long long *__restrict__ sums,
                                          u32 *__restrict__ too_large)
{
    const u32 o = blockIdx.x * blockDim.x + threadIdx.x;
    u64 c = 0;
    if (o < nk) {
        const u32 *row = match + (u64)o * a.n;
        bool kept = true;
        for (u32 j = 0; j < a.n; ++j) kept = kept && (row[j] != 0xFFFFFFFFu || !((required >> j) & 1u));
        if (kept) {
            c = 1;
            for (u32 j = 0; j < a.n && c; ++j) {
                if (row[j] == 0xFFFFFFFFu) continue;
                const u64 len = a.offs[j][row[j] + 1] - a.offs[j][row[j]];
                const u64 p = c * len;
                if (__umul64hi(c, len) || (p >> 63)) { atomicOr(too_large, 1u); c = 0; }
                else c = p;
            }
        }
        cnt[o] = c;
    }
    u64 hi = c >> 32, lo = c & 0xFFFFFFFFull;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        hi += __shfl_down_sync(0xffffffffu, hi, off);
        lo += __shfl_down_sync(0xffffffffu, lo, off);
    }
    if ((threadIdx.x & 31) == 0 && (hi | lo)) {
        atomicAdd(&sums[0], (unsigned long long)hi);
        atomicAdd(&sums[1], (unsigned long long)lo);
    }
}

// One thread per output row, as join_n_expand_kernel: the digit of a side that lacks the key has radix 1 (always 0)
// and gives a None slot.  KEYS: write out.k (the string join writes its keys once per key instead, and leaves out.k,
// out.new_keys and out.nk0 unset).
template <bool KEYS>
__device__ __forceinline__ void join_n_outer_expand_rows(const CogroupNSides &a, const u64 *__restrict__ pos, u32 nk, u64 total,
                                                         const u32 *__restrict__ match, const JoinNOuterOut &out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += stride) {
        u32 lo = 0, hi = nk;
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (pos[mid] <= o) lo = mid; else hi = mid;
        }
        const u32 *row = match + (u64)lo * a.n;
        u64 local = o - pos[lo];
        for (u32 j = a.n; j-- > 0;) {
            const u32 m = row[j];
            if (m == 0xFFFFFFFFu) {
                out.v[j][o] = 0;
                if (out.valid[j]) out.valid[j][o] = 0;
                continue;
            }
            const u64 b = a.offs[j][m];
            u64 d = local;
            if (j) {
                const u64 len = a.offs[j][m + 1] - b;
                local = d / len;
                d -= local * len;
            }
            out.v[j][o] = a.vals[j][b + d];
            if (out.valid[j]) out.valid[j][o] = 1;
        }
        if (KEYS) out.k[o] = lo < out.nk0 ? a.keys[0][a.kb[0] + lo] : out.new_keys[lo - out.nk0];
    }
}

__global__ void join_n_outer_expand_kernel(const __grid_constant__ CogroupNSides a, const u64 *__restrict__ pos, u32 nk,
                                           u64 total, const u32 *__restrict__ match, const __grid_constant__ JoinNOuterOut out)
{
    join_n_outer_expand_rows<true>(a, pos, nk, total, match, out);
}

__global__ void join_n_outer_expand_nokey_kernel(const __grid_constant__ CogroupNSides a, const u64 *__restrict__ pos, u32 nk,
                                                 u64 total, const u32 *__restrict__ match, const __grid_constant__ JoinNOuterOut out)
{
    join_n_outer_expand_rows<false>(a, pos, nk, total, match, out);
}

// ---------------------------------------------------------------------------------------------
// bincode 1.2.1 blob codec (SURVEY §8(f) N1): pure byte shuffling, HBM-bound
// ---------------------------------------------------------------------------------------------
// Vec<(u64,u64)>: out = u64 n | n x (k, c)
__global__ void blob_pairs_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ comb, u64 n, u64 *__restrict__ out)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    if (i == 0) out[0] = n;
    for (; i < n; i += stride) {
        out[1 + 2 * i] = keys[i];
        out[2 + 2 * i] = comb ? comb[i] : 0ull;
    }
}

// Vec<(u64,Vec<u64>)>: record i starts at word 1 + 2 i + offs[i] - base: (k, len, values...)
__global__ void blob_group_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ offs /*[nk+1], absolute*/, u64 nk,
                                  const u64 *__restrict__ vals /*absolute index*/, u64 *__restrict__ out)
{
    const u64 base = offs[0], nv = offs[nk] - base;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    if (t == 0) out[0] = nk;
    for (u64 i = t; i < nk; i += stride) {
        const u64 w = 1 + 2 * i + (offs[i] - base);
        out[w] = keys[i];
        out[w + 1] = offs[i + 1] - offs[i];
    }
    for (u64 j = t; j < nv; j += stride) {      // value j belongs to the key i with offs[i] <= base + j < offs[i+1]
        u64 lo = 0, hi = nk;
        while (hi - lo > 1) {
            const u64 mid = (lo + hi) >> 1;
            if (offs[mid] - base <= j) lo = mid; else hi = mid;
        }
        out[1 + 2 * (lo + 1) + j] = vals[base + j];
    }
}

// OR and AND over all (order-transformed) keys: a radix digit on which every key agrees needs no pass.
__global__ void key_bits_kernel(const u64 *__restrict__ keys, u64 stride_words, u64 n, int tx, unsigned long long *__restrict__ out /*[2]: or, and*/)
{
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 step = (u64)gridDim.x * blockDim.x;
    const u64 pol = policy_evict_first();
    u64 o = 0, a = ~0ull;
    for (; i < n; i += step) {
        const u64 k = tx_fwd(ld_stream_u64(keys + i * stride_words, pol), tx);
        o |= k; a &= k;
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        o |= __shfl_xor_sync(0xffffffffu, o, off);
        a &= __shfl_xor_sync(0xffffffffu, a, off);
    }
    if ((threadIdx.x & 31u) == 0) { atomicOr(&out[0], (unsigned long long)o); atomicAnd(&out[1], (unsigned long long)a); }
}

// ---------------------------------------------------------------------------------------------
// sort_by_key partition cuts: start of partition p = floor(p*n/R) moved past equal keys
// ---------------------------------------------------------------------------------------------
__global__ void sort_cuts_kernel(const u64 *__restrict__ keys, u64 n, u32 n_parts, u64 *__restrict__ starts)
{
    u32 p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > n_parts) return;
    if (p == 0) { starts[0] = 0; return; }
    if (p == n_parts) { starts[p] = n; return; }
    u64 c = ((u64)p * n) / n_parts;   // n < 2^32 and p < 2^32: no overflow
    if (c > 0 && c < n && keys[c] == keys[c - 1]) {   // upper bound of keys[c-1] in [c, n)
        const u64 k = keys[c - 1];
        u64 lo = c, hi = n;
        while (lo < hi) {
            u64 mid = lo + ((hi - lo) >> 1);
            if (keys[mid] == k) lo = mid + 1; else hi = mid;
        }
        c = lo;
    }
    starts[p] = c;
}

// ---------------------------------------------------------------------------------------------
// Synthetic input (SURVEY.md §8(d)); must match oracle/vega_oracle.c:vo_gen_uniform bit for bit
// ---------------------------------------------------------------------------------------------
enum : int { GEN_UNIFORM = 0, GEN_ZIPF = 1, GEN_UNIQUE = 2 };

__global__ void gen_pairs_kernel(u64 *__restrict__ rows, u64 *__restrict__ keys, u64 *__restrict__ vals, u64 first, u64 n,
                                 int mode, u64 n_distinct, u64 rank_base, u64 seed_k, u64 seed_v,
                                 const double *__restrict__ zipf_cdf)
{
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        const u64 i = first + t;
        u64 rank;
        if (mode == GEN_UNIQUE) {
            rank = rank_base + i;
        } else if (mode == GEN_ZIPF) {
            const double u = (double)(splitmix64(seed_k + i) >> 11) * (1.0 / 9007199254740992.0);
            u64 lo = 0, hi = n_distinct - 1;     // first index with cdf[idx] >= u
            while (lo < hi) {
                u64 mid = (lo + hi) >> 1;
                if (zipf_cdf[mid] >= u) hi = mid; else lo = mid + 1;
            }
            rank = lo;
        } else {
            rank = splitmix64(seed_k + i) % n_distinct;
        }
        const u64 k = splitmix64(rank ^ 0xA5A5A5A5A5A5A5A5ull);
        const u64 v = splitmix64(seed_v + i) & 0xFFFFFull;
        if (rows) {
            ulonglong2 r; r.x = k; r.y = v;
            *reinterpret_cast<ulonglong2 *>(rows + 2 * t) = r;
        } else {
            keys[t] = k;
            if (vals) vals[t] = v;
        }
    }
}

}  // namespace vb
