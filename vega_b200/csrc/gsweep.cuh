// gsweep.cuh — the scatter of every LSD sort pass (DG_BITS digits) over row streams, third generation.
// rp_sweep_kernel (sweep.cuh) is kept for the (u64,u64) multisplits; measured on the sort passes, it was the slower one:
//
// rp_sweep_kernel spends half of a pass issue-bound in the ballot ranking and the other half bound by the
// shared-memory pipe while it permutes whole rows into a staging buffer (bank conflicts; mio_throttle + short_scoreboard
// stalls) — one after the other, separated by CTA barriers, with nothing else resident on the SM to fill the idle unit.
// This kernel changes three things:
//
//   * rows are never permuted in shared memory.  The tile stays where the copy engine put it (cp.async.bulk + mbarrier);
//     ranking reads only the keys, the scatter phase writes one u16 per row (perm[output position] = source row), and
//     the write-out gathers key and value through perm and recomputes the digit from the key (a shift and a mask) —
//     no staged copy of the values, no staged digit bytes, fewer shared-memory wavefronts per row;
//   * no row lives in registers across a barrier (only digit|rank words), so a tile is 7-11 rows deep per thread and its
//     buffers are filled by the copy engine while the previous tile is processed: the keys of tile t+1 land in a SECOND
//     key buffer during tile t, the value buffer is refilled right after tile t's write-out and has the whole
//     ranking/scan/scatter of tile t+1 to arrive.  (With one tile buffer and two 512-thread CTAs per SM hiding the load
//     behind each other, the mbarrier wait was the top stall.)  CTA shapes: 1024 threads x 1 CTA per SM for rows with a
//     value (11264-row tiles of (u32,u64)), 512 x 2 for key-only rows;
//   * the ranking is the minimal ballot sequence in PTX (R2P, 8 x VOTE, predicated NOT, 3-input LOP3: 25 instructions
//     per row instead of the 48 the compiler emitted for the C loop), the leader test is `no lower peer` instead of
//     ffs + shfl, the digit bases are folded into the warp counters by the column scan, and the full-tile path carries
//     no validity checks.
//
// Stable: output order inside a digit = (part, tile, warp, item, lane) = input order, exactly as rp_sweep_kernel.
// Offsets from the per-part histogram (rp_hist_kernel + rp_scan_kernel), one contiguous part per CTA; DG_BITS digits only.
// (Tried and dropped: tiles in global order with a per-tile histogram and a column scan — the scatter itself was no
//  faster, so the write pattern of 256 x 300 separate streams is not what bounds it, and the per-tile histogram added
//  a costly pass of its own.)
#pragma once
#include "sweep.cuh"

namespace vb {

// CTA shape by row type (A/B on 1e9 rows): key-only rows 512 threads x 2 CTAs per SM,
// rows with a value 1024 x 1 (the longest runs per digit)
#ifndef VB_GS_THREADS_KEY
#define VB_GS_THREADS_KEY 512
#endif
#ifndef VB_GS_THREADS_VAL
#define VB_GS_THREADS_VAL 1024
#endif
// which row types keep TWO key buffers (the keys of tile t+1 land while tile t is processed; the value buffer is refilled right
// after a tile's write-out and has the whole ranking/scan/scatter of the next tile to arrive).  bit 0: u64 key only, bit 1: (u64,u64) SoA,
// bit 2: (u32 id, u64) SoA, bit 3: u32 id + values inside AoS rows.  AoS (u64,u64) rows arrive as one 16-byte unit: single buffer.
#ifndef VB_GS_DB
#define VB_GS_DB 0xF
#endif

template <typename KeyT, bool HAS_VAL, int LDM>
struct GsPlan {
    static constexpr bool AOS = (LDM == LD_AOS64);                 // (u64,u64) rows: key and value arrive together
    static constexpr bool VAL_AOS = (LDM == LD_KEY32_VAL_AOS);     // u32 ids (SoA) + values inside 16-byte rows
    static constexpr int THREADS = HAS_VAL ? VB_GS_THREADS_VAL : VB_GS_THREADS_KEY;
    static constexpr int CTAS = 1024 / THREADS;
    static constexpr int WARPS = THREADS / 32;
    static constexpr int KEY_B = AOS ? 16 : (int)sizeof(KeyT);     // bytes per row in the key buffer
    static constexpr int VAL_B = AOS ? 0 : VAL_AOS ? 16 : (HAS_VAL ? 8 : 0);
    static constexpr int DB_BIT = AOS ? -1 : VAL_AOS ? 3 : LDM == LD_KEY32_VAL_SOA ? 2 : HAS_VAL ? 1 : 0;
    static constexpr bool DB = DB_BIT >= 0 && ((VB_GS_DB >> (DB_BIT < 0 ? 0 : DB_BIT)) & 1);   // two key buffers
    static constexpr int ROW_B = KEY_B * (DB ? 2 : 1) + VAL_B + 2; // + the u16 perm entry
    static constexpr int CNT_B = WARPS * SW_NB * 2;                // warp-private u16 counters
    // 227 KB per SM, 1 KB reserved per resident CTA, ~4 KB of static shared memory per CTA
    static constexpr int BUDGET = (232448 - CTAS * 1024) / CTAS - 4096 - CNT_B;
    static constexpr int K = BUDGET / (ROW_B * THREADS);           // rows per thread per tile
    static constexpr int T = K * THREADS;
    static constexpr size_t key_bytes = (size_t)T * KEY_B;
    static constexpr size_t val_bytes = (size_t)T * VAL_B;
    static constexpr size_t perm_bytes = (size_t)T * 2;
    static constexpr size_t total = key_bytes * (DB ? 2 : 1) + val_bytes + perm_bytes + CNT_B;
    static constexpr int WU = K <= 12 ? K : (K % 5 == 0 ? 5 : (K % 7 == 0 ? 7 : (K % 4 == 0 ? 4 : (K % 3 == 0 ? 3 : (K % 2 == 0 ? 2 : 1)))));   // write-out unroll: divides K
    static_assert(K >= 4 && T <= 65536, "tile must fit u16 positions");
    static_assert(total + 4096 <= (size_t)(232448 - CTAS * 1024) / CTAS, "CTAS resident CTAs fit the 227 KB of an SM");
    static_assert(key_bytes % 128 == 0 && val_bytes % 128 == 0, "bulk copy destinations stay 128-byte aligned");
};

// Lanes of the (fully active) warp whose 8-bit digit equals mine.
VB_D u32 match_digit8(u32 d)
{
    u32 peers;
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .b32 m0, m1, m2, m3, m4, m5, m6, m7, t;\n\t"
        "and.b32 t, %1, 1;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m0, p, 0xffffffff;\n\t@!p not.b32 m0, m0;\n\t"
        "and.b32 t, %1, 2;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m1, p, 0xffffffff;\n\t@!p not.b32 m1, m1;\n\t"
        "and.b32 t, %1, 4;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m2, p, 0xffffffff;\n\t@!p not.b32 m2, m2;\n\t"
        "and.b32 t, %1, 8;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m3, p, 0xffffffff;\n\t@!p not.b32 m3, m3;\n\t"
        "and.b32 t, %1, 16;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m4, p, 0xffffffff;\n\t@!p not.b32 m4, m4;\n\t"
        "and.b32 t, %1, 32;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m5, p, 0xffffffff;\n\t@!p not.b32 m5, m5;\n\t"
        "and.b32 t, %1, 64;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m6, p, 0xffffffff;\n\t@!p not.b32 m6, m6;\n\t"
        "and.b32 t, %1, 128;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 m7, p, 0xffffffff;\n\t@!p not.b32 m7, m7;\n\t"
        "lop3.b32 m0, m0, m1, m2, 0x80;\n\tlop3.b32 m3, m3, m4, m5, 0x80;\n\tlop3.b32 m6, m6, m7, m0, 0x80;\n\tand.b32 %0, m6, m3;\n\t"
        "}"
        : "=r"(peers)
        : "r"(d));
    return peers;
}

// CSR = the LAST pass of group_by_key's (dense id, value) sort: the ids are not written out any more; instead every row whose
// predecessor in the output has a different id records its output position as the start of that id's value run
// (a.csr[id] = min(position); a.csr is pre-set to all ones).  A run that continues an id from an earlier tile reports a
// larger position than the true start, which the atomicMin discards.  Replaces csr_bounds_kernel and 8 bytes/row of traffic.
template <typename KeyT, bool HAS_VAL, int LDM, bool CSR = false>
__global__ void __launch_bounds__((GsPlan<KeyT, HAS_VAL, LDM>::THREADS), (GsPlan<KeyT, HAS_VAL, LDM>::CTAS))
rp_gsweep_kernel(SweepArgs a, Digit dg)
{
    static_assert(!CSR || (LDM == LD_KEY32_VAL_SOA && sizeof(KeyT) == 4 && HAS_VAL), "CSR: (u32 id, u64 value) rows");
    using P = GsPlan<KeyT, HAS_VAL, LDM>;
    constexpr int THREADS = P::THREADS, WARPS = P::WARPS, K = P::K, T = P::T;
    constexpr bool AOS = P::AOS, VAL_AOS = P::VAL_AOS;
    constexpr bool VBUF = P::VAL_B != 0;                       // values arrive in their own buffer
    static_assert(LDM == LD_SOA64 || LDM == LD_AOS64 || LDM == LD_KEY32_VAL_SOA || LDM == LD_KEY32_VAL_AOS, "row-stream loaders only");
    static_assert(!AOS || (sizeof(KeyT) == 8 && HAS_VAL), "AoS rows are (u64,u64)");
    static_assert(SW_NB <= THREADS, "one thread per digit in the column scan");

    extern __shared__ __align__(128) unsigned char gs_smem[];
    constexpr bool DB = P::DB;
    constexpr int NKB = DB ? 2 : 1;
    unsigned char *kbuf0 = gs_smem;                                                 // NKB x ([T] KeyT, or [T] 16-byte rows (AoS))
    unsigned char *vbuf = gs_smem + NKB * P::key_bytes;                             // [T] u64, or [T] 16-byte rows (VAL_AOS)
    unsigned short *perm = (unsigned short *)(gs_smem + NKB * P::key_bytes + P::val_bytes);   // [T] source row of output position p
    unsigned short *cnt = perm + T;                                                 // [WARPS][256]
    __shared__ __align__(8) u64 bar_k[2], bar_v;
    __shared__ u32 wtot[SW_NB / 32];
    __shared__ u32 gbase[SW_NB];              // global offset of the first row of digit d of this tile, minus its tile position
    __shared__ u32 run_off[SW_NB];            // global offset of the next row of digit d of this part

    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
    const u32 lt = lanemask_lt();
    unsigned short *my_cnt = cnt + warp * SW_NB;
    const u64 pol = policy_evict_first();
    // CTA p owns the contiguous rows [p*rows_per_part, (p+1)*rows_per_part) and starts digit d at part_off[d*num_parts + p]
    const u64 begin = (u64)blockIdx.x * a.rows_per_part;
    const u64 end = min(a.n, begin + a.rows_per_part);
    if (begin >= end) return;
    const u32 n_full = (u32)((end - begin) / T);          // full tiles of this part; one partial tile may follow

    // one lane: copy-engine loads of full tile `it` of this part
    auto issue_keys = [&](u32 it) {
        const u64 r0 = begin + (u64)it * T;
        const u32 slot = DB ? (it & 1u) : 0u;
        unsigned char *kb = kbuf0 + slot * P::key_bytes;
        mbar_arrive_expect_tx(&bar_k[slot], (u32)P::key_bytes);
        if (AOS) bulk_g2s(kb, (const u64 *)a.keys + 2 * r0, (u32)P::key_bytes, &bar_k[slot], pol);
        else bulk_g2s(kb, (const KeyT *)a.keys + r0, (u32)P::key_bytes, &bar_k[slot], pol);
    };
    auto issue_vals = [&](u32 it) {
        if (!VBUF) return;
        const u64 r0 = begin + (u64)it * T;
        mbar_arrive_expect_tx(&bar_v, (u32)P::val_bytes);
        if (VAL_AOS) bulk_g2s(vbuf, (const u64 *)a.vals + 2 * r0, (u32)P::val_bytes, &bar_v, pol);
        else bulk_g2s(vbuf, (const u64 *)a.vals + r0, (u32)P::val_bytes, &bar_v, pol);
    };

    for (u32 d = tid; d < SW_NB; d += THREADS) run_off[d] = a.part_off[(size_t)d * a.num_parts + blockIdx.x];
    for (u32 i = lane; i < SW_NB / 2; i += 32) ((u32 *)my_cnt)[i] = 0;
    if (tid == 0) {
        mbar_init(&bar_k[0], 1);
        mbar_init(&bar_k[1], 1);
        mbar_init(&bar_v, 1);
        mbar_fence_init();
        if (n_full >= 1) { issue_keys(0); issue_vals(0); }
        if (DB && n_full >= 2) issue_keys(1);
    }
    __syncthreads();

    auto tile_body = [&](auto full_c, const u32 it, const u32 rows_here) {
        constexpr bool FULL = decltype(full_c)::value;
        const u64 t0 = begin + (u64)it * T;
        const u32 slot = DB ? (it & 1u) : 0u;
        unsigned char *kbuf = kbuf0 + slot * P::key_bytes;
        if (FULL) {
            mbar_wait(&bar_k[slot], DB ? ((it >> 1) & 1u) : (it & 1u));
        } else {
            // the part's last, partial tile: plain loads into the same buffers (no copy is in flight into them)
            for (u32 r = tid; r < rows_here; r += THREADS) {
                if (AOS) reinterpret_cast<ulonglong2 *>(kbuf)[r] = ld_stream_u64x2((const u64 *)a.keys + 2 * (t0 + r), pol);
                else if (sizeof(KeyT) == 8) reinterpret_cast<u64 *>(kbuf)[r] = ld_stream_u64((const u64 *)a.keys + (t0 + r), pol);
                else reinterpret_cast<u32 *>(kbuf)[r] = ld_stream_u32((const u32 *)a.keys + (t0 + r), pol);
                if (VBUF) {
                    if (VAL_AOS) reinterpret_cast<ulonglong2 *>(vbuf)[r] = ld_stream_u64x2((const u64 *)a.vals + 2 * (t0 + r), pol);
                    else reinterpret_cast<u64 *>(vbuf)[r] = ld_stream_u64((const u64 *)a.vals + (t0 + r), pol);
                }
            }
            __syncthreads();
        }
        auto smem_key = [&](u32 r) -> KeyT {
            if (AOS) return (KeyT) reinterpret_cast<const ulonglong2 *>(kbuf)[r].x;
            return reinterpret_cast<const KeyT *>(kbuf)[r];
        };

        // ---- 1. digit and warp-local rank of this thread's K rows: item i of lane l is tile row warp*32K + i*32 + l
        u32 dr[K];                      // digit | rank << 16   (digit 256 = row past the end)
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const u32 r = warp * (32 * K) + (u32)i * 32 + lane;
            dr[i] = (FULL || r < rows_here) ? rp_digit<KeyT, DG_BITS>(dg, smem_key(r)) : (u32)SW_NB;
        }
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const u32 d = dr[i];
            const u32 peers = FULL ? match_digit8(d) : warp_match_digit(d);
            const u32 lower = peers & lt;
            u32 base = 0;
            if (FULL || d < SW_NB) base = my_cnt[d];                      // every lane of the group reads the same counter
            __syncwarp();
            if (lower == 0 && (FULL || d < SW_NB)) my_cnt[d] = (unsigned short)(base + __popc(peers));   // the lowest lane advances it
            __syncwarp();
            dr[i] = d | ((base + __popc(lower)) << 16);
        }
        __syncthreads();                                                        // B1: warp counters complete

        // ---- 2. thread d < 256: exclusive scan of digit d over the warps and over the digits; afterwards
        //         cnt[w][d] = tile position of warp w's first row of digit d
        constexpr bool KEEP = WARPS <= 16;      // the column of counts stays in registers between the two sweeps
        u32 total = 0;
        u32 c[KEEP ? WARPS : 1];
        if (tid < SW_NB) {
#pragma unroll
            for (int w = 0; w < WARPS; ++w) { const u32 x = cnt[w * SW_NB + tid]; if (KEEP) c[w] = x; total += x; }
        }
        u32 incl = total;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const u32 t = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= (u32)off) incl += t;
        }
        if (tid < SW_NB && lane == 31) wtot[warp] = incl;
        __syncthreads();                                                        // B2: warp totals visible
        if (tid < SW_NB) {
            u32 excl = incl - total;
            for (u32 w = 0; w < warp; ++w) excl += wtot[w];
            const u32 ro = run_off[tid];
            gbase[tid] = ro - excl;
            run_off[tid] = ro + total;
#pragma unroll
            for (int w = 0; w < WARPS; ++w) { const u32 x = KEEP ? c[w] : (u32)cnt[w * SW_NB + tid]; cnt[w * SW_NB + tid] = (unsigned short)excl; excl += x; }
        }
        __syncthreads();                                                        // B3: positions visible

        // ---- 3. perm[output position inside the tile] = source row
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const u32 d = dr[i] & 0xFFFFu;
            if (FULL || d < SW_NB) {
                const u32 pos = cnt[warp * SW_NB + d] + (dr[i] >> 16);
                perm[pos] = (unsigned short)(warp * (32 * K) + (u32)i * 32 + lane);
            }
        }
        __syncthreads();                                                        // B4: perm complete, counters consumed
        for (u32 i = lane; i < SW_NB / 2; i += 32) ((u32 *)my_cnt)[i] = 0;      // own counters: next tile's ranking
        if (FULL && VBUF) mbar_wait(&bar_v, it & 1u);

        // ---- 4. write-out: consecutive threads take consecutive output positions (runs of one digit are contiguous)
        [[maybe_unused]] KeyT *ok = (KeyT *)a.out_keys;
#pragma unroll (P::WU)
        for (int j = 0; j < K; ++j) {
            const u32 p = tid + (u32)j * THREADS;
            const bool valid = FULL || p < rows_here;
            if constexpr (CSR) {
                const u32 src = valid ? perm[p] : 0u;
                const u32 key = reinterpret_cast<const u32 *>(kbuf)[src];
                const u64 val = reinterpret_cast<const u64 *>(vbuf)[src];
                u32 prev = __shfl_up_sync(0xffffffffu, key, 1);              // output position p-1 is lane-1's row ...
                if (lane == 0) prev = (valid && p > 0) ? reinterpret_cast<const u32 *>(kbuf)[perm[p - 1]] : ~key;   // ... or the previous warp's last
                if (valid) {
                    const u32 o = gbase[rp_digit<KeyT, DG_BITS>(dg, (KeyT)key)] + p;
                    a.out_vals[o] = val;
                    if (prev != key) atomicMin((unsigned long long *)a.csr + key, (unsigned long long)o);
                }
            } else if (valid) {
                const u32 src = perm[p];
                KeyT key;
                u64 val = 0;
                if (AOS) {
                    const ulonglong2 row = reinterpret_cast<const ulonglong2 *>(kbuf)[src];
                    key = (KeyT)row.x; val = row.y;
                } else {
                    key = reinterpret_cast<const KeyT *>(kbuf)[src];
                    if (VAL_AOS) val = reinterpret_cast<const ulonglong2 *>(vbuf)[src].y;
                    else if (HAS_VAL) val = reinterpret_cast<const u64 *>(vbuf)[src];
                }
                const u32 o = gbase[rp_digit<KeyT, DG_BITS>(dg, key)] + p;
                ok[o] = key;
                if (HAS_VAL) a.out_vals[o] = val;
            }
        }
        if (FULL) fence_proxy_async();   // generic-proxy reads of the tile before the copy engine refills the buffers
        __syncthreads();                                                        // B5: tile buffers, perm and gbase reusable
        if (FULL && tid == 0) {
            const u32 nk = it + (DB ? 2u : 1u);
            if (nk < n_full) issue_keys(nk);
            if (it + 1 < n_full) issue_vals(it + 1);
        }
    };

    for (u32 it = 0; it < n_full; ++it) tile_body(std::true_type{}, it, (u32)T);
    if (begin + (u64)n_full * T < end) tile_body(std::false_type{}, n_full, (u32)(end - (begin + (u64)n_full * T)));
}

}  // namespace vb
