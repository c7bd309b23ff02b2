// sweep.cuh — the scatter of a radix pass over (u64, u64) row streams that the gather sweep (gsweep.cuh) does not take:
// the multisplits (DG_BUCKET, DG_DEST, DG_HASHTOP digits).
//
//   * offsets come from the per-part histogram (rp_hist_kernel + rp_scan_kernel): CTA p walks its own contiguous
//     part of the input and keeps running digit offsets in shared memory;
//   * input tiles are staged global → shared by the copy engine (cp.async.bulk + mbarrier): no registers,
//     no LSU instructions for the stream, and the next tile's copy is in flight while the current tile is
//     scanned, staged and written out;
//   * 4 CTA barriers per tile (rp_scatter_kernel has 5): warp-private u16 counters are cleared by their
//     own warp, the staging buffer is only rewritten after the next tile's third barrier.
//
// With 1024-thread CTAs (SW_THREADS) it is faster than rp_scatter_kernel on 1e9 rows.
// Stable: rows keep their input order inside every digit (tile order → warp order → lane-striped item order),
// which the group value order (SURVEY §8a, tests/test_pair_rdd.rs:30-36) relies on.
// Handles the row-stream loaders (all rows valid); table loaders and the REMOTE scatter stay on rp_scatter_kernel.
#pragma once
#include "kernels.cuh"

namespace vb {

// CTA shape (A/B on 1e9 rows): (u64,u64) rows want the longest runs per digit: 1024 threads x 1 CTA (6144-row tiles)
// beats 512 x 2 and 256 x 4.
#ifndef VB_SW_THREADS_VAL
#define VB_SW_THREADS_VAL 1024
#endif
constexpr int SW_THREADS = VB_SW_THREADS_VAL;
constexpr int SW_CTAS = 1024 / SW_THREADS;
constexpr int SW_NB = 256;
constexpr u64 SW_ROW_LIMIT = 1ull << 31;    // the sweeps take n < SW_ROW_LIMIT rows (u32 output positions); larger inputs use rp_scatter_kernel

// 6 items per thread: the tile buffers (raw + staged) of the resident CTAs fit the 227 KB of an SM
constexpr int SW_ITEMS = 6;
constexpr int SW_TILE = SW_THREADS * SW_ITEMS;

// shared-memory plan (bytes): [raw vals | raw keys] [staged vals | staged keys | staged digit] [warp counters u16]
template <int LDM>
struct SwSmem {
    static constexpr int T = SW_TILE;
    static constexpr bool AOS = (LDM == LD_AOS64);
    static constexpr size_t raw_vals = AOS ? 0 : (size_t)T * 8;
    static constexpr size_t raw_keys = AOS ? (size_t)T * 16 : (size_t)T * 8;
    static constexpr size_t raw = raw_vals + raw_keys;
    static constexpr size_t st_vals = (size_t)T * 8;
    static constexpr size_t st_keys = (size_t)T * 8;
    static constexpr size_t st_dig = (size_t)T;
    static constexpr size_t cnt = (size_t)(SW_THREADS / 32) * SW_NB * 2;
    static constexpr size_t total = raw + st_vals + st_keys + st_dig + cnt;
};

struct SweepArgs {
    const void *keys;         // u64* / u32* / AoS rows
    const void *vals;         // u64* or NULL; LD_KEY32_VAL_AOS: AoS rows whose .y is the value
    u64 n;
    u32 n_tiles;              // rp_sweep_kernel: tiles of the whole input
    void *out_keys;
    u64 *out_vals;
    // CTA p owns the contiguous rows [p*rows_per_part, (p+1)*rows_per_part) and starts digit d at
    // part_off[d*num_parts + p] (the scanned per-part histogram of rp_hist_kernel + rp_scan_kernel)
    const u32 *part_off;
    u32 num_parts;
    u64 rows_per_part;        // multiple of the tile size
    u64 *csr;                 // rp_gsweep_kernel<CSR>: csr[id] = min(output position of a row that starts a run of id)
};

// Each CTA walks its own contiguous part tile by tile (copy-engine staging, warp-private u16 counters, 4 barriers,
// full-tile fast path) and keeps running digit offsets in shared memory.
template <int LDM, int DGM>
__global__ void __launch_bounds__(SW_THREADS, SW_CTAS)
rp_sweep_kernel(SweepArgs a, Digit dg)
{
    constexpr int SW_WARPS = SW_THREADS / 32;
    static_assert(SW_NB <= SW_THREADS, "one thread per digit in the column scan");
    using SM = SwSmem<LDM>;
    constexpr int K = SW_ITEMS;
    constexpr int T = SM::T;
    constexpr bool AOS = SM::AOS;
    static_assert(LDM == LD_SOA64 || LDM == LD_AOS64, "(u64,u64) row-stream loaders only");

    extern __shared__ __align__(128) unsigned char sw_smem[];
    unsigned char *raw_vals_b = sw_smem;                                   // [T] u64 (SoA values)
    unsigned char *raw_keys_b = sw_smem + SM::raw_vals;                    // [T] u64 keys, or [T] 16-byte rows (AoS)
    u64 *st_vals = (u64 *)(sw_smem + SM::raw);
    u64 *st_keys = (u64 *)(sw_smem + SM::raw + SM::st_vals);
    unsigned char *st_dig = sw_smem + SM::raw + SM::st_vals + SM::st_keys;
    unsigned short *cnt = (unsigned short *)(sw_smem + SM::raw + SM::st_vals + SM::st_keys + SM::st_dig);   // [SW_WARPS][256]
    __shared__ __align__(8) u64 full_bar;
    __shared__ u32 s_tile[2];                 // tile ids: [current, next]
    __shared__ u32 wtot[SW_WARPS];
    __shared__ u32 dbase[SW_NB];              // tile-local start of digit d
    __shared__ u32 gbase[SW_NB];              // global offset of digit d's first row of this tile, minus dbase[d]
    __shared__ u32 run_off[SW_NB];            // global offset of the next row of digit d of this part

    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
    const u32 lt = lanemask_lt();
    unsigned short *my_cnt = cnt + warp * SW_NB;
    const u64 pol = policy_evict_first();
    const u64 n = a.n;

    // issue the copy-engine loads of full tile `t` into the raw buffer (one lane)
    auto issue_tile = [&](u32 t) {
        const u64 r0 = (u64)t * T;
        mbar_arrive_expect_tx(&full_bar, (u32)SM::raw);
        if (AOS) {
            bulk_g2s(raw_keys_b, (const u64 *)a.keys + 2 * r0, (u32)SM::raw_keys, &full_bar, pol);
        } else {
            bulk_g2s(raw_keys_b, (const u64 *)a.keys + r0, (u32)SM::raw_keys, &full_bar, pol);
            bulk_g2s(raw_vals_b, (const u64 *)a.vals + r0, (u32)SM::raw_vals, &full_bar, pol);
        }
    };
    auto tile_is_full = [&](u32 t) { return (u64)(t + 1) * T <= n; };

    // this CTA's tiles are [part_first, part_last); a.n_tiles doubles as the "no more tiles" sentinel
    const u32 part_first = (u32)(((u64)blockIdx.x * a.rows_per_part) / T);
    const u32 part_last = (u32)min((u64)a.n_tiles, (((u64)blockIdx.x + 1) * a.rows_per_part) / T);
    for (u32 d = tid; d < SW_NB; d += SW_THREADS) run_off[d] = a.part_off[(size_t)d * a.num_parts + blockIdx.x];
    if (tid == 0) {
        mbar_init(&full_bar, 1);
        mbar_fence_init();
        const u32 t0 = part_first < part_last ? part_first : a.n_tiles;
        s_tile[0] = t0;
        if (t0 < a.n_tiles && tile_is_full(t0)) issue_tile(t0);
    }
    for (u32 i = lane; i < SW_NB / 2; i += 32) ((u32 *)my_cnt)[i] = 0;
    __syncthreads();

    u32 phase = 0;
    for (u32 it = 0;; ++it) {
        const u32 tile = s_tile[it & 1u];
        if (tile >= a.n_tiles) break;
        const u64 row0 = (u64)tile * T;
        const bool full = tile_is_full(tile);
        const u32 rows_here = full ? (u32)T : (u32)(n - row0);

        // ---- 1. this thread's K items: warp-striped, item i of lane l is tile row warp*32K + i*32 + l
        u64 key[K];
        u64 val[K];
        u32 dr[K];                      // digit | rank << 16   (digit 256 = row past the end)
        if (full) {
            mbar_wait(&full_bar, phase);
            phase ^= 1u;
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const u32 r = warp * (32 * K) + (u32)i * 32 + lane;
                if (AOS) {
                    const ulonglong2 row = reinterpret_cast<const ulonglong2 *>(raw_keys_b)[r];
                    key[i] = row.x; val[i] = row.y;
                } else {
                    key[i] = reinterpret_cast<const u64 *>(raw_keys_b)[r];
                    val[i] = reinterpret_cast<const u64 *>(raw_vals_b)[r];
                }
                dr[i] = rp_digit<u64, DGM>(dg, key[i]);
            }
            fence_proxy_async();         // generic-proxy reads of the raw buffer before the copy engine refills it
        } else {
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const u32 r = warp * (32 * K) + (u32)i * 32 + lane;
                key[i] = 0; val[i] = 0;
                dr[i] = SW_NB;
                if (r < rows_here) {
                    Loader l{LDM, a.keys, a.vals, 0};
                    rp_load<u64, LDM>(l, row0 + r, key[i], val[i], pol);
                    dr[i] = rp_digit<u64, DGM>(dg, key[i]);
                }
            }
        }

        // ---- 2. rank inside the warp (ballots), warp-private counters
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const u32 d = dr[i];
            u32 peers;
            if (full) {
                peers = 0xffffffffu;
#pragma unroll
                for (int b = 0; b < 8; ++b) {
                    const bool bit = (d >> b) & 1u;
                    const u32 m = __ballot_sync(0xffffffffu, bit);
                    peers &= bit ? m : ~m;
                }
            } else {
                peers = warp_match_digit(d);
            }
            const u32 leader = (u32)(__ffs(peers) - 1);
            u32 base = 0;
            if (lane == leader && d < SW_NB) { base = my_cnt[d]; my_cnt[d] = (unsigned short)(base + __popc(peers)); }
            base = __shfl_sync(0xffffffffu, base, leader);
            dr[i] = d | ((base + __popc(peers & lt)) << 16);
            __syncwarp();
        }
        __syncthreads();                                                        // B1: counters complete, raw buffer consumed
        if (tid == 0) {                                                          // prefetch the next tile of the part
            const u32 nx = tile + 1 < part_last ? tile + 1 : a.n_tiles;
            s_tile[(it + 1) & 1u] = nx;
            if (nx < a.n_tiles && tile_is_full(nx)) issue_tile(nx);
        }

        // ---- 3. thread d < 256: column scan over the warps, block scan over digits
        u32 total = 0;
        if (tid < SW_NB) {
#pragma unroll
            for (int w = 0; w < SW_WARPS; ++w) { const u32 c = cnt[w * SW_NB + tid]; cnt[w * SW_NB + tid] = (unsigned short)total; total += c; }
        }
        u32 incl = total;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const u32 t = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= (u32)off) incl += t;
        }
        if (tid < SW_NB && lane == 31) wtot[warp] = incl;
        __syncthreads();                                                        // B2: warp totals + warp offsets visible
        u32 excl_local = 0;
        if (tid < SW_NB) {
            excl_local = incl - total;
            for (u32 w = 0; w < warp; ++w) excl_local += wtot[w];
            dbase[tid] = excl_local;
        }
        __syncthreads();                                                        // B3: dbase visible
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const u32 d = dr[i] & 0xFFFFu;
            if (d < SW_NB) {
                const u32 pos = dbase[d] + cnt[warp * SW_NB + d] + (dr[i] >> 16);
                st_keys[pos] = key[i];
                st_vals[pos] = val[i];
                st_dig[pos] = (unsigned char)d;
            }
        }
        // ---- 4. global offsets of this tile's digits from the part's running offsets
        if (tid < SW_NB) { const u32 ro = run_off[tid]; gbase[tid] = ro - excl_local; run_off[tid] = ro + total; }
        __syncthreads();                                                        // B4: tile staged
        for (u32 i = lane; i < SW_NB / 2; i += 32) ((u32 *)my_cnt)[i] = 0;      // own counters: next tile's ranking
        __syncwarp();
        u64 *ok = (u64 *)a.out_keys;
        for (u32 p = tid; p < rows_here; p += SW_THREADS) {
            const u32 o = gbase[st_dig[p]] + p;
            ok[o] = st_keys[p];
            a.out_vals[o] = st_vals[p];
        }
        // no barrier here: the staging buffer is rewritten only after the next tile's B3, dbase/gbase after its B2
    }
}

}  // namespace vb
