// Sorted value lists (vb_shuffle_set_value_order): every run vals[offs[i] .. offs[i+1]) of a reduce-side CSR sorted
// ascending in the value dtype's order, in place.  The order is tx_fwd's: unsigned for u64, signed for i64 and
// f64::total_cmp for f64, so two values tie only when their bits are equal.
//
//   seg_classify_kernel   each key with L >= 2 values into its size class: class c < SS_LOG_T holds 2^c < L <= 2^(c+1)
//                         (2 <= L <= SS_T over all of them), class SS_LOG_T the large runs (L > SS_T).  One pass counts
//                         (warp-aggregated atomics), a second writes the key ids into each class's list.
//   seg_sort_cta_kernel   one class of runs padded to C = 2^(c+1) values each, SS_T / C runs per CTA: loaded as
//                         tx_fwd keys into shared memory, bitonic-sorted within each C-block, written back with tx_inv.
//   seg_move_kernel       the large runs gathered into one buffer with each value's run rank, and scattered back
//                         after the engine's LSD passes have sorted that buffer by (rank, value).
#pragma once
#include "common.cuh"

namespace vb {

constexpr int SS_LOG_T = 13, SS_T = 1 << SS_LOG_T;   // 8192 values = 64 KB of shared memory: two CTAs per SM
constexpr int SS_THREADS = 512;
constexpr int SS_NCLS = SS_LOG_T + 1;                 // the CTA classes, then the large runs

// mode 0: cnt[class] += runs of that class;  mode 1: list[cur[class]++] = key id
__global__ void seg_classify_kernel(const u64 *__restrict__ offs, u64 D, u32 *__restrict__ ctr, u32 *__restrict__ list, int fill)
{
    const u32 lane = threadIdx.x & 31u;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 base = (((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5) << 5; base < D; base += warps << 5) {
        const u64 i = base + lane;
        const u64 L = i < D ? offs[i + 1] - offs[i] : 0;
        const int cls = L < 2 ? -1 : L > (u64)SS_T ? SS_LOG_T : 63 - __clzll((long long)(L - 1));
        const u32 peers = __match_any_sync(0xffffffffu, cls);
        const u32 leader = __ffs(peers) - 1;
        u32 at = 0;
        if (cls >= 0 && lane == leader) at = atomicAdd(&ctr[cls], (u32)__popc(peers));
        at = __shfl_sync(0xffffffffu, at, leader);
        if (cls >= 0 && fill) list[at + __popc(peers & ((1u << lane) - 1u))] = (u32)i;
    }
}

// One class: run j of `list` takes the C-block j % (SS_T / C) of CTA j / (SS_T / C).  Padding is ~0, the largest key:
// it sorts behind every value of its block, and where it ties a value the two are the same bits.
__global__ void __launch_bounds__(SS_THREADS, 2)
seg_sort_cta_kernel(u64 *__restrict__ vals, const u64 *__restrict__ offs, const u32 *__restrict__ list, u32 n_runs, u32 log_c, int tx)
{
    extern __shared__ u64 sk[];
    const u32 C = 1u << log_c;
    const u64 first = (u64)blockIdx.x << (SS_LOG_T - log_c);
    for (u32 e = threadIdx.x; e < (u32)SS_T; e += SS_THREADS) {
        const u64 j = first + (e >> log_c);
        const u32 k = e & (C - 1);
        u64 v = ~0ull;
        if (j < n_runs) {
            const u32 d = list[j];
            const u64 o = offs[d];
            if (k < offs[d + 1] - o) v = tx_fwd(vals[o + k], tx);
        }
        sk[e] = v;
    }
    for (u32 w = 2; w <= C; w <<= 1) {
        for (u32 h = w >> 1; h > 0; h >>= 1) {
            __syncthreads();
            for (u32 t = threadIdx.x; t < (u32)SS_T / 2; t += SS_THREADS) {
                const u32 a = 2 * t - (t & (h - 1)), b = a + h;
                const bool up = w == C || !(a & w);        // the last merge of a block ascends; before it, halves alternate
                const u64 x = sk[a], y = sk[b];
                if ((x > y) == up) { sk[a] = y; sk[b] = x; }
            }
        }
    }
    __syncthreads();
    for (u32 e = threadIdx.x; e < (u32)SS_T; e += SS_THREADS) {
        const u64 j = first + (e >> log_c);
        if (j >= n_runs) break;
        const u32 d = list[j];
        const u64 o = offs[d];
        const u32 k = e & (C - 1);
        if (k < offs[d + 1] - o) vals[o + k] = tx_inv(sk[e], tx);
    }
}

// starts[r] = offs[list[r]], lens[r] = its run length (the large runs, r < n)
__global__ void seg_bounds_kernel(const u64 *__restrict__ offs, const u32 *__restrict__ list, u32 n, u64 *__restrict__ starts,
                                  u64 *__restrict__ lens)
{
    const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) { const u32 d = list[r]; starts[r] = offs[d]; lens[r] = offs[d + 1] - offs[d]; }
}

// Buffer position p of run r (pref[r] <= p < pref[r+1]) is vals[starts[r] + p - pref[r]].  gather: buf[p] = that value,
// rank[p] = r;  otherwise: that value = buf[p].
__global__ void seg_move_kernel(u64 *__restrict__ vals, const u64 *__restrict__ starts, const u64 *__restrict__ pref, u32 n_runs, u64 total,
                                u64 *__restrict__ buf, u64 *__restrict__ rank, int gather)
{
    const u64 st = (u64)gridDim.x * blockDim.x;
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += st) {
        u32 lo = 0, hi = n_runs;                             // the last r with pref[r] <= p
        while (hi - lo > 1) { const u32 m = (lo + hi) >> 1; if (pref[m] <= p) lo = m; else hi = m; }
        const u64 src = starts[lo] + (p - pref[lo]);
        if (gather) { buf[p] = vals[src]; rank[p] = lo; }
        else vals[src] = buf[p];
    }
}

__global__ void narrow_u32_kernel(const u64 *__restrict__ in, u64 n, u32 *__restrict__ out)
{
    const u64 st = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += st) out[i] = (u32)in[i];
}

}  // namespace vb
