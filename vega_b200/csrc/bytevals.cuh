// bytevals.cuh — byte-string values (a Rust `String` as its UTF-8 bytes, any `V: Serialize` as its bincode bytes) for
// the ops that move values without reading them: group_by_key, cogroup, the joins and the sort_by_key payload
// (engine.cu, "byte-string values").
//
// A map task's values are copied once into a store of the shuffle (offsets rebased to 0, bytes), and row i of map m
// enters the ordinary u64 map path as the reference ((m + 1) << 32) | i.  Grouping, joining and sorting move the
// references; the gather below turns any array of them back into Arrow-style offsets and bytes.  Reference 0 is never
// issued and gathers as the empty value (the 0 of a None slot).
#pragma once
#include "kernels.cuh"

namespace vb {

// one map task's value store on the device
struct ByteSrc {
    const u64 *offs;              // [n_rows + 1] from 0
    const unsigned char *bytes;
    u64 n_rows;                   // 0 for a map id never submitted
};

// refs[i] = tag | i, tag = (map_id + 1) << 32
__global__ void bytes_refs_kernel(u64 tag, u64 n, u64 *__restrict__ refs)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) refs[i] = tag | i;
}

// The store entry of a reference, or false for one the shuffle did not issue (reference 0 is handled by the callers)
__device__ __forceinline__ bool bytes_decode(u64 ref, const ByteSrc *__restrict__ tab, u32 n_map, u64 *m, u64 *row)
{
    *m = (ref >> 32) - 1;
    *row = ref & 0xFFFFFFFFull;
    return (ref >> 32) != 0 && *m < n_map && *row < tab[*m].n_rows;
}

// lens[i] = the length of value refs[i] (0 for reference 0); a reference the shuffle did not issue sets *bad
__global__ void bytes_len_kernel(const u64 *__restrict__ refs, u64 n, const ByteSrc *__restrict__ tab, u32 n_map,
                                 u64 *__restrict__ lens, u32 *bad)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    u32 f = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u64 ref = refs[i];
        u64 len = 0, m, row;
        if (ref) {
            if (bytes_decode(ref, tab, n_map, &m, &row)) len = tab[m].offs[row + 1] - tab[m].offs[row];
            else f = 1;
        }
        lens[i] = len;
    }
    if (f) atomicOr(bad, 1u);
}

// Gather: out_bytes[out_offs[i] .. out_offs[i + 1]) = value refs[i], for every i < n.
// Load balance over output bytes plus values (merge path): the items are the n value ends and the total output bytes,
// merged so that value i's end comes before byte j when it is <= j; tile b is items [b * GB_ITEMS, (b + 1) * GB_ITEMS).
// A tile therefore touches at most GB_ITEMS + 1 values and holds at most GB_ITEMS bytes, whatever the lengths are: one
// huge value is spread over many tiles, and long runs of empty values cost one item each.  A grid of resident CTAs
// walks the n_tiles tiles (tile b, b + gridDim.x, ...).  For each tile the CTA stages its values' output starts and
// source addresses in shared memory and writes its bytes in 16-byte-aligned
// chunks of the output: a chunk inside one value is assembled from aligned 4-byte source loads with funnel shifts and
// stored with one 16-byte store; a chunk that crosses value boundaries is assembled byte by byte; a chunk cut by the
// CTA's byte range (the first and last of each CTA) is written with byte stores, its other bytes belonging to the
// neighbouring CTA.
constexpr int GB_THREADS = 128;
constexpr u64 GB_ITEMS = (u64)GB_THREADS * 16;

// number of value ends among the first d merge items (value end A[i] = out_offs[i + 1] precedes byte j when A[i] <= j)
__device__ __forceinline__ u64 bytes_merge_path(const u64 *__restrict__ out_offs, u64 n, u64 total, u64 d)
{
    u64 lo = d > total ? d - total : 0, hi = d < n ? d : n;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if (out_offs[mid + 1] <= d - 1 - mid) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// 16 bytes starting at p (any alignment) as four little-endian words, from aligned 4-byte loads that each hold at
// least one of the bytes (so never past the allocation)
__device__ __forceinline__ uint4 bytes_load16(const unsigned char *p)
{
    const uintptr_t a = (uintptr_t)p;
    const u32 sh = (u32)(a & 3u);
    const u32 *w = (const u32 *)(a - sh);
    const u32 w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2), w3 = __ldg(w + 3);
    if (sh == 0) return make_uint4(w0, w1, w2, w3);
    const u32 w4 = __ldg(w + 4), s = 8 * sh;
    return make_uint4(__funnelshift_r(w0, w1, s), __funnelshift_r(w1, w2, s), __funnelshift_r(w2, w3, s), __funnelshift_r(w3, w4, s));
}

__global__ void __launch_bounds__(GB_THREADS)
bytes_gather_kernel(const u64 *__restrict__ refs, u64 n, const u64 *__restrict__ out_offs, u64 total, const ByteSrc *__restrict__ tab,
                    u32 n_map, unsigned char *__restrict__ out)
{
    __shared__ u64 s_start[GB_ITEMS + 2];   // output start of each staged value, then the end of the last one
    __shared__ u64 s_src[GB_ITEMS + 1];     // source address of output byte j of value k: s_src[k] + j
    __shared__ u64 s_cut[4];
    const u32 tid = threadIdx.x;
    const u64 n_tiles = (n + total + GB_ITEMS - 1) / GB_ITEMS;
    for (u64 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        __syncthreads();                           // the previous tile's shared state is no longer read
        if (tid < 2) {
            const u64 d = min((tile + tid) * GB_ITEMS, n + total);
            const u64 i = bytes_merge_path(out_offs, n, total, d);
            s_cut[2 * tid] = i;
            s_cut[2 * tid + 1] = d - i;
        }
        __syncthreads();
        const u64 i0 = s_cut[0], j0 = s_cut[1], i1 = s_cut[2], j1 = s_cut[3];
        if (j0 >= j1) continue;                    // only value ends (empty values): nothing to write
        const u64 last = min(i1, n - 1);           // bytes [j0, j1) belong to values i0 .. last
        const u32 cnt = (u32)(last - i0 + 1);
        for (u32 k = tid; k < cnt; k += GB_THREADS) {
            const u64 i = i0 + k, ref = refs[i], start = out_offs[i];
            u64 src = 0, m, row;
            if (ref && bytes_decode(ref, tab, n_map, &m, &row)) src = (u64)(uintptr_t)(tab[m].bytes + tab[m].offs[row]);
            s_start[k] = start;
            s_src[k] = src - start;
        }
        if (tid == 0) s_start[cnt] = out_offs[last + 1];
        __syncthreads();
        const uintptr_t base = (uintptr_t)out;
        const uintptr_t a0 = (base + j0) & ~(uintptr_t)15, a1 = base + j1;
        const u64 n_chunks = (a1 - a0 + 15) >> 4;
        for (u64 ch = tid; ch < n_chunks; ch += GB_THREADS) {
            const uintptr_t a = a0 + (ch << 4);
            const u64 ja = a - base;               // output byte at address a (may lie before j0 when a < base + j0)
            const u64 lo = a < base + j0 ? (u64)(base + j0 - a) : 0, hi = min((u64)16, (u64)(a1 - a));
            const u64 jlo = ja + lo;               // first byte of the chunk this CTA writes
            u32 lo_k = 0, hi_k = cnt;              // the staged value holding jlo: the last k with s_start[k] <= jlo
            while (hi_k - lo_k > 1) {
                const u32 mid = (lo_k + hi_k) >> 1;
                if (s_start[mid] <= jlo) lo_k = mid;
                else hi_k = mid;
            }
            u32 k = lo_k;
            if (lo == 0 && hi == 16 && s_start[k + 1] >= ja + 16) {
                *(uint4 *)a = bytes_load16((const unsigned char *)(uintptr_t)(s_src[k] + ja));
                continue;
            }
            if (lo == 0 && hi == 16) {
                u32 w[4] = {0, 0, 0, 0};
                for (u32 b = 0; b < 16; ++b) {
                    const u64 j = ja + b;
                    while (j >= s_start[k + 1]) ++k;
                    w[b >> 2] |= (u32)*(const unsigned char *)(uintptr_t)(s_src[k] + j) << (8 * (b & 3));
                }
                *(uint4 *)a = make_uint4(w[0], w[1], w[2], w[3]);
                continue;
            }
            for (u64 b = lo; b < hi; ++b) {
                const u64 j = ja + b;
                while (j >= s_start[k + 1]) ++k;
                ((unsigned char *)a)[b] = *(const unsigned char *)(uintptr_t)(s_src[k] + j);
            }
        }
    }
}

}  // namespace vb
