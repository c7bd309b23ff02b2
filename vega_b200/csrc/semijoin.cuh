// Semi and anti joins of n sides (vb_semi_join_n*, engine.cu "semi and anti joins"): a key of side 0 is kept when every
// side of `required` has it and no side of `excluded` does.  The filter sides' keys share one presence dictionary
// (build_table OPK_DICT) with a u32 mask per slot, bit j set when side j has the slot's key.
//
//   presence_mark_kernel    mask[slot] |= side bits, through build_table's slot id per input row
//   presence_probe_kernel   one table_find per row of a lazy side 0: keep or drop the row
//   presence_count_kernel   one table_find per key of a grouped side 0's partition: its list length if kept, else 0
//   semi_str_count_kernel   the same over string sides, each filter side's key index probed by hash, then bytes
//
// The counts, scanned, are a one-side join plan (match row k = the key's own index), which the existing expand and
// gather kernels write out.
#pragma once
#include "kernels.cuh"
#include "strkeys.cuh"

namespace vb {

// The keep rule on a key's presence mask; no filter side keeps every key without a lookup
VB_D bool presence_keep(const Table &t, const u32 *mask, u64 key, u32 required, u32 excluded)
{
    if (!(required | excluded)) return true;
    u32 m = 0;
    if (t.keys) {
        const u32 s = table_find(t, key);
        if (s != 0xFFFFFFFFu) m = mask[s];
    }
    return (m & required) == required && !(m & excluded);
}

// The n rows of one filter input: mask[slot[i]] |= bits (the bits of every side that input is).  A slot whose bits are
// already set is not written again, so a hot key costs one atomic per warp that first meets it, not one per row.
__global__ void presence_mark_kernel(const u32 *__restrict__ slot, u64 n, u32 bits, u32 *mask)
{
    const u64 st = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += st) {
        u32 *m = mask + slot[i];
        if ((*m & bits) != bits) atomicOr(m, bits);
    }
}

// keep[i] = the rule on row i of a lazy side 0
__global__ void presence_probe_kernel(const u64 *__restrict__ keys, u64 n, Table t, const u32 *__restrict__ mask, u32 required,
                                      u32 excluded, unsigned char *__restrict__ keep)
{
    const u64 st = (u64)gridDim.x * blockDim.x;
    const u64 pol = policy_evict_first();
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += st)
        keep[i] = presence_keep(t, mask, ld_stream_u64(keys + i, pol), required, excluded) ? 1 : 0;
}

// Keys kb .. kb + nk of a grouped side 0 (CSR keys / offsets): cnt[k] = the key's list length if kept, else 0, and
// match[k] = kb + k, the key's row of a one-side plan
__global__ void presence_count_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ offs, u32 kb, u32 nk, Table t,
                                      const u32 *__restrict__ mask, u32 required, u32 excluded, u64 *__restrict__ cnt,
                                      u32 *__restrict__ match)
{
    const u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nk) return;
    const u32 e = kb + k;
    cnt[k] = presence_keep(t, mask, keys[e], required, excluded) ? offs[e + 1] - offs[e] : 0;
    match[k] = e;
}

// presence_count_kernel over string sides: side 0's key kb_0 + k is looked up in the key index of every side of
// `required | excluded` (a fingerprint match counts only with equal length and bytes)
__global__ void semi_str_count_kernel(const __grid_constant__ StrNSides a, const u64 *__restrict__ offs, u32 nk, u32 required,
                                      u32 excluded, u64 *__restrict__ cnt, u32 *__restrict__ match)
{
    const u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nk) return;
    const u32 e = a.kb[0] + k;
    const u64 h = a.hash[0][e], o = a.key_off[0][e], len = a.key_off[0][e + 1] - o;
    const unsigned char *key = a.bytes[0] + o;
    const u32 filter = required | excluded;
    u32 m = 0;
    for (u32 j = 1; j < a.n; ++j)
        if ((filter >> j & 1u) && str_side_find(a, j, h, key, len) != 0xFFFFFFFFu) m |= 1u << j;
    cnt[k] = (m & required) == required && !(m & excluded) ? offs[e + 1] - offs[e] : 0;
    match[k] = e;
}

}  // namespace vb
