// strkeys.cuh — byte-string keys (Rust `String` / `&str`): the hash the reference's HashPartitioner gives them, the
// per-shuffle dictionary of distinct keys, and the seal-side kernels of the string-key shuffle (engine.cu,
// "string keys").
//
// A key is a byte run of a caller column (Arrow-style offsets + bytes).  `impl Hash for str` writes the bytes and then
// one 0xFF byte; the buffering MetroHasher hashes that stream with MetroHash64_1 (seed 0) at finish.  The suffix is
// never materialised: every word of the stream is assembled from aligned 8-byte loads of the key and the 0xFF byte.
// A shuffle of byte-slice keys (`Vec<u8>` and kin) hashes `le64(len) ‖ key` instead, built the same way; everything
// else (equality, order, the dictionary) is the same for both kinds.
//
// Dictionary: dense entries (hash, arena offset, length) indexed by a u32 entry id, an arena holding each distinct
// key's bytes once, and an open-addressing index of 4-slot buckets (fingerprint, entry id).  Entries are the source of
// truth; the index is rebuilt from them whenever it has to grow.
#pragma once
#include "kernels.cuh"

namespace vb {

// Bytes [pos, pos + n) of p (1 <= n <= 8) as a little-endian word.  On the device: one or two aligned 8-byte loads,
// never one of an aligned word that holds none of the requested bytes (so never past the end of the allocation).
// CG: read through L2 only (arena bytes another thread of the same kernel may have just published).
template <bool CG>
VB_HD u64 load_le(const unsigned char *p, u64 pos, u32 n)
{
#ifdef __CUDA_ARCH__
    const uintptr_t a = (uintptr_t)(p + pos);
    const u32 sh = (u32)(a & 7u);
    const unsigned long long *w = (const unsigned long long *)(a - sh);
    u64 v = (CG ? __ldcg(w) : __ldg(w)) >> (8 * sh);
    if (sh + n > 8) v |= (u64)(CG ? __ldcg(w + 1) : __ldg(w + 1)) << (64 - 8 * sh);
#else
    u64 v = 0;
    for (u32 i = 0; i < n; ++i) v |= (u64)p[pos + i] << (8 * i);
#endif
    return n < 8 ? v & ((1ull << (8 * n)) - 1) : v;
}

// Bytes [pos, pos + n) of the hashed stream `key[0..len) ‖ 0xFF` (pos + n <= len + 1).
VB_HD u64 str_word(const unsigned char *p, u64 len, u64 pos, u32 n)
{
    const u32 take = pos >= len ? 0u : (u32)((len - pos) < n ? (len - pos) : n);
    u64 v = take ? load_le<false>(p, pos, take) : 0ull;
    if (take < n) v |= 0xFFull << (8 * take);
    return v;
}

// How a shuffle's keys hash (vb_shuffle_set_str_key): as a Rust `String` / `&str`, or as a byte slice (`Vec<u8>`,
// `&[u8]`, `Box<[u8]>`, `[u8; N]`), whose `Hash` writes the length as a usize and then the bytes.
enum { STRKEY_STR = 0, STRKEY_BYTES = 1 };

// Bytes [pos, pos + n) of the hashed stream `le64(len) ‖ key[0..len)` (pos + n <= len + 8).  The stream is at least 8
// bytes long, so MetroHash64_1 reads its first word whole: pos 0 is always the length word, and every later read lies
// in the key at pos - 8.
VB_HD u64 bytes_word(const unsigned char *p, u64 len, u64 pos, u32 n)
{
    return pos == 0 ? len : load_le<false>(p, pos - 8, n);
}

template <int KIND>
VB_HD u64 key_word(const unsigned char *p, u64 len, u64 pos, u32 n)
{
    static_assert(KIND == STRKEY_STR || KIND == STRKEY_BYTES, "String or byte-slice keys");
    return KIND == STRKEY_STR ? str_word(p, len, pos, n) : bytes_word(p, len, pos, n);
}

// MetroHash64_1(stream, seed 0) as the reference's MetroHasher (fasthash 0.4.0) computes it at finish.  KIND STRKEY_STR:
// the stream `str::hash` writes, key ‖ 0xFF; STRKEY_BYTES: the one `<[u8]>::hash` writes, le64(len) ‖ key.
template <int KIND>
VB_HD u64 metro64_1_key(const unsigned char *p, u64 len)
{
    const u64 k0 = 0xC83A91E1ull, k1 = 0x8648DBDBull, k2 = 0x7BDEC03Bull, k3 = 0x2F5870A5ull;
    const u64 n = len + (KIND == STRKEY_STR ? 1 : 8);
    u64 h = (k2 * k0) + n;
    u64 pos = 0;
    if (n >= 32) {
        u64 v0 = h, v1 = h, v2 = h, v3 = h;
        do {
            v0 += key_word<KIND>(p, len, pos, 8) * k0;      v0 = rotr64(v0, 29) + v2;
            v1 += key_word<KIND>(p, len, pos + 8, 8) * k1;  v1 = rotr64(v1, 29) + v3;
            v2 += key_word<KIND>(p, len, pos + 16, 8) * k2; v2 = rotr64(v2, 29) + v0;
            v3 += key_word<KIND>(p, len, pos + 24, 8) * k3; v3 = rotr64(v3, 29) + v1;
            pos += 32;
        } while (pos + 32 <= n);
        v2 ^= rotr64(((v0 + v3) * k0) + v1, 33) * k1;
        v3 ^= rotr64(((v1 + v2) * k1) + v0, 33) * k0;
        v0 ^= rotr64(((v0 + v2) * k0) + v3, 33) * k1;
        v1 ^= rotr64(((v1 + v3) * k1) + v2, 33) * k0;
        h += v0 ^ v1;
    }
    if (n - pos >= 16) {
        u64 a = h + key_word<KIND>(p, len, pos, 8) * k0;     a = rotr64(a, 33) * k1;
        u64 b = h + key_word<KIND>(p, len, pos + 8, 8) * k1; b = rotr64(b, 33) * k2;
        a ^= rotr64(a * k0, 35) + b;
        b ^= rotr64(b * k3, 35) + a;
        h += b;
        pos += 16;
    }
    if (n - pos >= 8) { h += key_word<KIND>(p, len, pos, 8) * k3; h ^= rotr64(h, 33) * k1; pos += 8; }
    if (n - pos >= 4) { h += key_word<KIND>(p, len, pos, 4) * k3; h ^= rotr64(h, 15) * k1; pos += 4; }
    if (n - pos >= 2) { h += key_word<KIND>(p, len, pos, 2) * k3; h ^= rotr64(h, 13) * k1; pos += 2; }
    if (n - pos >= 1) { h += key_word<KIND>(p, len, pos, 1) * k3; h ^= rotr64(h, 25) * k1; }
    h ^= rotr64(h, 33);
    h *= k0;
    h ^= rotr64(h, 33);
    return h;
}

// MetroHash64_1(key ‖ 0xFF, seed 0): `str::hash` fed to the reference's MetroHasher.
VB_HD u64 metro64_1_str(const unsigned char *p, u64 len) { return metro64_1_key<STRKEY_STR>(p, len); }
// MetroHash64_1(le64(len) ‖ key, seed 0): `<[u8]>::hash` fed to the same hasher.
VB_HD u64 metro64_1_bytes(const unsigned char *p, u64 len) { return metro64_1_key<STRKEY_BYTES>(p, len); }

constexpr u32 STR_UNPUBLISHED = 0xFFFFFFFFu;   // index slot claimed, entry id not written yet (or slot empty)
constexpr u32 STR_MAX_PROBE = 64;              // buckets probed before a call gives up (str_encode: grow or lift)

struct StrDict {
    u64 *fp;                  // [cap] index fingerprints: 0 = empty slot
    u32 *id;                  // [cap] entry id of the slot
    u32 log_cap;              // cap = 1 << log_cap slots, 4 per 32-byte bucket of fingerprints
    u64 fp_mask;              // bits of the hash kept in the fingerprint (all of them unless VEGA_B200_STR_FP_BITS)
    u64 *e_hash;              // [entries] full 64-bit hash
    u64 *e_off;               // [entries] offset of the key's bytes in the arena
    u32 *e_len;               // [entries] key length in bytes
    unsigned char *arena;     // each distinct key's bytes, once
};

struct StrCtl {
    u32 abort;                     // the index is too full or a probe ran too long: the host grows it or lifts the probe limit, and reruns the call
    u32 n_entries;                 // entries in use (persistent across calls)
    unsigned long long n_arena;    // arena bytes in use (persistent across calls)
};

VB_HD u64 str_fp(u64 h, u64 mask)
{
    const u64 f = h & mask;
    return f ? f : 1ull;           // 0 marks an empty slot
}
// The probe starts at the bucket of the FULL hash: a masked fingerprint shortens only the compare, not the spread.
VB_HD u64 str_bucket(u64 h, u32 log_cap) { return log_cap > 2 ? (h >> (66 - log_cap)) : 0ull; }

VB_D u32 ld_acquire_u32(const u32 *p)
{
    u32 r;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
VB_D void st_release_u32(u32 *p, u32 v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

VB_D bool str_equal(const unsigned char *key, const unsigned char *stored, u64 len)
{
    for (u64 pos = 0; pos < len; pos += 8) {
        const u32 n = (len - pos) < 8 ? (u32)(len - pos) : 8u;
        if (load_le<false>(key, pos, n) != load_le<true>(stored, pos, n)) return false;
    }
    return true;
}

// One thread per row: hash the key, find or create its dictionary entry, write the entry id.  Key i is
// bytes[offs[i] - base .. offs[i + 1] - base).  Entries and arena are reserved by the host for the worst case of the
// call, so only the index can overflow; that is decided BEFORE a slot is claimed (load or probe length), so a claimed
// slot is always published and no thread waits on one forever.  An aborted call is rerun whole after the index grows
// or the probe limit is lifted: rows already encoded find the same entries again.  max_probe (<= the bucket count, set
// by str_encode): buckets a probe walks before it gives up.  A walk of every bucket that finds neither the key nor an
// empty slot means the index is full, so the host, which sees n_entries >= max_entries, grows it for load.  KIND: the
// shuffle's key hash (STRKEY_*).  The byte-slice hash asks ptxas for 4 blocks per SM: left to its default it holds 40
// registers and spills the row index (8 bytes); the String instantiation keeps the bare bound (0: none), and with it
// the code it always had.
template <int KIND>
__global__ void __launch_bounds__(256, KIND == STRKEY_BYTES ? 4 : 0) str_encode_kernel(const u64 *__restrict__ offs, const unsigned char *__restrict__ bytes, u64 base,
                                                         u64 n, StrDict d, StrCtl *ctl, u32 max_entries, u32 max_probe,
                                                         u32 *__restrict__ ids_out)
{
    const u64 nb = 1ull << (d.log_cap - 2);
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (ld_volatile_u32(&ctl->abort)) return;
        const u64 o0 = offs[i], len = offs[i + 1] - o0;
        const unsigned char *p = bytes + (o0 - base);
        const u64 h = metro64_1_key<KIND>(p, len);
        const u64 f = str_fp(h, d.fp_mask);
        u64 b = str_bucket(h, d.log_cap);
        u32 found = STR_UNPUBLISHED;
        for (u32 probe = 0; probe < max_probe && found == STR_UNPUBLISHED; ++probe, b = (b + 1) & (nb - 1)) {
            for (u32 j = 0; j < BUCKET; ++j) {
                const u64 slot = BUCKET * b + j;
                u64 cur = __ldcg((const unsigned long long *)&d.fp[slot]);
                if (cur == 0) {
                    if (ld_volatile_u32(&ctl->n_entries) >= max_entries) { atomicExch(&ctl->abort, 1u); return; }
                    cur = atomicCAS((unsigned long long *)&d.fp[slot], 0ull, (unsigned long long)f);
                    if (cur == 0) {                          // claimed: create the entry, then publish its id
                        const u32 e = atomicAdd(&ctl->n_entries, 1u);
                        const u64 ao = atomicAdd(&ctl->n_arena, (unsigned long long)len);
                        for (u64 k = 0; k < len; ++k) d.arena[ao + k] = p[k];
                        d.e_hash[e] = h;
                        d.e_off[e] = ao;
                        d.e_len[e] = (u32)len;
                        __threadfence();
                        st_release_u32(&d.id[slot], e);
                        found = e;
                        break;
                    }
                }
                if (cur == f) {                              // same fingerprint: equal only if the bytes are
                    u32 e, ns = 32;
                    while ((e = ld_acquire_u32(&d.id[slot])) == STR_UNPUBLISHED) {
                        __nanosleep(ns);
                        if (ns < 1024) ns *= 2;
                    }
                    if (__ldcg(&d.e_len[e]) == len && str_equal(p, d.arena + __ldcg((const unsigned long long *)&d.e_off[e]), len)) {
                        found = e;
                        break;
                    }
                }
            }
        }
        if (found == STR_UNPUBLISHED) { atomicExch(&ctl->abort, 1u); return; }
        ids_out[i] = found;
    }
}

// Re-insert entries [0, n) into an empty index (all keys distinct: no compares).
__global__ void str_index_rebuild_kernel(StrDict d, u32 n, StrCtl *ctl)
{
    const u64 nb = 1ull << (d.log_cap - 2);
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
        const u64 h = d.e_hash[e], f = str_fp(h, d.fp_mask);
        u64 b = str_bucket(h, d.log_cap);
        bool placed = false;
        for (u64 probe = 0; probe < nb && !placed; ++probe, b = (b + 1) & (nb - 1))
            for (u32 j = 0; j < BUCKET; ++j)
                if (atomicCAS((unsigned long long *)&d.fp[BUCKET * b + j], 0ull, (unsigned long long)f) == 0ull) {
                    d.id[BUCKET * b + j] = (u32)e;
                    placed = true;
                    break;
                }
        if (!placed) atomicExch(&ctl->abort, 1u);
    }
}

// Key offsets of a device-resident call: flags bit 0 = decreasing or beyond n_bytes, bit 1 = a key of 2^32 bytes or more.
__global__ void str_check_offsets_kernel(const u64 *__restrict__ offs, u64 n, u64 n_bytes, u32 *flags)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    u32 f = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) {
        const u64 o = offs[i];
        if (o > n_bytes) f |= 1u;
        if (i < n) {
            const u64 nx = offs[i + 1];
            if (nx < o) f |= 1u;
            else if (nx - o >= (1ull << 32)) f |= 2u;
        }
    }
    if (f) atomicOr(flags, f);
}

// ---- seal ------------------------------------------------------------------------------------------------------
__global__ void str_mark_live_kernel(const u32 *__restrict__ ids, u64 n, u32 *__restrict__ live)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) live[ids[i]] = 1u;
}

// Partition of every live entry (h % n_reduce) and the per-partition key counts.
__global__ void str_part_count_kernel(const u64 *__restrict__ e_hash, const u32 *__restrict__ live, u32 n, FastMod fm,
                                      u32 *__restrict__ part_of, u32 *__restrict__ cnt)
{
    const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n || !live[e]) return;
    const u32 p = fastmod(e_hash[e], fm);
    part_of[e] = p;
    atomicAdd(&cnt[p], 1u);
}

// Partition-major dense ids (order inside a partition unspecified) and each dense key's length.
__global__ void str_dense_kernel(const u32 *__restrict__ live, const u32 *__restrict__ part_of, u32 n, const u64 *__restrict__ part_base,
                                 u32 *__restrict__ cursor, const u32 *__restrict__ e_len, u32 *__restrict__ dense_of_entry,
                                 u32 *__restrict__ entry_of_dense, u64 *__restrict__ klen)
{
    const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    if (!live[e]) { dense_of_entry[e] = STR_UNPUBLISHED; return; }
    const u32 p = part_of[e];
    const u32 dn = (u32)part_base[p] + atomicAdd(&cursor[p], 1u);
    dense_of_entry[e] = dn;
    entry_of_dense[dn] = e;
    klen[dn] = e_len[e];
}

// Key bytes in dense order: one warp per key.
__global__ void str_gather_bytes_kernel(const u32 *__restrict__ entry_of_dense, u32 n, const u64 *__restrict__ e_off,
                                        const u64 *__restrict__ key_off, const unsigned char *__restrict__ arena, unsigned char *__restrict__ out)
{
    const u64 w = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= n) return;
    const u64 src = e_off[entry_of_dense[w]], dst = key_off[w], len = key_off[w + 1] - dst;
    for (u64 k = lane_id(); k < len; k += 32) out[dst + k] = arena[src + k];
}

__global__ void str_fill_kernel(u64 *__restrict__ a, u64 n, u64 v)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) a[i] = v;
}

// One RED per distinct id of each warp into acc[dense id]: lanes of a warp that carry the same id (match-any) are
// combined first, so a frequent key costs one RED per warp, not per row.  OPK_COUNT counts rows (vals unused);
// TX / NaN handling as hash_agg_kernel's: values enter MIN/MAX order-transformed, an f64 NaN becomes the identity.
template <int OPK, int TX>
__global__ void __launch_bounds__(256) str_reduce_kernel(const u32 *__restrict__ ids, const u64 *__restrict__ vals, u64 n,
                                                         const u32 *__restrict__ dense_of_entry, u64 *__restrict__ acc)
{
    constexpr int RED = OPK == OPK_COUNT ? OPK_ADD_U64 : OPK;
    constexpr bool NAN_IS_IDENTITY = (TX == TX_F64) && (OPK == OPK_MIN_U64 || OPK == OPK_MAX_U64);
    const u32 lane = lane_id();
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 w = warp0; w < n; w += stride) {
        const u64 i = w + lane;
        const bool ok = i < n;
        u32 dn = STR_UNPUBLISHED;
        u64 v = OPK == OPK_COUNT ? 1ull : 0ull;
        if (ok) {
            dn = dense_of_entry[ids[i]];
            if (OPK != OPK_COUNT) {
                v = vals[i];
                if (NAN_IS_IDENTITY && (v & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull) v = op_identity(OPK);
                else v = tx_fwd(v, TX);
            }
        }
        const u32 peers = __match_any_sync(0xFFFFFFFFu, dn);
        const bool lead = (__ffs(peers) - 1) == (int)lane;
        if (!__all_sync(0xFFFFFFFFu, peers == (1u << lane))) {       // some id repeats in this warp: fold into its leader
            for (u32 j = 0; j < 32; ++j) {
                const u64 x = __shfl_sync(0xFFFFFFFFu, v, j);
                if (!lead || j == lane || !((peers >> j) & 1u)) continue;
                if (RED == OPK_ADD_U64) v += x;
                else if (RED == OPK_ADD_F64) v = (u64)__double_as_longlong(__longlong_as_double((long long)v) + __longlong_as_double((long long)x));
                else if (RED == OPK_MIN_U64) v = x < v ? x : v;
                else v = x > v ? x : v;
            }
        }
        if (ok && lead) op_red<RED>(&acc[dn], v);
    }
}

// v op x for a run-time reduce op (warp-uniform); str_reduce_kernel's fold with the op taken from an AccSpec
VB_D u64 op_fold_rt(int opk, u64 v, u64 x)
{
    switch (opk) {
    case OPK_ADD_F64: return (u64)__double_as_longlong(__longlong_as_double((long long)v) + __longlong_as_double((long long)x));
    case OPK_MIN_U64: return x < v ? x : v;
    case OPK_MAX_U64: return x > v ? x : v;
    default: return v + x;                                        // OPK_ADD_U64, and a COUNT's ones
    }
}

// combine_by_key over dense ids: str_reduce_kernel with the accumulator list of `sp` (acc is [sp.n][D], each column
// initialised to its op's identity).  One match-any per warp on the dense id; then, accumulator by accumulator (a
// run-time loop: hash_agg_multi spilled when unrolled), load the value, ma_prep it, fold it into the id's leader lane
// and issue one RED.  IN_SOA: value src(a) of map row i from cols.c[src] (a COUNT counts ones); IN_ACCS: partial a of
// received row i at cols.c[0][a * cols.stride + i], merged with the merge spec (COUNT as ADD).
template <int IN>
__global__ void __launch_bounds__(256) str_reduce_multi_kernel(const u32 *__restrict__ ids, MaCols cols, u64 n,
                                                               const u32 *__restrict__ dense_of_entry, AccSpec sp, u64 D, u64 *__restrict__ acc)
{
    static_assert(IN == IN_SOA || IN == IN_ACCS, "map rows or received partials");
    const u32 lane = lane_id();
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 ops = sp.op, txs = sp.tx, srcs = sp.src;
    const int n_acc = (int)sp.n;
    for (u64 w = warp0; w < n; w += stride) {
        const u64 i = w + lane;
        const bool ok = i < n;
        const u32 dn = ok ? dense_of_entry[ids[i]] : STR_UNPUBLISHED;
        const u32 peers = __match_any_sync(0xFFFFFFFFu, dn);
        const bool lead = (__ffs(peers) - 1) == (int)lane;
        const bool distinct = __all_sync(0xFFFFFFFFu, peers == (1u << lane));
#pragma unroll 1
        for (int a = 0; a < n_acc; ++a) {
            const int op = spec_at(ops, a), red = merge_op(op);
            u64 v = 0;
            if (ok) {
                if constexpr (IN == IN_ACCS) {
                    v = ma_prep(cols.c[0][(u64)a * cols.stride + i], op, spec_at(txs, a));
                } else if (op == OPK_COUNT) {
                    v = 1;
                } else {
                    const int src = spec_at(srcs, a);
                    const u64 *col = cols.c[0];
#pragma unroll
                    for (int c = 1; c < MA_MAX_COLS; ++c)
                        if (src == c) col = cols.c[c];
                    v = ma_prep(col[i], op, spec_at(txs, a));
                }
            }
            if (!distinct) {                                          // some id repeats in this warp: fold into its leader
                for (u32 j = 0; j < 32; ++j) {
                    const u64 x = __shfl_sync(0xFFFFFFFFu, v, j);
                    if (!lead || j == lane || !((peers >> j) & 1u)) continue;
                    v = op_fold_rt(red, v, x);
                }
            }
            if (ok && lead) op_red_rt(&acc[(u64)a * D + dn], red, v);
        }
    }
}

// ---- across ranks (engine.cu, "string keys across ranks") --------------------------------------------------------
// The wire columns carry a u32 length per key and, for GROUP, a u32 value count per key, so that the host can
// concatenate slices of them without rebasing anything.

// out[i] = off[i + 1] - off[i] as u32: key lengths from key byte offsets, value counts from CSR offsets
__global__ void str_diff_u32_kernel(const u64 *__restrict__ off, u64 n, u32 *__restrict__ out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (u32)(off[i + 1] - off[i]);
}

// out[i] = in[i]: received lengths / counts widened for exclusive_scan_u64
__global__ void str_widen_u32_kernel(const u32 *__restrict__ in, u64 n, u64 *__restrict__ out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = in[i];
}

// Imported GROUP rows: row j belongs to the received key k with voff[k] <= j < voff[k + 1] (voff: the scanned value
// counts, voff[nk] = n), found by a binary search per row, and gets that key's entry id.  A key with no values is
// skipped by the search (the last k with voff[k] <= j is the one whose run holds j).
__global__ void str_expand_ids_kernel(const u64 *__restrict__ voff, u64 nk, const u32 *__restrict__ key_ids, u64 n,
                                      u32 *__restrict__ row_ids)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        u64 lo = 0, hi = nk;
        while (hi - lo > 1) {
            const u64 mid = (lo + hi) >> 1;
            if (voff[mid] <= j) lo = mid; else hi = mid;
        }
        row_ids[j] = key_ids[lo];
    }
}

// ---- cogroup and join of string GROUP shuffles (engine.cu, "cogroup and join of string keys") --------------------
// Seal drops the dictionary, so a side read by a cogroup or join first gets a key index of its result keys: each dense
// key's hash, and an index of StrDict's layout (4-slot buckets of fingerprints, parallel dense key ids).  The N-way
// plan (cogroup_n_*) then runs unchanged on the match matrix; only the probe, and the output keys, read bytes.
struct StrNSides {
    const u64 *fp[CGN_MAX_SIDES];                 // index fingerprints, 0 = empty slot; NULL: the side has no keys
    const u32 *id[CGN_MAX_SIDES];                 // dense key id of each index slot
    u32 log_cap[CGN_MAX_SIDES];
    const u64 *hash[CGN_MAX_SIDES];               // [n_keys] hash of each dense key
    const u64 *key_off[CGN_MAX_SIDES];            // [n_keys + 1] byte offset of each dense key (StrState::key_off)
    const unsigned char *bytes[CGN_MAX_SIDES];    // the keys' bytes (StrState::key_bytes)
    u32 kb[CGN_MAX_SIDES];                        // the partition's first key on each side
    u64 fp_mask;
    u32 n;
};

// One thread per dense key: hash its bytes, then claim a slot.  The keys are distinct, so nothing is compared; the
// index is sized for load <= 0.6, so every key finds a free slot.  KIND: the shuffle's key hash, as str_encode_kernel's.
template <int KIND>
__global__ void str_key_index_kernel(const u64 *__restrict__ key_off, const unsigned char *__restrict__ bytes, u32 n, u64 *fp,
                                     u32 *__restrict__ id, u32 log_cap, u64 fp_mask, u64 *__restrict__ hash)
{
    const u64 nb = 1ull << (log_cap - 2);
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
        const u64 o = key_off[e];
        const u64 h = metro64_1_key<KIND>(bytes + o, key_off[e + 1] - o), f = str_fp(h, fp_mask);
        hash[e] = h;
        u64 b = str_bucket(h, log_cap);
        bool placed = false;
        for (u64 probe = 0; probe < nb && !placed; ++probe, b = (b + 1) & (nb - 1))
            for (u32 j = 0; j < BUCKET; ++j)
                if (atomicCAS((unsigned long long *)&fp[BUCKET * b + j], 0ull, (unsigned long long)f) == 0ull) {
                    id[BUCKET * b + j] = (u32)e;
                    placed = true;
                    break;
                }
    }
}

// Side j's dense key id of the key (h, key[0..len)), or 0xFFFFFFFF: a fingerprint match is a key only if its length
// and bytes are equal too; an empty slot ends the probe.
VB_D u32 str_side_find(const StrNSides &a, u32 j, u64 h, const unsigned char *key, u64 len)
{
    if (!a.fp[j]) return 0xFFFFFFFFu;
    const u64 nb = 1ull << (a.log_cap[j] - 2), f = str_fp(h, a.fp_mask);
    u64 b = str_bucket(h, a.log_cap[j]);
    for (u64 probe = 0; probe < nb; ++probe, b = (b + 1) & (nb - 1))
        for (u32 s = 0; s < BUCKET; ++s) {
            const u64 slot = BUCKET * b + s, cur = a.fp[j][slot];
            if (cur == 0) return 0xFFFFFFFFu;
            if (cur != f) continue;
            const u32 e = a.id[j][slot];
            const u64 o = a.key_off[j][e];
            if (a.key_off[j][e + 1] - o == len && str_equal(key, a.bytes[j] + o, len)) return e;
        }
    return 0xFFFFFFFFu;
}

// cogroup_n_probe_kernel over string sides: the same rows, flags and lidx, with the key looked up by hash and bytes.
// A key's hash decides its partition, so a key found through a side's shuffle-wide index is in the same partition.
__global__ void cogroup_n_str_probe_kernel(const __grid_constant__ StrNSides a, u32 i, u32 nk, u32 *__restrict__ rows,
                                           unsigned char *__restrict__ flag, u64 *__restrict__ lidx)
{
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nk) return;
    const u32 e = a.kb[i] + t;
    const u64 h = a.hash[i][e], o = a.key_off[i][e], len = a.key_off[i][e + 1] - o;
    const unsigned char *key = a.bytes[i] + o;
    for (u32 j = 0; j < a.n; ++j) {
        const u32 m = j == i ? e : str_side_find(a, j, h, key, len);
        if (j < i && m != 0xFFFFFFFFu) { flag[t] = 0; return; }     // an earlier side already gave this key
        if (i == 0 || j > i) rows[(u64)t * a.n + j] = m;
    }
    if (i) { flag[t] = 1; lidx[t] = t; }
}

// The side an output key's bytes come from: the first side of its match row that has it.
VB_D u32 str_key_owner(const u32 *row, u32 n)
{
    u32 j = 0;
    while (j + 1 < n && row[j] == 0xFFFFFFFFu) ++j;
    return j;
}

// len[o] = the byte length of output key sel[o] (sel NULL: o) of the plan
__global__ void str_n_key_len_kernel(const __grid_constant__ StrNSides a, const u32 *__restrict__ match, const u64 *__restrict__ sel,
                                     u64 nk, u64 *__restrict__ len)
{
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nk) return;
    const u32 *row = match + (sel ? sel[o] : o) * a.n;
    const u32 j = str_key_owner(row, a.n);
    len[o] = a.key_off[j][row[j] + 1] - a.key_off[j][row[j]];
}

// Output key o's bytes at out[off[o] .. off[o + 1]): one warp per key, as str_gather_bytes_kernel
__global__ void str_n_key_bytes_kernel(const __grid_constant__ StrNSides a, const u32 *__restrict__ match, const u64 *__restrict__ sel,
                                       u64 nk, const u64 *__restrict__ off, unsigned char *__restrict__ out)
{
    const u64 w = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= nk) return;
    const u32 *row = match + (sel ? sel[w] : w) * a.n;
    const u32 j = str_key_owner(row, a.n);
    const unsigned char *src = a.bytes[j] + a.key_off[j][row[j]];
    const u64 dst = off[w], len = off[w + 1] - dst;
    for (u64 k = lane_id(); k < len; k += 32) out[dst + k] = src[k];
}

// flag[o] = 1 for a join plan key with rows (pos[o + 1] > pos[o], pos[nk] read as total), idx[o] = o
__global__ void str_join_keep_kernel(const u64 *__restrict__ pos, u64 nk, u64 total, unsigned char *__restrict__ flag,
                                     u64 *__restrict__ idx)
{
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nk) return;
    flag[o] = (o + 1 < nk ? pos[o + 1] : total) > pos[o];
    idx[o] = o;
}

// ---- sort_by_key over string keys (engine.cu, "sort_by_key over string keys") -----------------------------------
// The distinct keys are ordered by rounds over 7-byte big-endian words.  Every active entry carries `start`, the first
// rank of the group of keys it still ties with; round w stably sorts the active entries by (start, its round-w key)
// with the LSD radix passes, then gives each run of equal (start, key) the rank start + (run head − group head).  A
// run of one is final; a longer run can only hold keys that go on past the word, and stays active for round w + 1.

// Round w's sort key of a key of `len` bytes at arena + off: bytes [7w, 7w + 7) big-endian in bits 63..8 (zero past
// the key's end), and min(len − 7w, 8) in bits 7..0 (0..7: the key ends inside the word; 8: it goes on).  Comparing
// these u64s compares the keys' bytes from 7w on, a proper prefix first, so one sort key per round carries both.
VB_D u64 str_sort_key(const unsigned char *arena, u64 off, u32 len, u32 w)
{
    const u64 pos = 7ull * w;
    const u64 rest = len > pos ? len - pos : 0ull;
    const u64 le = rest ? load_le<false>(arena + off, pos, rest < 7 ? (u32)rest : 7u) : 0ull;   // byte k at bits 8k
    const u64 be = ((u64)__byte_perm((u32)le, 0u, 0x0123u) << 32) | __byte_perm((u32)(le >> 32), 0u, 0x0123u);
    return be | (rest < 8 ? rest : 8ull);
}

// keys[i] = key_of[act[i]] = the round-w sort key of active entry act[i]
__global__ void str_sort_word_kernel(const u64 *__restrict__ act, u64 na, const u64 *__restrict__ e_off, const u32 *__restrict__ e_len,
                                     const unsigned char *__restrict__ arena, u32 w, u64 *__restrict__ keys, u64 *__restrict__ key_of)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < na; i += stride) {
        const u64 e = act[i];
        const u64 k = str_sort_key(arena, e_off[e], e_len[e], w);
        keys[i] = k;
        key_of[e] = k;
    }
}

// keys[i] = start_of[se[i]]: the group starts in the order of the key passes, for the passes over the start
__global__ void str_sort_start_kernel(const u64 *__restrict__ se, u64 na, const u32 *__restrict__ start_of, u64 *__restrict__ keys)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < na; i += stride) keys[i] = start_of[se[i]];
}

// Over the sorted active entries se: head[i] = 1 where a run of equal (start, key) begins; gpos[start] = the position
// where the group of `start` begins.
__global__ void str_sort_heads_kernel(const u64 *__restrict__ se, u64 na, const u64 *__restrict__ key_of, const u32 *__restrict__ start_of,
                                      u64 *__restrict__ head, u32 *__restrict__ gpos)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < na; i += stride) {
        const u64 e = se[i];
        const u32 g = start_of[e];
        bool gh = true, rh = true;
        if (i) {
            const u64 p = se[i - 1];
            gh = start_of[p] != g;
            rh = gh || key_of[p] != key_of[e];
        }
        head[i] = rh;
        if (gh) gpos[g] = (u32)i;
    }
}

// runpos[hx[i]] = i for every run head (hx: the exclusive scan of head, i.e. the run's index)
__global__ void str_sort_runpos_kernel(const u64 *__restrict__ head, const u64 *__restrict__ hx, u64 na, u32 *__restrict__ runpos)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < na; i += stride)
        if (head[i]) runpos[hx[i]] = (u32)i;
}

// Each sorted entry's new start: start + (its run head's position − its group head's position).  A run of one entry
// is final (rank_of = the new start, stay = 0); the entries of a longer run keep the new start and stay active.
// *n_runs: the number of runs (the total of the head scan).
__global__ void str_sort_split_kernel(const u64 *__restrict__ se, const u64 *__restrict__ head, const u64 *__restrict__ hx, u64 na,
                                      const u32 *__restrict__ runpos, const u64 *__restrict__ n_runs, const u32 *__restrict__ gpos,
                                      u32 *__restrict__ start_of, u32 *__restrict__ rank_of, u64 *__restrict__ stay)
{
    const u64 nr = *n_runs;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < na; i += stride) {
        const u64 e = se[i];
        const u64 r = hx[i] + head[i] - 1;
        const u32 rp = runpos[r];
        const u64 rend = r + 1 < nr ? runpos[r + 1] : na;
        const u32 g = start_of[e];
        const u32 ns = g + (rp - gpos[g]);
        if (rend - rp == 1) {
            rank_of[e] = ns;
            stay[i] = 0;
        } else {
            start_of[e] = ns;
            stay[i] = 1;
        }
    }
}

// out[pos[i]] = src[i] (src NULL: i) where flag[i]; pos is the exclusive scan of flag: a stable compaction
__global__ void str_compact_kernel(const u64 *__restrict__ flag, const u64 *__restrict__ pos, const u64 *__restrict__ src, u64 n,
                                   u64 *__restrict__ out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        if (flag[i]) out[pos[i]] = src ? src[i] : i;
}

// entry_of_rank and each rank's key length, from the ranks of the D live entries
__global__ void str_sort_rank_kernel(const u64 *__restrict__ live, u64 D, const u32 *__restrict__ rank_of, const u32 *__restrict__ e_len,
                                     u32 *__restrict__ entry_of_rank, u64 *__restrict__ klen)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < D; i += stride) {
        const u64 e = live[i];
        const u32 r = rank_of[e];
        entry_of_rank[r] = (u32)e;
        klen[r] = e_len[e];
    }
}

// out[k] = the bytes the rows of rank k carry: (roff[k + 1] − roff[k]) · (koff[k + 1] − koff[k])
__global__ void str_sort_row_bytes_kernel(const u64 *__restrict__ roff, const u64 *__restrict__ koff, u64 D, u64 *__restrict__ out)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < D; k += stride)
        out[k] = (roff[k + 1] - roff[k]) * (koff[k + 1] - koff[k]);
}

// sort_cuts_kernel's rule over the rows' CSR by rank (roff [D + 1], roff[D] = n, every rank with rows): partition p
// starts at the first rank boundary at or after floor(p·n/R), so no key is split.  starts[p]: its first row;
// rank_cut[p]: its first rank.
__global__ void str_sort_cuts_kernel(const u64 *__restrict__ roff, u64 D, u64 n, u32 n_parts, u64 *__restrict__ starts, u64 *__restrict__ rank_cut)
{
    const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > n_parts) return;
    const u64 c = ((u64)p * n) / n_parts;
    u64 lo = 0, hi = D;                                   // the first k with roff[k] >= c (roff[D] = n >= c)
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (roff[mid] < c) lo = mid + 1; else hi = mid;
    }
    starts[p] = roff[lo];
    rank_cut[p] = lo;
}

// One partition's rows [row0, row0 + nr), ranks [k0, k1): row j's rank by binary search in the CSR (so a hot key costs
// what any key costs), its key's byte offset in the partition (the byte scan at its rank, plus its place in the
// rank's run times the key's length, less byte0), and off[nr] = the partition's bytes.
__global__ void str_sort_expand_kernel(const u64 *__restrict__ roff, const u64 *__restrict__ boff, const u64 *__restrict__ koff, u64 k0,
                                       u64 k1, u64 row0, u64 nr, u64 byte0, u64 *__restrict__ off, u32 *__restrict__ rank_of_row)
{
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < nr; j += stride) {
        const u64 g = row0 + j;
        u64 lo = k0, hi = k1;
        while (hi - lo > 1) {
            const u64 mid = (lo + hi) >> 1;
            if (roff[mid] <= g) lo = mid; else hi = mid;
        }
        off[j] = boff[lo] + (g - roff[lo]) * (koff[lo + 1] - koff[lo]) - byte0;
        rank_of_row[j] = (u32)lo;
        if (j == 0) off[nr] = boff[k1] - byte0;
    }
}

// ---- sort_by_key over string keys across ranks (engine.cu, exchange_str_sort_locked) ---------------------------
// The ranks agree on each exact cut key word by word (str_sort_key's words).  A cut's state on one rank is ab[2i ..
// 2i + 2) = [a, b): the local key ranks whose words 0 .. w-1 equal the words agreed so far, so that their word w is
// non-decreasing over [a, b).  One thread per cut runs the round's command cmd[2i] = op | w << 8, cmd[2i + 1] = v.
enum { SCUT_IDLE = 0, SCUT_MINMAX = 1, SCUT_COUNT = 2, SCUT_NARROW = 3, SCUT_FINAL = 4 };

// the first key rank in [a, b) whose round-w word is greater than v (b if none), over the keys koff / kbytes
VB_D u64 str_word_upper(const u64 *__restrict__ koff, const unsigned char *__restrict__ kbytes, u64 a, u64 b, u32 w, u64 v)
{
    while (a < b) {
        const u64 mid = a + ((b - a) >> 1);
        if (str_sort_key(kbytes, koff[mid], (u32)(koff[mid + 1] - koff[mid]), w) <= v) a = mid + 1; else b = mid;
    }
    return a;
}

// One round of the cut agreement, out[3i .. 3i + 3) per cut:
//   MINMAX w       (word w of a, word w of b - 1, b - a), or (~0, 0, 0) for an empty interval;
//   COUNT w, v     (roff[first rank past v at word w], 0, 0): the local rows whose key is at most the probed prefix;
//   NARROW w, v    [a, b) becomes the ranks whose word w equals v, then MINMAX w + 1;
//   FINAL w, v     a = b = the first rank past v at word w: the local key cut;
//   IDLE           (0, 0, 0).
__global__ void str_cut_round_kernel(const u64 *__restrict__ cmd, u32 n_cuts, const u64 *__restrict__ koff,
                                     const unsigned char *__restrict__ kbytes, const u64 *__restrict__ roff, u64 *__restrict__ ab,
                                     u64 *__restrict__ out)
{
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cuts) return;
    const u32 op = (u32)(cmd[2 * i] & 0xFF);
    u32 w = (u32)(cmd[2 * i] >> 8);
    const u64 v = cmd[2 * i + 1];
    u64 a = ab[2 * i], b = ab[2 * i + 1];
    u64 x = 0, y = 0, z = 0;
    if (op == SCUT_COUNT) {
        x = roff[str_word_upper(koff, kbytes, a, b, w, v)];
    } else if (op == SCUT_FINAL) {
        a = b = str_word_upper(koff, kbytes, a, b, w, v);
    } else if (op == SCUT_MINMAX || op == SCUT_NARROW) {
        if (op == SCUT_NARROW) {
            const u64 hi = str_word_upper(koff, kbytes, a, b, w, v);
            a = v ? str_word_upper(koff, kbytes, a, hi, w, v - 1) : a;
            b = hi;
            ++w;
        }
        x = ~0ull;
        if (a < b) {
            x = str_sort_key(kbytes, koff[a], (u32)(koff[a + 1] - koff[a]), w);
            y = str_sort_key(kbytes, koff[b - 1], (u32)(koff[b] - koff[b - 1]), w);
        }
        z = b - a;
    }
    ab[2 * i] = a;
    ab[2 * i + 1] = b;
    out[3 * i] = x;
    out[3 * i + 1] = y;
    out[3 * i + 2] = z;
}

// str_sort_cuts_kernel with explicit row targets: rank_cut[p] = the first k with roff[k] >= target[p], starts[p] =
// roff[k].  The owner of a cross-rank sort gets its partitions' first rows from the received totals.
__global__ void str_sort_cuts_at_kernel(const u64 *__restrict__ roff, u64 D, const u64 *__restrict__ target, u32 n_parts,
                                        u64 *__restrict__ starts, u64 *__restrict__ rank_cut)
{
    const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > n_parts) return;
    const u64 c = target[p];
    u64 lo = 0, hi = D;
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (roff[mid] < c) lo = mid + 1; else hi = mid;
    }
    starts[p] = roff[lo];
    rank_cut[p] = lo;
}

// ---- bincode blobs of string reduce ops (engine.cu, vb_shuffle_reduce_blob / vb_shuffle_map_blob) ----------------
// Vec<(String, u64)>: u64 n, then per record u64 len | len key bytes | u64 value, unaligned.  Record i starts at
// 8 + 16 i + (key_off[i] - key_off[0]), so the key offsets place every record without a scan.  Both kernels are
// output-driven: a thread assembles one aligned 16-byte chunk of its destination from shifted aligned loads (load_le)
// and stores it once.

// x with its byte 0 at byte d of a word: the part of x that lands in the word (none when |d| >= 8)
VB_D u64 place_le(u64 x, i64 d)
{
    if (d <= -8 || d >= 8) return 0;
    return d >= 0 ? x << (8 * d) : x >> (-8 * d);
}

// Bytes [p, p + 8) of a blob from the record that starts at st, whose key is the len bytes at kb + ksrc and whose value
// is v (zero where the record has no byte)
VB_D u64 blob_record_word(u64 p, u64 st, u64 len, const unsigned char *kb, u64 ksrc, u64 v)
{
    const u64 k0 = st + 8, k1 = k0 + len;
    u64 w = place_le(len, (i64)(st - p)) | place_le(v, (i64)(k1 - p));
    const u64 a = p > k0 ? p : k0, b = p + 8 < k1 ? p + 8 : k1;
    if (a < b) w |= load_le<false>(kb, ksrc + (a - k0), (u32)(b - a)) << (8 * (a - p));
    return w;
}

// One partition's blob (n_bytes = 8 + 16 nk + key bytes, nk >= 1) into out (16-byte aligned).  key_off [nk + 1]: the
// partition's offsets into key_bytes (key_off[0] need not be 0); vals [nk]: its values.  The first record that reaches
// chunk p is the last one starting at or before p (a binary search over the closed-form starts; record i starts at or
// after 8 + 16 i, so i < p / 16).  Records are at least 16 bytes long, so only it and the next reach the chunk.  The
// last chunk is stored in pieces when the blob does not end on a 16-byte boundary.
__global__ void str_blob_encode_kernel(const u64 *__restrict__ key_off, const unsigned char *__restrict__ key_bytes,
                                       const u64 *__restrict__ vals, u64 nk, u64 n_bytes, unsigned char *__restrict__ out)
{
    const u64 kb0 = key_off[0], n_chunks = (n_bytes + 15) / 16;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < n_chunks; q += stride) {
        const u64 p = 16 * q;
        u64 lo = 0, hi = p / 16 < nk ? p / 16 : nk;
        while (hi - lo > 1) {
            const u64 mid = (lo + hi) >> 1;
            if (8 + 16 * mid + (key_off[mid] - kb0) <= p) lo = mid; else hi = mid;
        }
        u64 w0 = p == 0 ? nk : 0, w1 = 0;
        for (u64 i = lo; i < lo + 2 && i < nk; ++i) {
            const u64 ko = key_off[i], len = key_off[i + 1] - ko, st = 8 + 16 * i + (ko - kb0);
            if (st >= p + 16) break;
            const u64 v = vals[i];
            w0 |= blob_record_word(p, st, len, key_bytes, ko, v);
            w1 |= blob_record_word(p + 8, st, len, key_bytes, ko, v);
        }
        if (p + 16 <= n_bytes) {
            *(ulonglong2 *)(out + p) = make_ulonglong2(w0, w1);
            continue;
        }
        u64 at = p, rest = n_bytes - p, w = w0;    // 1..15 bytes: 8, 4, 2, 1 in turn keep every store aligned
        if (rest >= 8) { *(u64 *)(out + at) = w0; at += 8; rest -= 8; w = w1; }
        if (rest & 4) { *(u32 *)(out + at) = (u32)w; at += 4; w >>= 32; }
        if (rest & 2) { *(unsigned short *)(out + at) = (unsigned short)w; at += 2; w >>= 16; }
        if (rest & 1) out[at] = (unsigned char)w;
    }
}

// The inverse, over a blob of n >= 1 records whose key lengths the host walk checked: koff [n + 1] (the scanned
// lengths) → the key bytes, contiguous (out_bytes padded to whole 16-byte chunks), and the values.  Key byte j of record
// i sits at blob offset 16 + 16 i + j and its value at 16 + 16 i + koff[i + 1].  A chunk starts in the last record with
// koff[i] <= j0 (which skips empty keys) and walks forward through the records that end inside it.
__global__ void str_blob_decode_kernel(const unsigned char *__restrict__ blob, const u64 *__restrict__ koff, u64 n,
                                       unsigned char *__restrict__ out_bytes, u64 *__restrict__ out_vals)
{
    const u64 nkb = koff[n], n_chunks = (nkb + 15) / 16, total = n_chunks > n ? n_chunks : n;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        if (t < n) out_vals[t] = load_le<false>(blob, 16 + 16 * t + koff[t + 1], 8);
        if (t >= n_chunks) continue;
        const u64 j0 = 16 * t, j1 = j0 + 16 < nkb ? j0 + 16 : nkb;
        u64 lo = 0, hi = n;
        while (hi - lo > 1) {
            const u64 mid = (lo + hi) >> 1;
            if (koff[mid] <= j0) lo = mid; else hi = mid;
        }
        u64 w[2] = {0, 0};
        for (u64 i = lo, j = j0; j < j1; ++i) {                  // [j, e): the part of record i's key in the chunk
            const u64 e = koff[i + 1] < j1 ? koff[i + 1] : j1;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const u64 lo_h = j0 + 8 * h, a = j > lo_h ? j : lo_h, b = e < lo_h + 8 ? e : lo_h + 8;
                if (a < b) w[h] |= load_le<false>(blob, 16 + 16 * i + a, (u32)(b - a)) << (8 * (a - lo_h));
            }
            j = e;
        }
        *(ulonglong2 *)(out_bytes + j0) = make_ulonglong2(w[0], w[1]);
    }
}

}  // namespace vb
