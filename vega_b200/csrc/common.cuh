// common.cuh — shared types, hashing, PTX helpers for libvega_b200 (sm_90a only).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

typedef uint64_t u64;
typedef uint32_t u32;
typedef int64_t i64;
typedef int32_t i32;

#define VB_HD __host__ __device__ __forceinline__
#define VB_D __device__ __forceinline__

namespace vb {

// ---------------------------------------------------------------------------------------------
// MetroHash64_1 specialised for 8- and 4-byte keys, seed 0 — the reference's partitioner hash
// (src/partitioner.rs:21-25; fasthash 0.4.0 MetroHasher).  The constants are 32-bit, so each
// 64-bit multiply is two IMADs on the device.
// ---------------------------------------------------------------------------------------------
VB_HD u64 rotr64(u64 v, unsigned k) { return (v >> k) | (v << (64 - k)); }

VB_HD u64 metro64_1_u64(u64 key)
{
    const u64 k0 = 0xC83A91E1ull, k1 = 0x8648DBDBull, k2 = 0x7BDEC03Bull, k3 = 0x2F5870A5ull;
    u64 h = (k2 * k0) + 8ull;            // ((seed + k2) * k0) + len, seed = 0, len = 8
    h += key * k3;
    h ^= rotr64(h, 33) * k1;
    h ^= rotr64(h, 33);
    h *= k0;
    h ^= rotr64(h, 33);
    return h;
}

VB_HD u64 metro64_1_u32(u32 key)
{
    const u64 k0 = 0xC83A91E1ull, k1 = 0x8648DBDBull, k2 = 0x7BDEC03Bull, k3 = 0x2F5870A5ull;
    u64 h = (k2 * k0) + 4ull;
    h += (u64)key * k3;
    h ^= rotr64(h, 15) * k1;
    h ^= rotr64(h, 33);
    h *= k0;
    h ^= rotr64(h, 33);
    return h;
}

VB_HD u64 hash_key(u64 key, u32 key_width) { return key_width == 4 ? metro64_1_u32((u32)key) : metro64_1_u64(key); }

// Exact x % d for a run-time d < 2^32 without a 64-bit divide: q = mulhi(x, floor((2^64-1)/d))
// is floor(x/d) or one less, so a single conditional subtract finishes it.
struct FastMod {
    u64 magic;   // floor((2^64 - 1) / d)
    u64 d;
    u32 pow2_mask;   // d - 1 when d is a power of two, else 0xFFFFFFFF marker unused
    u32 is_pow2;
};

inline FastMod make_fastmod(u32 d)
{
    FastMod f;
    f.d = d;
    f.magic = ~0ull / (u64)d;
    f.is_pow2 = (d & (d - 1)) == 0;
    f.pow2_mask = d - 1;
    return f;
}

VB_HD u64 mulhi64(u64 a, u64 b)
{
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (u64)(((unsigned __int128)a * b) >> 64);
#endif
}

VB_HD u32 fastmod(u64 x, const FastMod &f)
{
    if (f.is_pow2) return (u32)x & f.pow2_mask;
    u64 q = mulhi64(x, f.magic);
    u64 r = x - q * f.d;
    if (r >= f.d) r -= f.d;
    return (u32)r;
}

// HashPartitioner::get_partition (src/partitioner.rs:54-57)
VB_HD u32 get_partition(u64 key, u32 key_width, const FastMod &f) { return fastmod(hash_key(key, key_width), f); }

// Hash-table slot hash: NOT the partitioner (placement inside our own device table is free to
// differ); two multiplies, high bits taken by the caller.
VB_HD u64 slot_hash(u64 key)
{
    u64 x = key;
    x ^= x >> 32;
    x *= 0xD6E8FEB86659FD93ull;
    x ^= x >> 32;
    x *= 0x9E3779B97F4A7C15ull;
    return x;
}

VB_HD u64 splitmix64(u64 x)
{
    x += 0x9E3779B97F4A7C15ull;
    u64 z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// Order-preserving maps into u64 so one unsigned atomicMin/Max / radix sort serves all dtypes.
enum : int { TX_NONE = 0, TX_I64 = 1, TX_F64 = 2 };
VB_HD u64 tx_fwd(u64 v, int tx)
{
    if (tx == TX_I64) return v ^ 0x8000000000000000ull;
    if (tx == TX_F64) return (v >> 63) ? ~v : (v | 0x8000000000000000ull);
    return v;
}
VB_HD u64 tx_inv(u64 v, int tx)
{
    if (tx == TX_I64) return v ^ 0x8000000000000000ull;
    if (tx == TX_F64) return (v >> 63) ? (v & 0x7FFFFFFFFFFFFFFFull) : ~v;
    return v;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------
// PTX helpers (sm_90a)
// ---------------------------------------------------------------------------------------------
VB_D u64 policy_evict_first()
{
    u64 p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}

VB_D u64 policy_evict_normal()
{
    u64 p;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
VB_D u64 policy_evict_last()
{
    u64 p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// 128-bit streaming load: read-only path, no L1 allocation, L2 evict-first (the input is read
// exactly once and must not push the hash table out of the 50 MB L2).
VB_D ulonglong2 ld_stream_u64x2(const void *p, u64 pol)
{
    ulonglong2 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;"
                 : "=l"(r.x), "=l"(r.y)
                 : "l"(p), "l"(pol));
    return r;
}
VB_D u64 ld_stream_u64(const void *p, u64 pol)
{
    u64 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(r) : "l"(p), "l"(pol));
    return r;
}
VB_D u32 ld_stream_u32(const void *p, u64 pol)
{
    u32 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
    return r;
}
// L2-only (cache-global) load for table probes: the table lives in L2, L1 lines would be stale.
VB_D u64 ld_cg_u64(const u64 *p)
{
    u64 r;
    asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(r) : "l"(p));
    return r;
}
VB_D u32 ld_volatile_u32(const u32 *p)
{
    u32 r;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
VB_D void st_stream_u64(void *p, u64 v)
{
    asm volatile("st.global.L1::no_allocate.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
VB_D void st_stream_u32(void *p, u32 v)
{
    asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// ---- mbarrier + bulk async copy (TMA engine, SASS: UBLKCP / SYNCS) ---------------------------------
// Input tiles are staged global → shared by the copy engine, not through registers: a producer lane
// posts the expected byte count on an mbarrier and issues one cp.async.bulk per tile; consumers wait
// on the barrier's phase parity.  (16-byte aligned addresses, sizes multiple of 16.)
VB_D u32 smem_u32(const void *p) { return (u32)__cvta_generic_to_shared(p); }
VB_D void mbar_init(u64 *bar, u32 count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
VB_D void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
VB_D void mbar_arrive(u64 *bar)
{
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
VB_D void mbar_arrive_expect_tx(u64 *bar, u32 bytes)
{
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
VB_D void mbar_wait(u64 *bar, u32 parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra D_%=;\n\t"
        "bra W_%=;\n\t"
        "D_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global → shared bulk copy, completion counted in bytes on `bar`; L2 policy from createpolicy
VB_D void bulk_g2s(void *dst_smem, const void *src_gmem, u32 bytes, u64 *bar, u64 pol)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
                 : "memory");
}
// shared → global bulk store (bulk_group completion)
VB_D void bulk_s2g(void *dst_gmem, const void *src_smem, u32 bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
VB_D void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> VB_D void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> VB_D void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
VB_D void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
VB_D void named_bar_sync(u32 id, u32 nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
VB_D void named_bar_arrive(u32 id, u32 nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

VB_D u32 lane_id() { return threadIdx.x & 31u; }
VB_D u32 lanemask_lt()
{
    u32 m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
#endif  // __CUDACC__

}  // namespace vb
