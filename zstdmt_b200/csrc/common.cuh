// common.cuh — device helpers shared by the sm_90a kernels (LZ4 + zstd paths).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define ZMT_FULL_MASK 0xFFFFFFFFu

// ---------------------------------------------------------------- XXH32 constants
#define XXP1 0x9E3779B1u
#define XXP2 0x85EBCA77u
#define XXP3 0xC2B2AE3Du
#define XXP4 0x27D4EB2Fu
#define XXP5 0x165667B1u

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return __funnelshift_l(x, x, r); }
__device__ __forceinline__ uint32_t xxh32_round(uint32_t acc, uint32_t lane) { return rotl32(acc + lane * XXP2, 13) * XXP1; }

// XXH32 of a tiny (<16 byte) buffer held in registers/local memory — LZ4F header checksum.
__device__ __forceinline__ uint32_t xxh32_small(const uint8_t* p, uint32_t len, uint32_t seed)
{
    uint32_t h = seed + XXP5 + len;
    uint32_t i = 0;
    for (; i + 4 <= len; i += 4) {
        uint32_t w = (uint32_t)p[i] | ((uint32_t)p[i + 1] << 8) | ((uint32_t)p[i + 2] << 16) | ((uint32_t)p[i + 3] << 24);
        h = rotl32(h + w * XXP3, 17) * XXP4;
    }
    for (; i < len; i++) h = rotl32(h + p[i] * XXP5, 11) * XXP1;
    h ^= h >> 15; h *= XXP2; h ^= h >> 13; h *= XXP3; h ^= h >> 16;
    return h;
}

// ---------------------------------------------------------------- shared-memory unaligned loads
// 32-bit little-endian load from an arbitrary byte offset of a 4-byte-aligned shared array:
// two aligned LDS + one funnel shift (no byte loads, no bank conflicts for consecutive lanes).
__device__ __forceinline__ uint32_t lds32u(const uint8_t* base, uint32_t pos)
{
    const uint32_t* w = reinterpret_cast<const uint32_t*>(base) + (pos >> 2);
    return __funnelshift_r(w[0], w[1], (pos & 3) * 8);
}

// ---------------------------------------------------------------- global little-endian loads (any alignment)
__device__ __forceinline__ uint32_t ldg_le32(const uint8_t* p)
{
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t ldg_le64(const uint8_t* p) { return (uint64_t)ldg_le32(p) | ((uint64_t)ldg_le32(p + 4) << 32); }
__device__ __forceinline__ void stg_le32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
__device__ __forceinline__ void stg_le64(uint8_t* p, uint64_t v) { stg_le32(p, (uint32_t)v); stg_le32(p + 4, (uint32_t)(v >> 32)); }

// ---------------------------------------------------------------- mbarrier + 1-D bulk async copy (TMA unit, SASS UBLKCP)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void* sdst, const void* gsrc, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// shared -> global bulk copy (bulk_group completion)
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* ssrc, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- cooperative byte copy (global -> global)
// All `nt` threads of a group call with their rank `t`.  Destination stores are 16-byte
// vectors once dst is aligned; the source is re-aligned with funnel shifts when needed.
__device__ __forceinline__ void coop_copy_g2g(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n, uint32_t t, uint32_t nt)
{
    uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (head > n) head = n;
    for (uint32_t i = t; i < head; i += nt) dst[i] = src[i];
    uint32_t nv = (n - head) >> 4;
    const uint8_t* s = src + head;
    uint4* d4 = reinterpret_cast<uint4*>(dst + head);
    uint32_t mis = (uint32_t)((uintptr_t)s & 15);
    if (mis == 0) {
        const uint4* s4 = reinterpret_cast<const uint4*>(s);
        for (uint32_t i = t; i < nv; i += nt) d4[i] = s4[i];
    } else if ((mis & 3) == 0) {
        const uint32_t* s1 = reinterpret_cast<const uint32_t*>(s);
        for (uint32_t i = t; i < nv; i += nt) {
            uint4 v; v.x = s1[4 * i]; v.y = s1[4 * i + 1]; v.z = s1[4 * i + 2]; v.w = s1[4 * i + 3];
            d4[i] = v;
        }
    } else {
        const uint32_t* s1 = reinterpret_cast<const uint32_t*>(s - (mis & 3));
        uint32_t sh = (mis & 3) * 8;
        for (uint32_t i = t; i < nv; i += nt) {
            uint32_t w0 = s1[4 * i], w1 = s1[4 * i + 1], w2 = s1[4 * i + 2], w3 = s1[4 * i + 3], w4 = s1[4 * i + 4];
            uint4 v;
            v.x = __funnelshift_r(w0, w1, sh); v.y = __funnelshift_r(w1, w2, sh);
            v.z = __funnelshift_r(w2, w3, sh); v.w = __funnelshift_r(w3, w4, sh);
            d4[i] = v;
        }
    }
    uint32_t done = head + (nv << 4);
    for (uint32_t i = done + t; i < n; i += nt) dst[i] = src[i];
}

// ---------------------------------------------------------------- block-wide exclusive scan (<= 1024 threads)
// Returns the exclusive prefix of `v` over the CTA; *total receives the CTA sum.
// `ws` is a shared array of >= 33 uint32_t.  Contains three __syncthreads() (the first
// protects `ws` against the previous call's readers).
__device__ __forceinline__ uint32_t block_exscan(uint32_t v, uint32_t* ws, uint32_t* total)
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc += y; }
    __syncwarp();
    __syncthreads();
    if (lane == 31) ws[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t x = lane < nw ? ws[lane] : 0, xi = x;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, xi, d); if (lane >= (uint32_t)d) xi += y; }
        ws[lane] = xi - x;
        if (lane == 31) ws[32] = xi;
    }
    __syncthreads();
    *total = ws[32];
    return inc - v + ws[wid];
}
