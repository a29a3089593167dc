// zstd_lazy.cuh — the zstd search class of levels 6-12: hash chains over the whole chunk and a lazy parse
// (rule: zstd_lazy_rule.h; CPU twin: oracle/chain_twin.c).  Included by lz4_kernels.cu after the level-3 encoder;
// it feeds the same entropy stage (z_encode_block) and the same frame kernels.
//
// Per group of chunks (at most ZL_GROUP_BYTES of positions, so the per-position arrays stay bounded):
//   zstd_lazy_hash_kernel    one thread per position: key h(p), value p
//   cub::DeviceRadixSort     stable sort by key: equal keys end up next to each other in position order
//   zstd_lazy_prev_kernel    prev[p] = the sorted neighbour with the same key (the walk stops at the chunk's start)
//   zstd_lazy_search_kernel  one thread per position walks prev[] (input bytes through L2) and writes best[p]
//                            (the LZ4 class of levels 10-12, lz4_hc.cuh, runs these four with its block and margins)
//   zstd_lazy_blocks_kernel  one CTA per 64 KiB window, its four 16 KiB blocks in order: lazy parse, merge, sequences
//                            and literals to the CTA's ZScratch, z_encode_block
#pragma once
#include "zstd_lazy_rule.h"

#define ZL_NONE        0xFFFFFFFFu
#define ZL_RANGE       64u                       // positions per thread in the block parse (16 KiB / 256 threads)
#define ZL_PAD(p)      ((p) + 2u * ((p) >> 6))   // u16 index with one spare word per range: the ranges of a warp's 32
                                                 // threads start in 32 different banks
#define ZL_GROUP_BYTES (256u << 20)

__global__ void __launch_bounds__(256)
zstd_lazy_hash_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                      uint32_t c0, uint32_t npos, uint32_t mm, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npos) return;
    const uint32_t c = c0 + i / chunk_size, o = i % chunk_size;
    uint32_t h = 0;                              // positions without a hash sit at the end of their chunk: no chain reaches them
    if ((uint64_t)o + mm <= zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size)) {
        const uint8_t* p = in + (uint64_t)c * chunk_size + o;
        uint64_t v = 0;
        for (uint32_t k = 0; k < mm; k++) v |= (uint64_t)p[k] << (8 * k);
        h = zl_hash(v, mm);
    }
    keys[i] = h; vals[i] = i;
}

__global__ void __launch_bounds__(256)
zstd_lazy_prev_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, uint32_t npos, uint32_t* __restrict__ prev)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npos) return;
    prev[vals[i]] = (i && keys[i - 1] == keys[i]) ? vals[i - 1] : ZL_NONE;
}

// 32-bit little-endian load from any byte address (aligned loads through the read-only path; the second word is only
// read when the four bytes straddle it)
__device__ __forceinline__ uint32_t zl_ld32(const uint8_t* p)
{
    const uintptr_t a = (uintptr_t)p;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3) * 8, lo = __ldg(w);
    return sh ? __funnelshift_r(lo, __ldg(w + 1), sh) : lo;
}

// BLK: the parse unit (zstd: 16 KiB blocks, LZ4: 64 KiB blocks).  START: a match starts at o only if o + START <= the
// block's end (0: o + mm, the zstd rule; LZ4: 12).  END: matches end at or before the block's end - END (zstd 0, LZ4 5).
template <uint32_t BLK, uint32_t START, uint32_t END>
__global__ void __launch_bounds__(256)
zstd_lazy_search_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                        uint32_t c0, uint32_t npos, uint32_t mm, uint32_t depth, uint32_t W,
                        const uint32_t* __restrict__ prev, uint32_t* __restrict__ best)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npos) return;
    const uint32_t c = c0 + i / chunk_size, o = i % chunk_size;
    const uint64_t len = zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size);
    uint32_t res = 0;
    const uint64_t bend = ((uint64_t)(o / BLK) + 1) * BLK < len ? ((uint64_t)(o / BLK) + 1) * BLK : len;
    if ((uint64_t)o + (START ? START : mm) <= bend) {
        const uint32_t cap = bend - END - o < ZL_LCAP ? (uint32_t)(bend - END - o) : ZL_LCAP;
        const uint8_t* base = in + (uint64_t)c * chunk_size;
        const uint8_t* ps = base + o;
        const uint32_t cs0 = i - o;              // group-relative start of the chunk
        uint32_t bl = 0, bo = 0, q = prev[i];
        for (uint32_t step = 0; step < depth && q != ZL_NONE && q >= cs0 && i - q <= W; step++, q = prev[q]) {
            const uint8_t* qs = base + (q - cs0);
            if (bl && qs[bl] != ps[bl]) continue;                       // cannot be longer than the best so far
            uint32_t l = 0;
            for (;;) {
                if (l + 4 > cap) { while (l < cap && qs[l] == ps[l]) l++; break; }
                const uint32_t x = zl_ld32(qs + l) ^ zl_ld32(ps + l);
                if (x) { l += (uint32_t)(__ffs(x) - 1) >> 3; break; }
                l += 4;
            }
            if (l >= mm && l > bl) { bl = l; bo = i - q; if (l == cap) break; }
        }
        res = bl ? bl | (bo << ZL_LEN_BITS) : 0;
    }
    best[i] = res;
}

// ---- the parallel lazy parse of one 16 KiB unit (a zstd block, or a quarter of an LZ4 block).  The parse is a walk
// over nx[]: nx[p] = p + 1 (literal) or p + length (match), and nx[p] depends only on best[p .. p+2].  Thread t owns the
// range [64 t, 64 t + 64): it resolves ex[] backwards over its range (64 steps), thread 0 chains the ranges' entries
// (<= 256 dependent loads), then every thread re-walks its range from its true entry twice — to count, then to emit.
// A match that folds into the sequence before it (literal length 0, same offset) is found by its own range when the
// two are in one range; a range's entry match is flagged by the range the parse came from.  The kernels call the steps
// below between their own CTA_SYNC()s and keep their own scans.
struct ZlParse {
    uint16_t nx[ZL_PAD(ZL_BLOCK)];        // next free position of the parse from p
    uint16_t ex[ZL_PAD(ZL_BLOCK)];        // first position at or past the end of p's range that the parse reaches from p
    uint16_t entry[256];                  // first position of the true parse in each range (0xFFFF: none)
    uint32_t fold[256];                   // the range's entry match folds into the sequence before it
};

// nx[] of the unit's nb positions (bb: their best[]) under the class's lazy decision; entry[] and fold[] reset.
// best[p] != 0 only where p + minMatch <= the block's end (zstd: minMatch >= 4, the block is the unit; LZ4: p + 12 <=
// the end of its 64 KiB block), so best[p+1] and best[p+2] are read without bounds checks: they lie inside the unit,
// or for LZ4 inside the same block.
template <int (*DEFER)(uint32_t, uint32_t, uint32_t, uint32_t)>
__device__ __forceinline__ void zl_parse_nx(ZlParse& P, const uint32_t* bb, uint32_t nb, uint32_t lazy)
{
    for (uint32_t p = threadIdx.x; p < nb; p += 256) {
        const uint32_t m = bb[p];
        uint32_t x = p + 1;
        if (m && !DEFER(m, bb[p + 1], lazy >= 2 ? bb[p + 2] : 0, lazy)) x = p + zl_len(m);
        P.nx[ZL_PAD(p)] = (uint16_t)x;
    }
    P.entry[threadIdx.x] = 0xFFFF; P.fold[threadIdx.x] = 0;
}

// ex[] over this thread's range [r0, r1)
__device__ __forceinline__ void zl_parse_ex(ZlParse& P, uint32_t r0, uint32_t r1)
{
    for (uint32_t p = r1; p > r0;) { p--; const uint32_t x = P.nx[ZL_PAD(p)]; P.ex[ZL_PAD(p)] = (uint16_t)(x >= r1 ? x : P.ex[ZL_PAD(x)]); }
}

// thread 0: entry[] of the ranges the parse reaches from p; returns the first position at or past the unit's end
__device__ __forceinline__ uint32_t zl_parse_entries(ZlParse& P, uint32_t p, uint32_t nb)
{
    for (; p < nb; p = P.ex[ZL_PAD(p)]) P.entry[p / ZL_RANGE] = (uint16_t)p;
    return p;
}

struct ZlCount { uint32_t nseq, nlit, lend; bool ematch; };

// walk 1 of the range [e, r1) from its entry e (0xFFFF: none, nothing to walk): new sequences, literals, the last
// match end, whether the entry is a match; flags a fold at the next range's entry
__device__ __forceinline__ ZlCount zl_parse_count(ZlParse& P, const uint32_t* bb, uint32_t e, uint32_t r1, uint32_t nb)
{
    ZlCount c = {0, 0, 0, false};
    uint32_t poff = 0;
    for (uint32_t p = e; p < r1;) {
        const uint32_t x = P.nx[ZL_PAD(p)];
        if (x == p + 1) { c.nlit++; poff = 0; }
        else {
            const uint32_t off = zl_off(bb[p]);
            if (p == e) c.ematch = true;
            if (off != poff) c.nseq++;
            poff = off; c.lend = x;
            if (x >= r1 && x < nb && P.nx[ZL_PAD(x)] != x + 1 && zl_off(bb[x]) == off) P.fold[x / ZL_RANGE] = 1;
        }
        p = x;
    }
    return c;
}

// walk 2: put(si, start, anchor, off, merged length) for each sequence the range opens, numbered from si; lit(p) for
// each literal; anchor: the end of the last match before the range.  A fold at the entry (efold), and folds before the
// range's first new sequence, belong to the sequence of an earlier range: their length is returned, for the caller to
// add once that sequence's owner has written it.
template <class Put, class Lit>
__device__ __forceinline__ uint32_t zl_parse_emit(const ZlParse& P, const uint32_t* bb, uint32_t e, uint32_t r1, bool efold,
                                                  uint32_t si, uint32_t anchor, Put put, Lit lit)
{
    uint32_t poff = 0, carry = 0, qs = 0, qa = 0, qo = 0, ql = 0;
    bool open = false;
    for (uint32_t p = e; p < r1;) {
        const uint32_t x = P.nx[ZL_PAD(p)];
        if (x == p + 1) { lit(p); poff = 0; }
        else {
            const uint32_t off = zl_off(bb[p]), len = x - p;
            if (p == e ? efold : off == poff) { if (open) ql += len; else carry += len; }
            else {
                if (open) put(si++, qs, qa, qo, ql);
                qs = p; qa = anchor; qo = off; ql = len; open = true;
            }
            poff = off; anchor = x;
        }
        p = x;
    }
    if (open) put(si, qs, qa, qo, ql);
    return carry;
}

struct __align__(16) ZlSmem {
    uint8_t blk[ZL_BLOCK];                        // the block (literals and the raw fallback)
    union {
        ZlParse p;
        ZEnt ent;
    };
    ZFseShared fse;
    __align__(16) uint32_t scanws[48];            // block_exscan (33 words) | zl_block_exmax (8 words)
};
static_assert(sizeof(ZlSmem) + 1024 <= (228 * 1024) / 2, "two CTAs per SM");

// exclusive max over the CTA's threads in order (0 for thread 0); `ws` >= 8 words
__device__ __forceinline__ uint32_t zl_block_exmax(uint32_t v, uint32_t* ws)
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc = max(inc, y); }
    uint32_t ex = __shfl_up_sync(ZMT_FULL_MASK, inc, 1);
    if (lane == 0) ex = 0;
    __syncwarp(); __syncthreads();
    if (lane == 31) ws[wid] = inc;
    __syncthreads();
    for (uint32_t w = 0; w < wid; w++) ex = max(ex, ws[w]);
    return ex;
}

// Each 16 KiB block: the range parse above, then the sequences and literals to the CTA's ZScratch and z_encode_block.
__global__ void __launch_bounds__(256, 2)
zstd_lazy_blocks_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                        uint32_t bpc, uint32_t c0, uint32_t nwin, uint32_t lazy, const uint32_t* __restrict__ best,
                        uint8_t* __restrict__ tmp, uint32_t* __restrict__ blk_csize, ZScratch* __restrict__ zscratch)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    ZlSmem& S = *reinterpret_cast<ZlSmem*>(smem_raw);
    constexpr uint32_t NT = 256;
    const uint32_t tid = threadIdx.x;
    ZScratch* const zs = zscratch + blockIdx.x;
    auto cta_sync = [] () { CTA_SYNC(); };
    z_load_fse_shared(S.fse, tid, NT);

    for (uint32_t w = blockIdx.x; w < nwin; w += gridDim.x) {
        const uint32_t blk = c0 * bpc + w, chunk = blk / bpc, bic = blk % bpc;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, chunk, in_bytes, chunk_size);
        const uint64_t boff = (uint64_t)bic * LZ4_BLK;
        uint32_t n = 0;
        if (boff < cbytes) n = (uint32_t)((cbytes - boff) < LZ4_BLK ? (cbytes - boff) : LZ4_BLK);
        if (n == 0) { if (tid == 0) blk_csize[blk] = 0; continue; }
        uint8_t* dst = tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE;
        const uint8_t* src = in + (uint64_t)chunk * chunk_size + boff;
        const uint32_t* bw = best + (uint64_t)(chunk - c0) * chunk_size + boff;
        uint32_t out_pos = 0;

        for (uint32_t b0 = 0; b0 < n; b0 += ZL_BLOCK) {
            const uint32_t nb = n - b0 < ZL_BLOCK ? n - b0 : ZL_BLOCK;
            const uint32_t* bb = bw + b0;
            CTA_SYNC();                                          // the previous block's entropy stage is done with the union
            for (uint32_t i = tid; i < nb; i += NT) S.blk[i] = src[b0 + i];
            zl_parse_nx<zl_defer>(S.p, bb, nb, lazy);
            CTA_SYNC();
            const uint32_t r0 = tid * ZL_RANGE, r1 = r0 + ZL_RANGE < nb ? r0 + ZL_RANGE : nb;
            zl_parse_ex(S.p, r0, r1);
            CTA_SYNC();
            if (tid == 0) zl_parse_entries(S.p, 0, nb);
            CTA_SYNC();
            const uint32_t e = S.p.entry[tid];
            const ZlCount c = zl_parse_count(S.p, bb, e, r1, nb);
            CTA_SYNC();
            const bool efold = c.ematch && S.p.fold[tid];
            uint32_t tot;
            const uint32_t pre = block_exscan(((c.nseq - efold) << 16) | c.nlit, S.scanws, &tot);
            const uint32_t anchor0 = zl_block_exmax(c.lend, S.scanws + 36);
            uint32_t li = pre & 0xFFFFu;
            const uint32_t carry = zl_parse_emit(S.p, bb, e, r1, efold, pre >> 16, anchor0,
                [&] (uint32_t si, uint32_t st, uint32_t a, uint32_t off, uint32_t len) {   // len <= 16 KiB: fits mlen
                    zs->seq[si] = ZSeq{(st - a) | ((off >> 16) << 24), (uint16_t)off, (uint16_t)len};
                },
                [&] (uint32_t p) { zs->lit[li++] = S.blk[p]; });
            CTA_SYNC();
            if (carry) atomicAdd(reinterpret_cast<uint32_t*>(&zs->seq[(pre >> 16) - 1].off), carry << 16);     // mlen = the word's high half
            CTA_SYNC();
            const bool last = boff + b0 + nb == cbytes;
            out_pos += z_encode_block(S.ent, S.fse, zs, tot >> 16, tot & 0xFFFFu, S.blk, nb, last, dst + out_pos, S.scanws, cta_sync);
        }
        if (tid == 0) blk_csize[blk] = out_pos;
    }
}
