// lz4_kernels.cu — hand-written sm_90a kernels: the LZ77 front end shared by both codecs, the LZ4 back end
// (block format, XXH32, frame pack; the decoder is in lz4_decode.cuh) and the launchers of the Zstandard encoder (entropy stage in
// zstd_entropy.cuh; the Zstandard decoder lives in zstd_decode.cu).
//
// Replaces the arithmetic the reference reaches through
//   LZ4F_compressFrame   (lib/lz4-mt_compress.c:280-283)
//   LZ4F_decompress      (lib/lz4-mt_decompress.c:349-351)
// plus the 12-byte skippable container write (lib/lz4-mt_compress.c:293-298).
//
// Kernels
//   lz4_blocks_pipe_kernel      (lz4_pipe.cuh) one CTA per 64 KiB LZ4F block, block staged in SMEM by the TMA unit
//                               (cp.async.bulk); round-synchronous hash candidates, speculative-chain parallel greedy
//                               parse, scan-based emission, as two teams pipelined over 4 KiB tiles.
//   zstd_blocks_kernel          one CTA per 64 KiB zstd match window: the same parse functions run by a single team,
//                               sequences and literals to a scratch, entropy stage (zstd_entropy.cuh) every 4 tiles.
//   zstd_lazy.cuh               the search class of zstd levels 6-12: chunk-wide hash chains (hash, radix sort, chain
//                               walk) and a lazy parse per 16 KiB block, into the same entropy stage.
//   xxh32_kernel                4 lanes per chunk (the 4 XXH32 accumulators), 8 chunks per warp.
//   lz4_frame_sizes_kernel / lz4_frame_pack_kernel
//                               frame size per chunk -> exclusive scan -> compaction of the block
//                               payloads + LZ4F header/end-mark/checksum + skippable header.
//   lz4_decode.cuh              the LZ4F decoder: frame scan, pass A (token parse + literals + match records), pass B (match
//                               execution by ticket, step window in SMEM), sequential fallback for partial-block frames.
//   match_exec.cuh              what pass B shares with the zstd execute pass (zstd_decode.cu): ticket order, step
//                               constants, dependency test, window copies.
//
// The compressor's match/parse rule is deterministic and restated on the CPU in
// oracle/lz4_oracle.c:orc_lz4_block_compress_b200 (tests compare bit-exact).
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <vector>
#include <cub/device/device_radix_sort.cuh>
#include "common.cuh"
#include "frame_format.h"
#include "host_common.h"
#include "launch.h"
#include "zmt_dev.h"
#include "zstd_entropy.cuh"

// bytes of chunk c: explicit per-chunk sizes (host pipeline: any fn_read may come back short)
// or derived from a contiguous input of in_bytes cut every chunk_size bytes.
__device__ __forceinline__ uint64_t zmt_chunk_len(const uint32_t* __restrict__ cb, uint32_t c, uint64_t in_bytes, uint32_t chunk_size)
{
    if (cb) return cb[c];
    const uint64_t base = (uint64_t)c * chunk_size;
    if (in_bytes <= base) return 0;
    return (in_bytes - base) < chunk_size ? (in_bytes - base) : chunk_size;
}

// A CTA barrier preceded by a warp reconvergence: the data-dependent phases leave warps split into
// independently scheduled groups, and an aligned BAR.SYNC + the uniform-datapath branches ptxas places
// after it (BRA.U) must only ever be executed by whole warps (else: 'illegal instruction').
#define CTA_SYNC() do { __syncwarp(); __syncthreads(); } while (0)

// ============================================================================ compressor
#define LZ4_BLK      65536u
#define C_CHAINS     256u          // speculative chains per tile (one per 16-byte segment)
#define C_TILE       4096u         // positions parsed per tile
#define C_SEG        16u           // C_TILE / C_CHAINS : positions owned by one speculative chain
#define C_ROUND      1024u         // hash-table update granularity
#define C_HASHLOG    12
#define C_MAXPIECE   1280u         // 4096/4 match pieces + 256 continuation pieces, multiple of 256
#define C_LONGLIT    32u           // literal runs longer than this are copied cooperatively
#define C_END        0xFFFFu       // link: chain leaves the tile

// ---- shared-memory parts of the two LZ77 kernels (PipeSmem: LZ4, ZstdSmem: Zstandard)
struct __align__(16) LzStage {
    uint8_t  pad0[16];                    // bytes "before" the block (read by the 8-byte window of the candidate rounds, never matched)
    uint8_t  in[LZ4_BLK + 32];            // block bytes + zero pad
};

// what the front end hands the back end for one tile (double-buffered in the LZ4 pipeline)
struct __align__(16) PipeTile {
    uint16_t off[C_TILE];                 // candidate offset per tile position (0 = none)
    uint32_t M[C_TILE / 32];              // has-candidate bits
    uint32_t V[C_TILE / 32];              // visited-by-own-chain bits (chain k writes the 16-bit half k)
    uint32_t len4[C_TILE / 8];            // L - 4 of the candidate piece at each position a chain walk took, 4 bits each
    uint8_t  min_[C_CHAINS];              // entry position of a chain on the true path, relative to its own segment (< 16)
    uint32_t pathmask[C_CHAINS / 32];     // chains on the true path
    uint32_t k0, e_din, do_parse, pad;    // entry chain, offset of the match open at the entry, tile has work
};

// front end, per tile: chain walks and the true path
struct LzFront {
    uint32_t xfree[C_CHAINS];             // own-walk exit position (absolute); then the lanes on a chain's way inside its warp
    uint32_t mpos[C_CHAINS];              // merge position / tile exit (absolute)
    uint16_t xdin[C_CHAINS];              // own-walk exit: offset of the match we are still inside (0 = free)
    uint16_t link[C_CHAINS];              // chain this chain merges into (C_END: leaves the tile)
    uint8_t  jump[C_CHAINS];              // terminal chain reached without leaving the warp
    uint16_t entry[8];                    // per warp: first chain of the true path inside it (0xFFFF: none)
    uint32_t e_next, d_next;              // parse state entering the next tile: position, offset of the match still open there
};

// back end, per tile: marking, piece merge, emission
struct LzBack {
    uint32_t Sel[C_TILE / 32];            // pieces on the true greedy chain
    uint32_t Cont[C_TILE / 32];           // ... that continue the previous piece's match across a segment boundary
    uint8_t  clen[C_CHAINS];              // per segment: length of the Cont piece at its start (written by the marking walk)
    uint16_t piece[C_MAXPIECE];           // tile-relative start of the r-th selected piece
    union {                               // segprev is read by head detection, before the heads are written
        uint16_t hidx[C_TILE / 4];        // heads: one per sequence, sequences hold a match of >= 4 bytes
        uint16_t segprev[C_CHAINS];       // per segment: 1 + start of the last non-Cont piece before it (0: none)
    };
    uint32_t longl[2 * (C_TILE / (C_LONGLIT + 1) + 2)];   // jobs: literal runs > C_LONGLIT (start | length << 16, output offset) -- at most
                                                           // 4096/37 + 1 pending per tile -- and 255-runs of match lengths >= 1290 (count, offset | 1<<31)
};

// the 16 bytes at s + pos, any alignment: five aligned words
__device__ __forceinline__ uint4 lds128u(const uint8_t* s, uint32_t pos)
{
    const uint32_t* w = reinterpret_cast<const uint32_t*>(s) + (pos >> 2);
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4], sh = 8 * (pos & 3);
    return make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
}

// number of leading bytes (<= cap <= 16) in which the 16-byte strings a and b agree: one mismatch scan, no loop
__device__ __forceinline__ uint32_t c_agree16(uint4 a, uint4 b, uint32_t cap)
{
    const uint32_t x0 = a.x ^ b.x, x1 = a.y ^ b.y, x2 = a.z ^ b.z, x3 = a.w ^ b.w;
    // index of the first differing bit (128: none), by selects: __clz(__brev(0)) is 32
    uint32_t m = 96 + __clz(__brev(x3));
    m = x2 ? 64 + __clz(__brev(x2)) : m;
    m = x1 ? 32 + __clz(__brev(x1)) : m;
    m = x0 ? __clz(__brev(x0)) : m;
    m >>= 3;
    return m < cap ? m : cap;
}

// Length (<= cap <= 16) of a continuation piece: the bytes from the segment boundary p on that still match at offset d.
// Both 16-byte strings are loaded at once (p is 16-aligned, LzStage::in too; reads run at most 19 bytes past p - d).
__device__ __forceinline__ uint32_t c_cont_len(const uint8_t* s, uint32_t p, uint32_t d, uint32_t cap)
{
    return c_agree16(*reinterpret_cast<const uint4*>(s + p), lds128u(s, p - d), cap);
}

// L - 4 of the candidate piece at q (offset d, 4 bytes known equal), up to end = min(cut, limit) (q + 4 <= end <= q + 19):
// both 16-byte strings loaded at once, one mismatch scan
__device__ __forceinline__ uint32_t c_piece_len4(const uint8_t* s, uint32_t q, uint32_t d, uint32_t end)
{
    return c_agree16(lds128u(s, q + 4), lds128u(s, q + 4 - d), end - (q + 4));
}

// Walk one speculative chain through the tile.  The greedy parse is evaluated piecewise: a match is cut at
// the first segment boundary that leaves it >= 4 bytes, and continues ("inside", din = its offset) into the
// next segment, so no lane ever compares more than 19 bytes per step, in one compare (c_piece_len4, c_cont_len).
// Pieces are merged again at emission.
// A candidate piece's length L (4..19) depends only on its start q (offset, cut, limit), not on the chain that takes it,
// so the front end records L - 4 per start in T.len4 and the marking walk reads it back; only a Cont piece, whose
// length depends on the offset carried in, is measured again there.
// Walk 0 (c_walk0) covers the own segment; c_walk covers the rest:
//   MODE 1: continuation until it merges into another chain or leaves the tile (-> X.link/X.mpos; ORs the lengths of
//           its pieces into T.len4: chains that continue alike take the same pieces, and a position walk 0 took is a
//           merge, so the only writers that meet write the same nibble)                              X: LzFront
//   MODE 2: re-walk of a chain that is on the true path, from where the path enters it: marks X.Sel/X.Cont and the
//           Cont lengths X.clen.  The own segment's pieces are its V bits from there on (one step), the continuation
//           takes the steps of MODE 1 with the lengths from T.len4, so only Cont steps compare bytes.     X: LzBack
template <int MODE, class OUT>
__device__ __forceinline__ void c_walk(const uint8_t* in, PipeTile& T, OUT& X, uint32_t k, uint32_t p, uint32_t din, uint32_t t0, uint32_t limit)
{
    static_assert(MODE == 1 || MODE == 2, "walk 0 is c_walk0");
    const uint32_t t1 = t0 + C_TILE;
    uint32_t lk = 0xFFFFFFFFu, mp = 0;
    bool done = false;
    while (!done) {                                  // single exit: the warp reconverges before the next barrier
        if (p >= t1) { lk = C_END; mp = p; done = true; continue; }
        const uint32_t rel = p - t0, j = rel / C_SEG;
        if (din) {
            // inside a match with offset din that covered everything up to the boundary p
            if (j != k && ((T.M[rel >> 5] >> (rel & 31)) & 1) && T.off[rel] == din) {
                lk = j; mp = p; done = true; continue;          // chain j's own first step is this very match
            }
            uint32_t cap = p < limit ? limit - p : 0; if (cap > C_SEG) cap = C_SEG;
            const uint32_t E = c_cont_len(in, p, din, cap);
            if constexpr (MODE == 2) {
                if (E) { atomicOr(&X.Sel[rel >> 5], 1u << (rel & 31)); atomicOr(&X.Cont[rel >> 5], 1u << (rel & 31)); X.clen[j] = (uint8_t)E; }
            }
            p += E;
            if (E != C_SEG) din = 0;
            continue;
        }
        if constexpr (MODE == 2) {
            if (j == k) {
                // Free in the own segment: the path entered this chain on its walk-0 trajectory, so walk 0's pieces
                // from p on are its V bits.  Mark them at once and leave the segment where walk 0 left it.
                const uint32_t s0 = rel & ~(C_SEG - 1);
                const uint32_t own = (uint32_t)reinterpret_cast<const uint16_t*>(T.V)[k] & (0xFFFFu << (rel & 15));
                p = t0 + s0 + C_SEG;                                  // no piece left: free at the segment's end
                if (own) {
                    atomicOr(&X.Sel[rel >> 5], own << (rel & 16));
                    const uint32_t qr = s0 + 31 - __clz(own), q = t0 + qr;
                    uint32_t B = t0 + s0 + C_SEG;
                    if (B - q < 4) B += C_SEG;
                    const uint32_t e = q + 4 + ((T.len4[qr >> 3] >> (4 * (qr & 7))) & 15u);
                    if (e == B) din = T.off[qr];                      // still inside the match at the boundary
                    if (e > p) p = e;
                }
                continue;
            }
        }
        if (j != k && (rel & (C_SEG - 1)) == 0) { lk = j; mp = p; done = true; continue; }
        uint32_t bits = (T.M[rel >> 5] >> (rel & 16)) & 0xFFFFu;     // this segment's 16 candidate bits
        bits &= 0xFFFFu << (rel & 15);
        if (!bits) {                                                   // segment exhausted: free at its end
            if (j + 1 == C_CHAINS) { lk = C_END; mp = t1; done = true; }
            else { lk = j + 1; mp = t0 + (j + 1) * C_SEG; done = true; }   // (reached outside the own segment only)
            continue;
        }
        const uint32_t qr = (rel & ~15u) + (__ffs(bits) - 1), q = t0 + qr;
        if (j != k && ((T.V[qr >> 5] >> (qr & 31)) & 1)) { lk = j; mp = q; done = true; continue; }
        uint32_t B = (q & ~(C_SEG - 1)) + C_SEG;                     // cut at the first boundary leaving >= 4 bytes
        if (B - q < 4) B += C_SEG;
        const uint32_t d = T.off[qr];
        uint32_t L4;
        if constexpr (MODE == 2) {
            L4 = (T.len4[qr >> 3] >> (4 * (qr & 7))) & 15u;
            atomicOr(&X.Sel[qr >> 5], 1u << (qr & 31));
        } else {
            L4 = c_piece_len4(in, q, d, B < limit ? B : limit);       // q + 4 <= limit always
            atomicOr(&T.len4[qr >> 3], L4 << (4 * (qr & 7)));
        }
        p = q + 4 + L4;
        if (p == B) din = d;                                          // reached the boundary: still inside the match
    }
    if constexpr (MODE == 1) { X.link[k] = (uint16_t)lk; X.mpos[k] = mp; if (lk == C_END) X.xdin[k] = (uint16_t)din; }
}

// Walk 0 of chain k: its own segment only, from p (the segment start, or the tile's entry e in chain k0, with the
// offset din of the match open there).  The segment's 16 M bits are loaded once; a step loads the piece's offset and
// measures it in one compare.  Writes the chain's V half, the two len4 words of its segment (plain stores) and its exit
// state (X.xfree/X.xdin).
__device__ __forceinline__ void c_walk0(const uint8_t* in, PipeTile& T, LzFront& X, uint32_t k, uint32_t p, uint32_t din, uint32_t t0, uint32_t limit)
{
    const uint32_t s0 = t0 + k * C_SEG, s1 = s0 + C_SEG;
    const uint32_t mb = reinterpret_cast<const uint16_t*>(T.M)[k];
    uint32_t vb = 0, lo = 0, hi = 0;
    if (din) {                                       // entered at the segment start inside a match
        uint32_t cap = p < limit ? limit - p : 0; if (cap > C_SEG) cap = C_SEG;
        const uint32_t E = c_cont_len(in, p, din, cap);
        p += E;
        if (E != C_SEG) din = 0;
    }
    while (p < s1) {                                 // free inside the segment (din != 0 only at p == s1)
        const uint32_t bits = mb & (0xFFFFu << (p - s0));
        if (!bits) { p = s1; break; }                // segment exhausted: free at its end
        const uint32_t qr = __ffs(bits) - 1, q = s0 + qr;
        uint32_t B = s0 + C_SEG;                     // cut at the first boundary leaving >= 4 bytes
        if (B - q < 4) B += C_SEG;
        const uint32_t d = T.off[q - t0];
        const uint32_t L4 = c_piece_len4(in, q, d, B < limit ? B : limit);   // q + 4 <= limit always
        vb |= 1u << qr;
        if (qr & 8) hi |= L4 << (4 * (qr & 7)); else lo |= L4 << (4 * qr);
        p = q + 4 + L4;
        if (p == B) din = d;                         // reached the boundary: still inside the match
    }
    reinterpret_cast<uint16_t*>(T.V)[k] = (uint16_t)vb;
    *reinterpret_cast<uint2*>(&T.len4[2 * k]) = make_uint2(lo, hi);
    X.xfree[k] = p; X.xdin[k] = (uint16_t)din;
}

__device__ __forceinline__ uint32_t c_seq_size(uint32_t lit, uint32_t L)
{
    uint32_t s = 1 + lit + 2;
    if (lit >= 15) s += 1 + (lit - 15) / 255;
    if (L - 4 >= 15) s += 1 + (L - 19) / 255;
    return s;
}

// writes one LZ4 sequence at dst + o (token, lengths, offset) and returns its size.  No serial 255-runs: the 255 bytes of a
// literal length exist only when lit >= 270 > C_LONGLIT, and the warp that copies that literal run writes them
// (c_long_job); literal runs longer than C_LONGLIT and long match-length runs are queued as jobs in K.longl (K: LzBack,
// or the high-compression class's own job list).
template <class KL>
__device__ __forceinline__ uint32_t c_emit_seq(const uint8_t* in, KL& K, uint32_t& nlong, uint8_t* dst, uint32_t o,
                                               uint32_t lit_start, uint32_t lit, uint32_t off, uint32_t mlen)
{
    static_assert(C_LONGLIT < 15 + 255, "literal-length 255 runs must imply the cooperative path");
    uint8_t* op = dst + o;
    const uint32_t ml = mlen - 4;
    *op++ = (uint8_t)(((lit >= 15 ? 15u : lit) << 4) | (ml >= 15 ? 15u : ml));
    if (lit >= 15) { const uint32_t x = lit - 15, nf = x / 255; op += nf; *op++ = (uint8_t)(x - nf * 255); }
    if (lit <= C_LONGLIT) { for (uint32_t i = 0; i < lit; i++) op[i] = in[lit_start + i]; }
    else { const uint32_t s = atomicAdd(&nlong, 1u); K.longl[2 * s] = lit_start | (lit << 16); K.longl[2 * s + 1] = (uint32_t)(op - dst); }
    op += lit;
    *op++ = (uint8_t)off; *op++ = (uint8_t)(off >> 8);
    if (ml >= 15) {
        const uint32_t x = ml - 15, nf = x / 255;
        if (nf > 4) { const uint32_t s = atomicAdd(&nlong, 1u); K.longl[2 * s] = nf; K.longl[2 * s + 1] = (uint32_t)(op - dst) | 0x80000000u; op += nf; }
        else for (uint32_t i = 0; i < nf; i++) *op++ = 255;
        *op++ = (uint8_t)(x - nf * 255);
    }
    return (uint32_t)(op - (dst + o));
}

// one job of the long list, done by `nthr` threads (thread index t): a literal run with the 255 bytes of its length
// field, or a run of 255 bytes of a match length
template <class KL>
__device__ __forceinline__ void c_long_job(const uint8_t* in, const KL& K, uint8_t* dst, uint32_t s, uint32_t t, uint32_t nthr)
{
    const uint32_t a = K.longl[2 * s], dp = K.longl[2 * s + 1];
    if (dp & 0x80000000u) { uint8_t* q = dst + (dp & 0x7FFFFFFFu); for (uint32_t i = t; i < a; i += nthr) q[i] = 255; return; }
    const uint32_t sp = a & 0xFFFFu, ln = a >> 16;
    for (uint32_t i = t; i < ln; i += nthr) dst[dp + i] = in[sp + i];
    const uint32_t nf = (ln - 15) / 255;                       // ln > C_LONGLIT >= 15
    uint8_t* q = dst + dp - 1 - nf;
    for (uint32_t i = t; i < nf; i += nthr) q[i] = 255;
}

#include "lz4_pipe.cuh"

// ============================================================================ Zstandard encoder: LZ77 + entropy stage
// The LZ4 compressor's front and back end (lz4_pipe.cuh) run by one team of 256 threads, tile after tile, and the
// sequences go to the scratch instead of an LZ4 stream.  Every 4 tiles the entropy stage turns what was gathered into
// a Zstandard block; it is written for the whole CTA, and its shared memory reuses the tile arrays, which are dead
// between tiles.
struct __align__(16) ZstdSmem {
    LzStage  stage;
    uint32_t tab[1 << C_HASHLOG];         // hash -> 1 + position
    union {
        struct { PipeTile tile; LzFront fe; LzBack be; } lz;
        ZEnt ent;
    };
    ZFseShared fse;                       // predefined FSE encoding tables
    __align__(16) uint32_t scanws[40];    // team_exscan* (16 words) and the entropy stage's block_exscan (33 words)
    uint32_t any[2];                      // tile has a candidate, per tile parity (lz_candidates)
    uint32_t nlong;
    uint64_t mbar;
};
static_assert(sizeof(ZstdSmem) + 1024 <= (228 * 1024) / 2, "two CTAs per SM");

__global__ void __launch_bounds__(P_TEAM, 2)
zstd_blocks_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                   uint32_t bpc, uint8_t* __restrict__ tmp, uint32_t* __restrict__ blk_csize, uint32_t nblocks,
                   ZScratch* __restrict__ zscratch)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    ZstdSmem& S = *reinterpret_cast<ZstdSmem*>(smem_raw);
    constexpr uint32_t NT = P_TEAM;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    PipeTile& T = S.lz.tile;
    LzBack& K = S.lz.be;
    ZScratch* const zs = zscratch + blockIdx.x;
    auto cta_sync = [] () { CTA_SYNC(); };
    z_load_fse_shared(S.fse, tid, NT);

    for (uint32_t blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const uint32_t chunk = blk / bpc, bic = blk % bpc;
        const uint64_t cbase = (uint64_t)chunk * chunk_size;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, chunk, in_bytes, chunk_size);
        const uint64_t boff = (uint64_t)bic * LZ4_BLK;
        uint32_t n = 0;
        if (boff < cbytes) n = (uint32_t)((cbytes - boff) < LZ4_BLK ? (cbytes - boff) : LZ4_BLK);
        if (n == 0) { if (tid == 0) blk_csize[blk] = 0; continue; }
        uint8_t* dst = tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE;

        CTA_SYNC();                                       // previous block fully consumed
        if (tid == 0) { S.nlong = 0; S.any[0] = 0; S.any[1] = 0; }
        lz_stage<NT>(S.stage, S.tab, &S.mbar, in + cbase + boff, n, tid);

        const uint32_t limit = n >= 5 ? n - 5 : 0;        // matches end at or before n-5
        uint32_t e = 0, e_din = 0, out_pos = 0;
        LzPending pd = {0, 0, 0, 0, 0};
        // sequences / literals gathered for the current sub-block, content already emitted into blocks
        uint32_t z_nseq = 0, z_nlit = 0, z_pos = 0;
        const bool z_last_of_chunk = (boff + n == cbytes);

        for (uint32_t ti = 0, t0 = 0; t0 < n; ti++, t0 += C_TILE) {
            const uint32_t t1 = t0 + C_TILE;
            const bool has_match = lz_candidates<0>(S.stage.in, S.tab, T, S.any, ti & 1, t0, n, tid, lane);
            if (lz_chains<0>(S.stage.in, T, S.lz.fe, has_match, e, e_din, t0, limit, tid, lane)) {
                uint32_t tile_end;
                const uint32_t nh = lz_heads<0>(S.stage.in, T, K, S.scanws, pd, tile_end, t0, limit, tid, lane);
                if (nh) {
                    const LzRun R = lz_seq_run(T, K, pd, nh, t0, tid);
                    uint32_t sz = 0;                          // (sequences << 18) | literal bytes
#pragma unroll
                    for (uint32_t k = 0; k < LZ_SPT; k++) if (k < R.cnt) sz += (1u << 18) | R.lit[k];
                    uint32_t total;
                    const uint32_t o = team_exscan1<0>(sz, S.scanws, 0, &total, wid, lane);
                    uint32_t si = z_nseq + (o >> 18), li = z_nlit + (o & 0x3FFFF);
#pragma unroll
                    for (uint32_t k = 0; k < LZ_SPT; k++) {
                        if (k >= R.cnt) break;
                        ZSeq q; q.litlen = R.lit[k]; q.off = (uint16_t)R.off[k]; q.mlen = (uint16_t)R.len[k];
                        zs->seq[si++] = q;
                        if (R.lit[k] <= C_LONGLIT) { for (uint32_t i = 0; i < R.lit[k]; i++) zs->lit[li + i] = S.stage.in[R.lit0[k] + i]; }
                        else { const uint32_t s = atomicAdd(&S.nlong, 1u); K.longl[2 * s] = R.lit0[k] | (R.lit[k] << 16); K.longl[2 * s + 1] = li; }
                        li += R.lit[k];
                    }
                    team_sync<0>();
                    // long literal runs, one warp each (a plain copy: unlike the LZ4 jobs, no length field goes with them)
                    const uint32_t nl = S.nlong;
                    for (uint32_t s = wid; s < nl; s += NT / 32) {
                        const uint32_t a = K.longl[2 * s], dp = K.longl[2 * s + 1], sp = a & 0xFFFFu, ln = a >> 16;
                        for (uint32_t i = lane; i < ln; i += 32) zs->lit[dp + i] = S.stage.in[sp + i];
                    }
                    z_nseq += total >> 18; z_nlit += total & 0x3FFFF;
                    lz_next_pending(T, K, pd, nh, tile_end, t0);
                    team_sync<0>();
                    if (tid == 0) S.nlong = 0;
                }
            }

            // ---------------- close a block every 4 tiles (not at the end of the window: the final flush does that)
            if ((ti & 3) == 3 && t1 < n) {
                CTA_SYNC();
                // trailing literals up to C: everything before the pending match (or all parsed bytes when nothing is pending)
                const uint32_t cover = pd.valid ? pd.lit : z_pos;
                const uint32_t C = pd.valid ? pd.start : t1;
                for (uint32_t i = tid; i < C - cover; i += NT) zs->lit[z_nlit + i] = S.stage.in[cover + i];
                const uint32_t nl = z_nlit + (C - cover);
                CTA_SYNC();
                if (C > z_pos) out_pos += z_encode_block(S.ent, S.fse, zs, z_nseq, nl, S.stage.in + z_pos, C - z_pos, false, dst + out_pos, S.scanws, cta_sync);
                z_pos = C; pd.lit = C;                  // literals before C are emitted: the next sequence's literal run starts here
                z_nseq = 0; z_nlit = 0;
            }
        }

        // ---------------- flush the pending sequence + last literals
        CTA_SYNC();
        uint32_t anchor = z_pos;
        if (pd.valid) {
            anchor = pd.end;
            const uint32_t ll = pd.start - pd.lit;
            if (tid == 0) { ZSeq q; q.litlen = ll; q.off = (uint16_t)pd.off; q.mlen = (uint16_t)(pd.end - pd.start); zs->seq[z_nseq] = q; }
            for (uint32_t i = tid; i < ll; i += NT) zs->lit[z_nlit + i] = S.stage.in[pd.lit + i];
            z_nseq++; z_nlit += ll;
        }
        for (uint32_t i = tid; i < n - anchor; i += NT) zs->lit[z_nlit + i] = S.stage.in[anchor + i];
        z_nlit += n - anchor;
        CTA_SYNC();
        // the frame's last block carries the Last_Block bit; an empty raw block does when nothing is left
        out_pos += z_encode_block(S.ent, S.fse, zs, z_nseq, z_nlit, S.stage.in + z_pos, n - z_pos, z_last_of_chunk, dst + out_pos, S.scanws, cta_sync);
        if (tid == 0) blk_csize[blk] = out_pos;
    }
}

#include "zstd_lazy.cuh"
#include "lz4_hc.cuh"

// ============================================================================ XXH32 (content checksum)
// One warp per buffer.  XXH32 is four serial accumulator chains (one per 32-bit word of every 16-byte
// stripe), so the latency floor per buffer is (len/16) * ~12 cycles; everything else is about keeping the
// four chain lanes fed: all 32 lanes stream the buffer with 16-byte loads (X_DEPTH tiles of 512 B in flight
// per warp), park each tile in a per-warp shared-memory slot, and lanes 0..3 walk the slot word by word.
#define X_WARPS 8
#define X_DEPTH 4
// XXH32 accumulator j (seed 0) before the first stripe
__device__ __forceinline__ uint32_t xxh32_acc0(uint32_t j) { return j == 0 ? XXP1 + XXP2 : j == 1 ? XXP2 : j == 2 ? 0u : 0u - XXP1; }

// Folds the ns 16-byte stripes at p into the accumulators: lane l carries accumulator l & 3 in and out.
__device__ __forceinline__ uint32_t warp_xxh32_stripes(const uint8_t* p, uint64_t ns, uint4 (*tile)[32], uint32_t lane, uint32_t acc)
{
    const uint32_t j = lane & 3;
    uint64_t s = 0;
    if (((uintptr_t)p & 15) == 0) {
        const uint4* v = reinterpret_cast<const uint4*>(p);
        const uint64_t nt = ns >> 5;                         // full tiles of 32 stripes
        uint4 r[X_DEPTH];
#pragma unroll
        for (int d = 0; d < X_DEPTH; d++) if ((uint64_t)d < nt) r[d] = __ldg(v + (uint64_t)d * 32 + lane);
        for (uint64_t t = 0; t < nt; t += X_DEPTH) {
#pragma unroll
            for (int d = 0; d < X_DEPTH; d++) {
                if (t + d < nt) {
                    uint4* slot = tile[d & 1];
                    slot[lane] = r[d];
                    if (t + d + X_DEPTH < nt) r[d] = __ldg(v + (t + d + X_DEPTH) * 32 + lane);
                    __syncwarp();
                    const uint32_t* w = reinterpret_cast<const uint32_t*>(slot) + j;
#pragma unroll
                    for (int q = 0; q < 32; q++) acc = xxh32_round(acc, w[4 * q]);
                    __syncwarp();
                }
            }
        }
        s = nt << 5;
    }
    // remaining stripes (and unaligned buffers): the 4 chain lanes read global memory directly
    if (((uintptr_t)p & 3) == 0) { const uint32_t* w = reinterpret_cast<const uint32_t*>(p) + j; for (; s < ns; s++) acc = xxh32_round(acc, __ldg(w + 4 * s)); }
    else for (; s < ns; s++) acc = xxh32_round(acc, ldg_le32(p + 16 * s + 4 * j));
    return acc;
}

// XXH32 (seed 0) of p[0, n) by one warp; tile = the warp's 1 KiB of shared memory.  The hash is valid on lane 0.
__device__ __forceinline__ uint32_t warp_xxh32(const uint8_t* p, uint64_t n, uint4 (*tile)[32], uint32_t lane)
{
    const uint64_t ns = n >> 4;                              // 16-byte stripes
    const uint32_t acc = warp_xxh32_stripes(p, ns, tile, lane, xxh32_acc0(lane & 3));
    const uint32_t a1 = __shfl_sync(ZMT_FULL_MASK, acc, 0), a2 = __shfl_sync(ZMT_FULL_MASK, acc, 1);
    const uint32_t a3 = __shfl_sync(ZMT_FULL_MASK, acc, 2), a4 = __shfl_sync(ZMT_FULL_MASK, acc, 3);
    uint32_t h = 0;
    if (lane == 0) {
        h = n >= 16 ? rotl32(a1, 1) + rotl32(a2, 7) + rotl32(a3, 12) + rotl32(a4, 18) : XXP5;
        h += (uint32_t)n;
        const uint8_t* q = p + (ns << 4);
        const uint8_t* end = p + n;
        while (q + 4 <= end) { h = rotl32(h + ldg_le32(q) * XXP3, 17) * XXP4; q += 4; }
        while (q < end) { h = rotl32(h + (*q) * XXP5, 11) * XXP1; q++; }
        h ^= h >> 15; h *= XXP2; h ^= h >> 13; h *= XXP3; h ^= h >> 16;
    }
    return h;
}

__global__ void __launch_bounds__(32 * X_WARPS)
xxh32_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ offs, const uint64_t* __restrict__ lens,
             const uint32_t* __restrict__ lens32, uint64_t stride, uint64_t total_bytes, uint32_t* __restrict__ out, uint32_t nbuf)
{
    __shared__ uint4 tile[X_WARPS][2][32];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t g = blockIdx.x * X_WARPS + wid;
    if (g >= nbuf) return;                                   // whole warp leaves together
    uint64_t off, n;
    if (offs) { off = offs[g]; n = lens ? lens[g] : offs[g + 1] - off; }
    else { off = (uint64_t)g * stride; n = zmt_chunk_len(lens32, g, total_bytes, (uint32_t)stride); }
    const uint32_t h = warp_xxh32(base + off, n, tile[wid], lane);
    if (lane == 0) out[g] = h;
}

// Segments of LZ4F frames (zmt_lz4_segment): one warp per segment folds its decoded bytes into the frame's running
// XXH32 — the bytes pending from the previous segment are topped up to a stripe first, what is left behind the last
// whole stripe waits for the next segment — and advances `produced`.  The last segment finalises the hash into out[f].
__global__ void __launch_bounds__(32 * X_WARPS)
lz4_segment_xxh32_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ offs, const unsigned long long* __restrict__ lens,
                         const uint32_t* __restrict__ status, zmt_lz4_segment* __restrict__ seg, uint32_t* __restrict__ out, uint32_t nbuf)
{
    __shared__ uint4 tile[X_WARPS][2][32];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t f = blockIdx.x * X_WARPS + wid;
    if (f >= nbuf || (status[f] & 0xFF) != 0) return;       // a failed segment ends the frame: its state no longer matters
    zmt_lz4_segment& S = seg[f];
    const bool first = (S.flags & ZMT_SEG_FIRST) != 0;
    const uint8_t* p = base + offs[f];
    const uint64_t n = lens[f];
    uint8_t pend[16];
    uint32_t pl = first ? 0u : S.pending_len;
    for (uint32_t i = 0; i < 16; i++) pend[i] = i < pl ? S.pending[i] : (uint8_t)0;
    uint32_t acc = first ? xxh32_acc0(lane & 3) : S.acc[lane & 3];
    uint64_t k = 0;                                          // bytes of this segment that top up the pending stripe
    if (pl) {
        k = n < 16 - pl ? n : 16 - pl;
        for (uint32_t i = 0; i < (uint32_t)k; i++) pend[pl + i] = p[i];
        pl += (uint32_t)k;
        if (pl == 16) { acc = xxh32_round(acc, (uint32_t)pend[4 * (lane & 3)] | ((uint32_t)pend[4 * (lane & 3) + 1] << 8) |
                                                ((uint32_t)pend[4 * (lane & 3) + 2] << 16) | ((uint32_t)pend[4 * (lane & 3) + 3] << 24)); pl = 0; }
    }
    const uint64_t ns = (n - k) >> 4;
    acc = warp_xxh32_stripes(p + k, ns, tile[wid], lane, acc);
    const uint64_t t0 = k + (ns << 4);                       // the tail behind the last whole stripe
    if (t0 < n) { for (uint32_t i = 0; i < (uint32_t)(n - t0); i++) pend[i] = p[t0 + i]; pl = (uint32_t)(n - t0); }
    const uint64_t total = (first ? 0 : S.produced) + n;
    const uint32_t a1 = __shfl_sync(ZMT_FULL_MASK, acc, 0), a2 = __shfl_sync(ZMT_FULL_MASK, acc, 1);
    const uint32_t a3 = __shfl_sync(ZMT_FULL_MASK, acc, 2), a4 = __shfl_sync(ZMT_FULL_MASK, acc, 3);
    if (lane != 0) return;
    S.acc[0] = a1; S.acc[1] = a2; S.acc[2] = a3; S.acc[3] = a4;
    for (uint32_t i = 0; i < 16; i++) S.pending[i] = pend[i];
    S.pending_len = (uint16_t)pl; S.produced = total;
    if (!(S.flags & ZMT_SEG_LAST)) return;
    uint32_t h = total >= 16 ? rotl32(a1, 1) + rotl32(a2, 7) + rotl32(a3, 12) + rotl32(a4, 18) : XXP5;
    h += (uint32_t)total;
    uint32_t i = 0;
    for (; i + 4 <= pl; i += 4) h = rotl32(h + ((uint32_t)pend[i] | ((uint32_t)pend[i + 1] << 8) | ((uint32_t)pend[i + 2] << 16) | ((uint32_t)pend[i + 3] << 24)) * XXP3, 17) * XXP4;
    for (; i < pl; i++) h = rotl32(h + pend[i] * XXP5, 11) * XXP1;
    h ^= h >> 15; h *= XXP2; h ^= h >> 13; h *= XXP3; h ^= h >> 16;
    out[f] = h;
}

// ============================================================================ frame pack
// frame bytes = 12 (skippable hdr) + 4 magic + 2 (FLG,BD) + [8 content size] + 1 HC
//               + sum(4 + block bytes) + 4 end mark + 4 content checksum
__global__ void lz4_frame_sizes_kernel(const uint32_t* __restrict__ blk_csize, uint64_t in_bytes, uint32_t chunk_size,
                                       const uint32_t* __restrict__ chunk_bytes, uint32_t bpc, uint32_t nchunks, uint64_t* __restrict__ frame_size)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const uint64_t cbytes = zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size);
    uint64_t sz = 12 + 4 + 2 + (cbytes ? 8 : 0) + 1 + 4 + 4;
    for (uint32_t b = 0; b < bpc; b++) {
        const uint32_t cs = blk_csize[c * bpc + b];
        if (cs) sz += 4 + (cs & 0x7FFFFFFFu);
    }
    frame_size[c] = sz;
}

// Single-CTA exclusive scan of uint64 sizes -> offsets[0..n] (offsets[n] = total).
__global__ void __launch_bounds__(1024) scan_u64_kernel(const uint64_t* __restrict__ sizes, uint64_t* __restrict__ offsets, uint32_t n)
{
    __shared__ unsigned long long ws[33];
    __shared__ unsigned long long carry;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        unsigned long long v = i < n ? sizes[i] : 0, inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { unsigned long long y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc += y; }
        if (lane == 31) ws[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            unsigned long long x = ws[lane], xi = x;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { unsigned long long y = __shfl_up_sync(ZMT_FULL_MASK, xi, d); if (lane >= (uint32_t)d) xi += y; }
            ws[lane] = xi - x;
            if (lane == 31) ws[32] = xi;
        }
        __syncthreads();
        const unsigned long long c0 = carry;
        if (i < n) offsets[i] = c0 + ws[wid] + inc - v;
        __syncthreads();
        if (threadIdx.x == 0) carry = c0 + ws[32];
        __syncthreads();
    }
    if (threadIdx.x == 0) offsets[n] = carry;
}

// One CTA per (chunk, block): copies the block payload to its final place; block 0 also writes
// the headers, the last block the end mark + checksum.  indep: the FLG block-independence bit, 0x20 for the level-1
// class's independent blocks, 0 for the linked blocks of levels 10-12.
__global__ void __launch_bounds__(256)
lz4_frame_pack_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes, uint32_t bpc,
                      const uint8_t* __restrict__ tmp, const uint32_t* __restrict__ blk_csize,
                      const uint32_t* __restrict__ chk, const uint64_t* __restrict__ frame_off,
                      uint8_t* __restrict__ out, uint32_t nblocks, uint32_t indep)
{
    for (uint32_t blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const uint32_t c = blk / bpc, b = blk % bpc;
        const uint64_t cbase = (uint64_t)c * chunk_size;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size);
        const uint32_t hdr = 12 + 4 + 2 + (cbytes ? 8 : 0) + 1;
        uint8_t* f = out + frame_off[c];
        const uint32_t cs = blk_csize[blk];
        if (cs == 0 && b != 0) continue;                   // block beyond the end of a short chunk
        uint64_t pos = hdr;                                // payload offset of this block inside the frame
        for (uint32_t k = 0; k < b; k++) { const uint32_t x = blk_csize[c * bpc + k]; if (x) pos += 4 + (x & 0x7FFFFFFFu); }
        const bool last = (b + 1 == bpc) || blk_csize[blk + 1] == 0;
        if (threadIdx.x == 0) {
            if (b == 0) {
                const uint64_t fsz = frame_off[c + 1] - frame_off[c];
                uint8_t h[10];
                stg_le32(f, 0x184D2A50u); stg_le32(f + 4, 4); stg_le32(f + 8, (uint32_t)(fsz - 12));
                stg_le32(f + 12, 0x184D2204u);
                h[0] = (uint8_t)((cbytes ? 0x4C : 0x44) | indep); h[1] = 0x40;
                for (int i = 0; i < 8; i++) h[2 + i] = (uint8_t)(cbytes >> (8 * i));
                const uint32_t hl = cbytes ? 10 : 2;
                for (uint32_t i = 0; i < hl; i++) f[16 + i] = h[i];
                f[16 + hl] = (uint8_t)(xxh32_small(h, hl, 0) >> 8);
            }
            if (cs) stg_le32(f + pos, cs);
            if (last) {
                const uint64_t e = pos + (cs ? 4 + (cs & 0x7FFFFFFFu) : 0);
                stg_le32(f + e, 0); stg_le32(f + e + 4, chk[c]);
            }
        }
        if (cs) {
            const uint8_t* s = (cs & 0x80000000u) ? in + cbase + (uint64_t)b * LZ4_BLK : tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE;
            coop_copy_g2g(f + pos + 4, s, cs & 0x7FFFFFFFu, threadIdx.x, blockDim.x);
        }
    }
}

// ============================================================================ decoder
#include "lz4_decode.cuh"

// ============================================================================ zstd frame pack
// frame = 12 (skippable hdr) + magic 4 + FHD 1 + FCS (1 / 2 / 4) + the blocks of every 64 KiB window (+ an empty
// last block for an empty chunk); no checksum, single segment — the layout ZSTD_compress gives the reference
// (SURVEY.md Appendix A: 28 B5 2F FD A0 <LE32 size> for 1 MiB, 28 B5 2F FD 20 00 01 00 00 for empty input).
__device__ __forceinline__ uint32_t zstd_fcs_bytes(uint64_t n) { return n <= 255 ? 1u : n <= 65791 ? 2u : 4u; }

// Dictionary_ID field: 1, 2 or 4 bytes for IDs below 256, below 65536, or larger (FHD bits 0-1 = 1, 2, 3), none for ID 0
__device__ __forceinline__ uint32_t zstd_did_bytes(uint32_t id) { return id == 0 ? 0u : id < 256 ? 1u : id < 65536 ? 2u : 4u; }

// DICT: the frames carry the Dictionary_ID of the index cd (compressed against it, zmt_zstd_compress_dict_device)
template <bool DICT>
__global__ void zstd_frame_sizes_kernel(const uint32_t* __restrict__ blk_csize, uint64_t in_bytes, uint32_t chunk_size,
                                        const uint32_t* __restrict__ chunk_bytes, uint32_t bpc, uint32_t nchunks, uint64_t* __restrict__ frame_size,
                                        const ZlCDict* __restrict__ cd)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const uint64_t cbytes = zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size);
    uint64_t sz = 12 + 4 + 1 + zstd_fcs_bytes(cbytes);
    if (DICT) sz += zstd_did_bytes(cd->dict_id);
    if (cbytes == 0) sz += 3;
    for (uint32_t b = 0; b < bpc; b++) sz += blk_csize[c * bpc + b];
    frame_size[c] = sz;
}

template <bool DICT>
__global__ void __launch_bounds__(256)
zstd_frame_pack_kernel(uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes, uint32_t bpc,
                       const uint8_t* __restrict__ tmp, const uint32_t* __restrict__ blk_csize, const uint64_t* __restrict__ frame_off,
                       uint8_t* __restrict__ out, uint32_t nblocks, const ZlCDict* __restrict__ cd)
{
    const uint32_t did = DICT ? cd->dict_id : 0u, dl = DICT ? zstd_did_bytes(did) : 0u;
    for (uint32_t blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const uint32_t c = blk / bpc, b = blk % bpc;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size);
        const uint32_t fl = zstd_fcs_bytes(cbytes), hdr = 12 + 4 + 1 + dl + fl;
        uint8_t* f = out + frame_off[c];
        const uint32_t cs = blk_csize[blk];
        if (cs == 0 && b != 0) continue;
        uint64_t pos = hdr;
        for (uint32_t k = 0; k < b; k++) pos += blk_csize[c * bpc + k];
        if (threadIdx.x == 0 && b == 0) {
            const uint64_t fsz = frame_off[c + 1] - frame_off[c];
            stg_le32(f, 0x184D2A50u); stg_le32(f + 4, 4); stg_le32(f + 8, (uint32_t)(fsz - 12));
            stg_le32(f + 12, 0xFD2FB528u);
            f[16] = fl == 1 ? 0x20 : fl == 2 ? 0x60 : 0xA0;
            if (!DICT || dl == 0) {
                if (fl == 1) f[17] = (uint8_t)cbytes;
                else if (fl == 2) { const uint32_t v = (uint32_t)cbytes - 256; f[17] = (uint8_t)v; f[18] = (uint8_t)(v >> 8); }
                else stg_le32(f + 17, (uint32_t)cbytes);
            } else {                                                    // FHD, Dictionary_ID, Frame_Content_Size
                f[16] |= dl == 1 ? 1 : dl == 2 ? 2 : 3;
                for (uint32_t k = 0; k < dl; k++) f[17 + k] = (uint8_t)(did >> (8 * k));
                uint8_t* fcs = f + 17 + dl;
                if (fl == 1) fcs[0] = (uint8_t)cbytes;
                else if (fl == 2) { const uint32_t v = (uint32_t)cbytes - 256; fcs[0] = (uint8_t)v; fcs[1] = (uint8_t)(v >> 8); }
                else stg_le32(fcs, (uint32_t)cbytes);
            }
            if (cbytes == 0) { f[hdr] = 1; f[hdr + 1] = 0; f[hdr + 2] = 0; }        // empty raw last block
        }
        if (cs) coop_copy_g2g(f + pos, tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE, cs, threadIdx.x, blockDim.x);
    }
}

// ---- predefined FSE encoding tables (RFC 8878 §3.1.1.3.2.2.1 distributions; FSE_buildCTable construction [ext])
static void zstd_build_ctable(ZFseCTable& T, const int16_t* norm, int nsym, int log)
{
    const int size = 1 << log, step = (size >> 1) + (size >> 3) + 3;
    int cumul[64], high = size - 1, pos = 0;
    uint8_t sym[64];
    memset(&T, 0, sizeof(T)); T.log = (uint32_t)log;
    cumul[0] = 0;
    for (int u = 1; u <= nsym; u++) {
        if (norm[u - 1] == -1) { cumul[u] = cumul[u - 1] + 1; sym[high--] = (uint8_t)(u - 1); }
        else cumul[u] = cumul[u - 1] + norm[u - 1];
    }
    for (int s = 0; s < nsym; s++)
        for (int i = 0; i < norm[s]; i++) { sym[pos] = (uint8_t)s; do { pos = (pos + step) & (size - 1); } while (pos > high); }
    for (int u = 0; u < size; u++) { const int s = sym[u]; T.state[cumul[s]++] = (uint16_t)(size + u); }
    int total = 0;
    for (int s = 0; s < nsym; s++) {
        const int n = norm[s];
        if (n == 0) { T.dnb[s] = ((log + 1) << 16) - (1 << log); T.dfs[s] = 0; }
        else if (n == -1 || n == 1) { T.dnb[s] = (log << 16) - (1 << log); T.dfs[s] = total - 1; total++; }
        else {
            int hb = 0; while ((1 << (hb + 1)) <= n - 1) hb++;
            const int maxBitsOut = log - hb, minStatePlus = n << maxBitsOut;
            T.dnb[s] = (maxBitsOut << 16) - minStatePlus; T.dfs[s] = total - n; total += n;
        }
    }
}

static int zstd_tables_init()
{
    static std::mutex mu; static bool done[64];   // devices whose __constant__ copies are loaded (contexts may run on several host threads)
    int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return ZMT_ST_CUDA;
    std::lock_guard<std::mutex> guard(mu);
    if (done[dev]) return ZMT_ST_OK;
    ZFseCTable t;
    zstd_build_ctable(t, ZSTD_LL_NORM, 36, 6); if (cudaMemcpyToSymbol(c_fse_ll, &t, sizeof(t)) != cudaSuccess) return ZMT_ST_CUDA;
    zstd_build_ctable(t, ZSTD_OF_NORM, 29, 5); if (cudaMemcpyToSymbol(c_fse_of, &t, sizeof(t)) != cudaSuccess) return ZMT_ST_CUDA;
    zstd_build_ctable(t, ZSTD_ML_NORM, 53, 6); if (cudaMemcpyToSymbol(c_fse_ml, &t, sizeof(t)) != cudaSuccess) return ZMT_ST_CUDA;
    uint8_t llc[64], mlc[128];
    for (int v = 0; v < 64; v++) { int c = 0; while (c + 1 < 36 && ZSTD_LL_BASE[c + 1] <= (uint32_t)v) c++; llc[v] = (uint8_t)c; }
    for (int v = 0; v < 128; v++) { int c = 0; while (c + 1 < 53 && ZSTD_ML_BASE[c + 1] <= (uint32_t)v + 3) c++; mlc[v] = (uint8_t)c; }
    cudaMemcpyToSymbol(c_ll_code, llc, sizeof(llc)); cudaMemcpyToSymbol(c_ml_code, mlc, sizeof(mlc));
    cudaMemcpyToSymbol(c_ll_base, ZSTD_LL_BASE, sizeof(ZSTD_LL_BASE)); cudaMemcpyToSymbol(c_ml_base, ZSTD_ML_BASE, sizeof(ZSTD_ML_BASE));
    cudaMemcpyToSymbol(c_ll_bits, ZSTD_LL_BITS, sizeof(ZSTD_LL_BITS)); cudaMemcpyToSymbol(c_ml_bits, ZSTD_ML_BITS, sizeof(ZSTD_ML_BITS));
    if (cudaGetLastError() != cudaSuccess) return ZMT_ST_CUDA;
    if (cudaDeviceSynchronize() != cudaSuccess) return ZMT_ST_CUDA;    // the kernels run on non-blocking streams: nothing else orders the table copies before them
    done[dev] = true;
    return ZMT_ST_OK;
}

// ============================================================================ host launchers
// ZSTDMT_B200_DEBUG_SYNC=1: synchronise after every kernel and name the one that failed (debug only)
// ---- optional per-kernel timing (zmt_prof_begin / zmt_prof_end): CUDA events recorded on the launching
// stream around every kernel while enabled (ZmtProfScope, launch.h); used by bench.py for the roofline of the dominant kernel.
struct ZmtProfRec { int id; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::vector<ZmtProfRec> g_prof;
cudaEvent_t zmt_prof_open(cudaStream_t st) { cudaEvent_t a = nullptr; if (g_prof_on) { cudaEventCreate(&a); cudaEventRecord(a, st); } return a; }
void zmt_prof_close(int id, cudaEvent_t a, cudaStream_t st) { cudaEvent_t b; cudaEventCreate(&b); cudaEventRecord(b, st); g_prof.push_back({id, a, b}); }
extern "C" void zmt_prof_begin(void) { for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); } g_prof.clear(); g_prof_on = true; }
// ms[id] = summed device time, count[id] = launches (the caller synchronises the stream first)
extern "C" int zmt_prof_end(double* ms, int* count, int max_ids)
{
    g_prof_on = false;
    for (int i = 0; i < max_ids; i++) { ms[i] = 0; count[i] = 0; }
    for (auto& r : g_prof) {
        float t = 0; cudaEventSynchronize(r.b);
        if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess && r.id < max_ids) { ms[r.id] += t; count[r.id]++; }
        cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    }
    g_prof.clear();
    return ZMT_K_COUNT < max_ids ? ZMT_K_COUNT : max_ids;
}

#ifdef ZMT_PHASE_PROBE
// out[team * ZMT_NPHASE + phase] = cycles summed since the last call (lz4_pipe.cuh); clears the counters.  0 = ok.
extern "C" int zmt_phase_probe_take(unsigned long long* out)
{
    static const unsigned long long zero[2 * ZMT_NPHASE] = {};
    if (cudaMemcpyFromSymbol(out, zmt_phase_cycles, sizeof(zero)) != cudaSuccess) return 1;
    return cudaMemcpyToSymbol(zmt_phase_cycles, zero, sizeof(zero)) != cudaSuccess;
}
#endif

static bool zmt_dbg_check(cudaStream_t st, const char* what)
{
    static int on = -1;
    if (on < 0) on = getenv("ZSTDMT_B200_DEBUG_SYNC") ? 1 : 0;
    if (!on) return true;
    cudaError_t e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { fprintf(stderr, "[zstdmt_b200] %s failed: %s\n", what, cudaGetErrorString(e)); return false; }
    return true;
}

// side stream + fork / join events, one set per (device, host thread): a set must not be shared by two launch sequences
// that interleave, and every host thread enqueues its own sequences in order
struct ZmtSide { cudaStream_t stream = nullptr; cudaEvent_t fork = nullptr, join = nullptr; bool ok = false; };
static ZmtSide zmt_side_stream()
{
    thread_local ZmtSide side[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return ZmtSide();
    ZmtSide& s = side[dev];
    if (!s.ok && !s.stream) {
        bool ok = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) == cudaSuccess;
        ok = ok && cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming) == cudaSuccess;
        ok = ok && cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming) == cudaSuccess;
        if (!ok) cudaGetLastError();
        s.ok = ok;
    }
    return s;
}

extern "C" uint32_t zmt_chunk_count(uint64_t in_bytes, uint32_t chunk_size)
{
    if (chunk_size == 0) return 0;
    const uint64_t n = in_bytes ? (in_bytes + chunk_size - 1) / chunk_size : 1;   // empty input still yields one frame
    return n > 0x7FFFFFFFull ? 0 : (uint32_t)n;
}

static inline uint32_t zmt_bpc(uint32_t chunk_size) { return (uint32_t)(((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK); }   // 64 KiB blocks per chunk

#define ZSTD_MAX_GRID (132u * 2u * 4u)       // the workspace holds one ZScratch per CTA of the largest grid (H100 SXM: 132 SMs)
static inline uint32_t zstd_grid(uint32_t nblocks) { uint32_t m = (uint32_t)(zmt_sm_count() * 2 * 4); if (m > ZSTD_MAX_GRID) m = ZSTD_MAX_GRID; return nblocks < m ? nblocks : m; }

// chunks per group of the chain classes: the per-position arrays (keys, values, prev, best: 16 bytes per position) cover one group at a time
static inline uint32_t zl_group_chunks(uint32_t nchunks, uint32_t chunk_size)
{
    uint32_t g = ZL_GROUP_BYTES / chunk_size;
    if (g == 0) g = 1;
    return g < nchunks ? g : nchunks;
}
static size_t zl_sort_temp_bytes(uint32_t npos, int end_bit = ZL_HASHLOG)
{
    size_t t = 0;
    cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
    if (cub::DeviceRadixSort::SortPairs(nullptr, t, k, v, (int)npos, 0, end_bit) != cudaSuccess) { cudaGetLastError(); return 0; }
    return t;
}

// ---------------------------------------------------------------- encoder arguments
// A batch as every encoder entry point checks and sees it.  The chain classes (zstd levels 6-12, LZ4 levels 10-12) run
// group by group: G chunks, at most npos_max positions (both 0 for the other classes).
struct ZmtBatch {
    const uint8_t* in; uint64_t in_bytes; uint32_t chunk_size; const uint32_t* chunk_bytes; uint32_t nchunks;
    uint32_t bpc, nblocks;
    uint32_t G; uint64_t npos_max;
};
static int zmt_batch(ZmtBatch& b, const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes, uint32_t nchunks, bool chain)
{
    if (chunk_size == 0 || nchunks == 0) return ZMT_ST_BAD_ARG;
    if (!d_chunk_bytes && nchunks != zmt_chunk_count(in_bytes, chunk_size)) return ZMT_ST_BAD_ARG;
    const uint32_t bpc = zmt_bpc(chunk_size);
    if ((uint64_t)nchunks * bpc > 0x7FFFFFFFull) return ZMT_ST_BAD_ARG;
    const uint32_t G = chain ? zl_group_chunks(nchunks, chunk_size) : 0;
    const uint64_t npos_max = (uint64_t)G * chunk_size;
    if (npos_max > 0xFFFFFFFFull) return ZMT_ST_BAD_ARG;
    b = ZmtBatch{(const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, bpc, nchunks * bpc, G, npos_max};
    return ZMT_ST_OK;
}

// ---------------------------------------------------------------- encoder workspaces (ZmtCarve, launch.h)
// npos: the positions of one group for the chain classes, 0 for the others.

// chain classes: keys, values, prev and best of one group, then the radix sort's temporary storage
struct ZlChainWs { uint32_t* arr[4]; void* sort_tmp; size_t sort_cap; };
static void zl_chain_layout(ZmtCarve& c, uint64_t npos, ZlChainWs& ch)
{
    for (int k = 0; k < 4; k++) ch.arr[k] = c.take<uint32_t>(a256(npos * 4));
    ch.sort_cap = zl_sort_temp_bytes((uint32_t)npos);
    ch.sort_tmp = c.take<void>(a256(ch.sort_cap));
}

struct Lz4Ws { uint8_t* tmp; uint32_t* blk_csize; uint32_t* chk; uint64_t* frame_size; ZlChainWs ch; };
static uint64_t lz4_layout(uint8_t* base, uint64_t nchunks, uint64_t nblocks, uint64_t npos, Lz4Ws& w)
{
    ZmtCarve c{base, 0};
    w = Lz4Ws{};
    w.tmp = c.take<uint8_t>(nblocks * ZMT_LZ4_TMP_STRIDE);          // per-block temp slots
    w.blk_csize = c.take<uint32_t>(a256(nblocks * 4));
    w.chk = c.take<uint32_t>(a256(nchunks * 4));                    // content checksum per chunk
    w.frame_size = c.take<uint64_t>(a256((nchunks + 1) * 8));
    if (npos) zl_chain_layout(c, npos, w.ch);
    return c.off + 1024;
}

struct ZstdWs { uint8_t* tmp; uint32_t* blk_csize; uint64_t* frame_size; ZScratch* zsc; ZlChainWs ch; };
static uint64_t zstd_layout(uint8_t* base, uint64_t nchunks, uint64_t nblocks, uint64_t npos, ZstdWs& w)
{
    static_assert(sizeof(ZScratch) % 8 == 0, "scratch stride");
    ZmtCarve c{base, 0};
    w = ZstdWs{};
    w.tmp = c.take<uint8_t>(nblocks * ZMT_LZ4_TMP_STRIDE);
    w.blk_csize = c.take<uint32_t>(a256(nblocks * 4));
    w.frame_size = c.take<uint64_t>(a256((nchunks + 1) * 8));
    w.zsc = c.take<ZScratch>((uint64_t)(ZSTD_MAX_GRID + 8) * a256(sizeof(ZScratch)));    // per-CTA scratch, sized for the largest grid we launch
    if (npos) zl_chain_layout(c, npos, w.ch);
    return c.off + 1024;
}

extern "C" size_t zmt_lz4c_level_workspace_bytes(uint32_t nchunks, uint32_t chunk_size, int level)
{
    if (level < 1 || level > L4H_MAX_LEVEL || chunk_size == 0) return 0;
    const uint64_t npos = level >= L4H_MIN_LEVEL ? (uint64_t)zl_group_chunks(nchunks, chunk_size) * chunk_size : 0;
    if (npos > 0xFFFFFFFFull) return 0;
    Lz4Ws w;
    return (size_t)lz4_layout(nullptr, nchunks, (uint64_t)nchunks * zmt_bpc(chunk_size), npos, w);
}
extern "C" size_t zmt_lz4c_workspace_bytes(uint32_t nchunks, uint32_t chunk_size) { return zmt_lz4c_level_workspace_bytes(nchunks, chunk_size, 1); }

extern "C" size_t zmt_zstdc_level_workspace_bytes(uint32_t nchunks, uint32_t chunk_size, int level)
{
    if (chunk_size == 0) return 0;
    const uint64_t npos = level >= ZL_MIN_LEVEL ? (uint64_t)zl_group_chunks(nchunks, chunk_size) * chunk_size : 0;
    if (npos > 0xFFFFFFFFull) return 0;
    ZstdWs w;
    return (size_t)zstd_layout(nullptr, nchunks, (uint64_t)nchunks * zmt_bpc(chunk_size), npos, w);
}
extern "C" size_t zmt_zstdc_workspace_bytes(uint32_t nchunks, uint32_t chunk_size) { return zmt_zstdc_level_workspace_bytes(nchunks, chunk_size, 3); }

extern "C" uint64_t zmt_lz4c_out_bound(uint32_t nchunks, uint32_t chunk_size)
{
    if (chunk_size == 0) return 0;
    const uint64_t bpc = ((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK;
    return (uint64_t)nchunks * ((uint64_t)chunk_size + 12 + 15 + 8 + 4 * bpc) + 256;
}

extern "C" uint64_t zmt_zstdc_out_bound(uint32_t nchunks, uint32_t chunk_size)
{
    if (chunk_size == 0) return 0;
    const uint64_t bpc = ((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK;
    return (uint64_t)nchunks * ((uint64_t)chunk_size + 12 + 9 + 3 + 32 * bpc) + 256;     // <= 5 blocks x 3-byte headers per 64 KiB window
}

// ---------------------------------------------------------------- chain search (zstd_lazy.cuh), shared by both chain classes
// One group of G chunks at a time: hash every position, radix-sort the (hash, position) pairs, link each position to the
// previous one with its hash (prev[]), walk the chains into best[], then run the class's block kernel over the group's
// blocks through blocks(c0, nblk, best).  DICT: chains continue into the dictionary's index cd.
template <uint32_t BLK, uint32_t START, uint32_t END, bool DICT = false, class Blocks>
static int zl_chain_groups(const ZmtBatch& b, const ZlChainWs& ch, uint32_t min_match, uint32_t depth, uint32_t window, cudaStream_t stream, Blocks blocks,
                           const ZlCDict* cd = nullptr)
{
    for (uint32_t c0 = 0; c0 < b.nchunks; c0 += b.G) {
        const uint32_t ng = b.nchunks - c0 < b.G ? b.nchunks - c0 : b.G;
        uint64_t npos = (uint64_t)ng * b.chunk_size;
        if (!b.chunk_bytes) { const uint64_t s = (uint64_t)c0 * b.chunk_size; npos = b.in_bytes > s ? (b.in_bytes - s < npos ? b.in_bytes - s : npos) : 0; }
        cub::DoubleBuffer<uint32_t> K(ch.arr[0], ch.arr[1]), V(ch.arr[2], ch.arr[3]);
        if (npos) {
            const uint32_t np = (uint32_t)npos, g = (np + 255) / 256;
            { ZmtProfScope ps(ZMT_K_ZL_HASH, stream);
            zstd_lazy_hash_kernel<<<g, 256, 0, stream>>>(b.in, b.in_bytes, b.chunk_size, b.chunk_bytes, c0, np, min_match, K.Current(), V.Current()); }
            zmt_dbg_check(stream, "zstd_lazy_hash_kernel");
            {
                ZmtProfScope ps(ZMT_K_ZL_SORT, stream);
                size_t tb = 0;
                if (cub::DeviceRadixSort::SortPairs(nullptr, tb, K, V, (int)np, 0, ZL_HASHLOG, stream) != cudaSuccess || tb > ch.sort_cap) return ZMT_ST_CUDA;
                if (cub::DeviceRadixSort::SortPairs(ch.sort_tmp, tb, K, V, (int)np, 0, ZL_HASHLOG, stream) != cudaSuccess) return ZMT_ST_CUDA;
                zstd_lazy_prev_kernel<<<g, 256, 0, stream>>>(K.Current(), V.Current(), np, V.Alternate());
            }
            zmt_dbg_check(stream, "zstd_lazy sort + prev");
            { ZmtProfScope ps(ZMT_K_ZL_SEARCH, stream);
            zstd_lazy_search_kernel<BLK, START, END, DICT><<<g, 256, 0, stream>>>(b.in, b.in_bytes, b.chunk_size, b.chunk_bytes, c0, np, min_match, depth,
                                                                                  window, V.Alternate(), K.Alternate(), cd); }
            zmt_dbg_check(stream, "zstd_lazy_search_kernel");
        }
        blocks(c0, ng * b.bpc, K.Alternate());
    }
    return ZMT_ST_OK;
}

// ---------------------------------------------------------------- LZ4 compress, levels 1-12 (levels 10-12: lz4_hc.cuh)
// frame sizes -> frame offsets -> pack; indep: the FLG block-independence bit
static int lz4_frame_tail(const ZmtBatch& b, const Lz4Ws& w, uint8_t* out, uint64_t* frame_off, uint32_t indep, cudaStream_t stream)
{
    { ZmtProfScope ps(ZMT_K_LZ4_SIZES, stream);
    lz4_frame_sizes_kernel<<<(b.nchunks + 255) / 256, 256, 0, stream>>>(w.blk_csize, b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc, b.nchunks, w.frame_size); }
    zmt_dbg_check(stream, "lz4_frame_sizes_kernel");
    { ZmtProfScope ps(ZMT_K_SCAN, stream);
    scan_u64_kernel<<<1, 1024, 0, stream>>>(w.frame_size, frame_off, b.nchunks); }
    zmt_dbg_check(stream, "scan_u64_kernel");
    const uint32_t maxp = (uint32_t)(zmt_sm_count() * 16);
    { ZmtProfScope ps(ZMT_K_LZ4_PACK, stream);
    lz4_frame_pack_kernel<<<b.nblocks < maxp ? b.nblocks : maxp, 256, 0, stream>>>(b.in, b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc, w.tmp, w.blk_csize, w.chk,
                                                                                  frame_off, out, b.nblocks, indep); }
    zmt_dbg_check(stream, "lz4_frame_pack_kernel");
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

extern "C" int zmt_lz4_compress_level_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                             uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    if (level < 1 || level > L4H_MAX_LEVEL) return ZMT_ST_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const bool hc = level >= L4H_MIN_LEVEL;
    ZmtBatch b;
    const int st = zmt_batch(b, d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, hc);
    if (st != ZMT_ST_OK) return st;
    Lz4Ws w;
    lz4_layout((uint8_t*)d_work, nchunks, b.nblocks, b.npos_max, w);

    // The content checksum only reads the input: it runs on a side stream, forked before the first encoder launch and
    // joined before the frame tail.  Levels 1-9 enqueue it BEHIND the compressor's launch: it cannot share an SM with the
    // compressor (two compressor CTAs hold every register of an SM), but there it fills the SMs the compressor's last,
    // ragged wave leaves idle, instead of starting when the last CTA has retired.  Levels 10-12 run it beside the search.
    const ZmtSide side = zmt_side_stream();
    const cudaStream_t xs = side.ok ? side.stream : stream;
    if (side.ok) cudaEventRecord(side.fork, stream);
    if (!hc) {
        // 2 CTAs x 16 warps per SM: throughput scales ~linearly with resident warps (DESIGN.md §3)
        cudaFuncSetAttribute(lz4_blocks_pipe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PipeSmem));
        const uint32_t maxc = (uint32_t)(zmt_sm_count() * 2 * 8);
        { ZmtProfScope ps(ZMT_K_LZ4_COMPRESS, stream);
        lz4_blocks_pipe_kernel<<<b.nblocks < maxc ? b.nblocks : maxc, 2 * P_TEAM, sizeof(PipeSmem), stream>>>(b.in, b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc,
                                                                                                             w.tmp, w.blk_csize, b.nblocks); }
        zmt_dbg_check(stream, "lz4 block compressor");
    }
    if (side.ok) cudaStreamWaitEvent(side.stream, side.fork, 0);
    { ZmtProfScope ps(ZMT_K_XXH32, xs);
    xxh32_kernel<<<(nchunks + X_WARPS - 1) / X_WARPS, 32 * X_WARPS, 0, xs>>>(b.in, nullptr, nullptr, b.chunk_bytes, chunk_size, in_bytes, w.chk, nchunks); }
    if (side.ok) cudaEventRecord(side.join, side.stream);
    zmt_dbg_check(xs, "xxh32_kernel");
    if (hc) {
        const L4hParams P = l4h_params(level);
        cudaFuncSetAttribute(lz4_hc_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(L4hSmem));
        const int cs = zl_chain_groups<L4H_BLOCK, L4H_MFLIMIT, L4H_LASTLIT>(b, w.ch, L4H_MINMATCH, P.depth, L4H_WINDOW, stream,
            [&](uint32_t c0, uint32_t nblk, const uint32_t* best) {
                { ZmtProfScope ps(ZMT_K_L4H_BLOCKS, stream);
                lz4_hc_blocks_kernel<<<zstd_grid(nblk), 256, sizeof(L4hSmem), stream>>>(b.in, b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc, c0, nblk, P.lazy,
                                                                                         best, w.tmp, w.blk_csize); }
                zmt_dbg_check(stream, "lz4_hc_blocks_kernel");
            });
        if (cs != ZMT_ST_OK) return cs;
    }
    if (side.ok) cudaStreamWaitEvent(stream, side.join, 0);
    return lz4_frame_tail(b, w, (uint8_t*)d_out, d_frame_off, hc ? 0u : 0x20u, stream);
}

extern "C" int zmt_lz4_compress_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                       uint32_t nchunks, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    return zmt_lz4_compress_level_device(d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, 1, d_work, d_out, d_frame_off, stream_);
}

// ---------------------------------------------------------------- zstd compress, levels 1-22 (levels 6-22: zstd_lazy.cuh)
// frame sizes -> frame offsets -> pack; DICT: the frames name the Dictionary_ID of cd
template <bool DICT>
static int zstd_frame_tail(const ZmtBatch& b, const ZstdWs& w, uint8_t* out, uint64_t* frame_off, cudaStream_t stream, const ZlCDict* cd)
{
    zstd_frame_sizes_kernel<DICT><<<(b.nchunks + 255) / 256, 256, 0, stream>>>(w.blk_csize, b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc, b.nchunks,
                                                                               w.frame_size, cd);
    zmt_dbg_check(stream, "zstd_frame_sizes_kernel");
    scan_u64_kernel<<<1, 1024, 0, stream>>>(w.frame_size, frame_off, b.nchunks);
    zmt_dbg_check(stream, "scan_u64_kernel");
    const uint32_t maxp = (uint32_t)(zmt_sm_count() * 16);
    { ZmtProfScope ps(ZMT_K_ZSTD_PACK, stream);
    zstd_frame_pack_kernel<DICT><<<b.nblocks < maxp ? b.nblocks : maxp, 256, 0, stream>>>(b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc, w.tmp, w.blk_csize,
                                                                                         frame_off, out, b.nblocks, cd); }
    zmt_dbg_check(stream, "zstd_frame_pack_kernel");
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

// DICT: levels 6-22 only, their chains continuing into the dictionary's index cd
template <bool DICT>
static int zstd_compress(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes, uint32_t nchunks, int level,
                         void* d_work, void* d_out, uint64_t* d_frame_off, cudaStream_t stream, const ZlCDict* cd)
{
    const bool chain = level >= ZL_MIN_LEVEL;
    ZmtBatch b;
    int st = zmt_batch(b, d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, chain);
    if (st == ZMT_ST_OK) st = zstd_tables_init();
    if (st != ZMT_ST_OK) return st;
    ZstdWs w;
    zstd_layout((uint8_t*)d_work, nchunks, b.nblocks, b.npos_max, w);
    if (!chain) {
        cudaFuncSetAttribute(zstd_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ZstdSmem));
        { ZmtProfScope ps(ZMT_K_ZSTD_COMPRESS, stream);
        zstd_blocks_kernel<<<zstd_grid(b.nblocks), P_TEAM, sizeof(ZstdSmem), stream>>>(b.in, b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc, w.tmp, w.blk_csize,
                                                                                       b.nblocks, w.zsc); }
        zmt_dbg_check(stream, "zstd_blocks_kernel");
    } else {
        const ZlParams P = zl_params(level);
        cudaFuncSetAttribute(zstd_lazy_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ZlSmem));
        st = zl_chain_groups<ZL_BLOCK, 0, 0, DICT>(b, w.ch, P.min_match, P.depth, zl_window(level), stream,
            [&](uint32_t c0, uint32_t nwin, const uint32_t* best) {
                { ZmtProfScope ps(ZMT_K_ZL_BLOCKS, stream);
                zstd_lazy_blocks_kernel<<<zstd_grid(nwin), 256, sizeof(ZlSmem), stream>>>(b.in, b.in_bytes, b.chunk_size, b.chunk_bytes, b.bpc, c0, nwin, P.lazy,
                                                                                           best, w.tmp, w.blk_csize, w.zsc); }
                zmt_dbg_check(stream, "zstd_lazy_blocks_kernel");
            }, cd);
        if (st != ZMT_ST_OK) return st;
    }
    return zstd_frame_tail<DICT>(b, w, (uint8_t*)d_out, d_frame_off, stream, cd);
}

extern "C" int zmt_zstd_compress_level_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                              uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    return zstd_compress<false>(d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, level, d_work, d_out, d_frame_off, (cudaStream_t)stream_, nullptr);
}

extern "C" int zmt_zstd_compress_dict_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                             uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_,
                                             const void* d_cdict)
{
    if (level < ZL_MIN_LEVEL) return ZMT_ST_BAD_ARG;        // the level-3 class has no chains to continue
    const ZlCDict* cd = (const ZlCDict*)d_cdict;
    return cd ? zstd_compress<true>(d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, level, d_work, d_out, d_frame_off, (cudaStream_t)stream_, cd)
              : zstd_compress<false>(d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, level, d_work, d_out, d_frame_off, (cudaStream_t)stream_, nullptr);
}

// ---- a dictionary's compression index (ZlCDict, zstd_lazy.cuh): the header, head[], prev[] and the sort's pairs and
// scratch over dict_bytes positions
#define ZL_CDICT_KEY_BITS (ZL_HASHLOG + 1)          // the hashes and the key of unlinked positions
struct ZlCDictWs { ZlCDict* hdr; uint32_t* head; uint32_t* prev; uint32_t* arr[4]; void* sort_tmp; size_t sort_cap; };
static uint64_t zl_cdict_layout(uint8_t* base, uint32_t n, ZlCDictWs& w)
{
    ZmtCarve c{base, 0};
    w.hdr = c.take<ZlCDict>(a256(sizeof(ZlCDict)));
    w.head = c.take<uint32_t>(4ull << ZL_HASHLOG);
    w.prev = c.take<uint32_t>(a256(4ull * n));
    for (int k = 0; k < 4; k++) w.arr[k] = c.take<uint32_t>(a256(4ull * n));
    w.sort_cap = n ? zl_sort_temp_bytes(n, ZL_CDICT_KEY_BITS) : 0;
    w.sort_tmp = c.take<void>(a256(w.sort_cap));
    return c.off;
}

extern "C" size_t zmt_zstd_cdict_bytes(uint64_t dict_bytes)
{
    if (dict_bytes >= (1ull << 31)) return 0;
    ZlCDictWs w;
    return (size_t)zl_cdict_layout(nullptr, (uint32_t)dict_bytes, w);
}

extern "C" int zmt_zstd_cdict_build_device(const void* d_ddict, uint64_t dict_bytes, void* d_cdict, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!d_ddict || !d_cdict || dict_bytes >= (1ull << 31)) return ZMT_ST_BAD_ARG;
    const uint32_t n = (uint32_t)dict_bytes, mm = zl_params(ZL_MIN_LEVEL).min_match, g = (n + 255) / 256;
    const ZDDict* dd = (const ZDDict*)d_ddict;
    ZlCDictWs w;
    zl_cdict_layout((uint8_t*)d_cdict, n, w);
    if (cudaMemsetAsync(w.head, 0xFF, 4ull << ZL_HASHLOG, stream) != cudaSuccess) return ZMT_ST_CUDA;
    if (n) {
        cub::DoubleBuffer<uint32_t> K(w.arr[0], w.arr[1]), V(w.arr[2], w.arr[3]);
        { ZmtProfScope ps(ZMT_K_ZL_HASH, stream);
        zl_cdict_hash_kernel<<<g, 256, 0, stream>>>(dd, n, mm, K.Current(), V.Current()); }
        ZmtProfScope ps(ZMT_K_ZL_SORT, stream);
        size_t tb = 0;
        if (cub::DeviceRadixSort::SortPairs(nullptr, tb, K, V, (int)n, 0, ZL_CDICT_KEY_BITS, stream) != cudaSuccess || tb > w.sort_cap) return ZMT_ST_CUDA;
        if (cub::DeviceRadixSort::SortPairs(w.sort_tmp, tb, K, V, (int)n, 0, ZL_CDICT_KEY_BITS, stream) != cudaSuccess) return ZMT_ST_CUDA;
        zl_cdict_link_kernel<<<g, 256, 0, stream>>>(K.Current(), V.Current(), n, w.head, w.prev);
    }
    zl_cdict_header_kernel<<<1, 1, 0, stream>>>(dd, mm, w.head, w.prev, w.hdr);
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

extern "C" int zmt_zstd_compress_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                        uint32_t nchunks, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    return zmt_zstd_compress_level_device(d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, 3, d_work, d_out, d_frame_off, stream_);
}

// The decoder's workspace (ZmtCarve, launch.h).  zeroed: the bytes from stored[] through any_bchk, cleared before the kernels run.
struct Lz4dWs {
    uint32_t* stored; uint32_t* computed; uint32_t* needs_seq; unsigned long long* ticket; uint32_t* any_bchk; uint64_t zeroed;
    unsigned long long* wbase; uint64_t* slot_cnt; uint64_t* first_slot; LzBlk* tab; uint32_t* prog; unsigned long long* rec;
};
static uint64_t lz4d_layout(uint8_t* base, uint32_t nframes, uint32_t nslots, uint64_t in_bytes, Lz4dWs& w)
{
    ZmtCarve c{base, 0};
    w.stored = c.take<uint32_t>(a256((uint64_t)nframes * 4));
    w.computed = c.take<uint32_t>(a256((uint64_t)nframes * 4));
    w.needs_seq = c.take<uint32_t>(a256((uint64_t)nframes * 4));
    w.ticket = c.take<unsigned long long>(8);
    w.any_bchk = c.take<uint32_t>(248);                                 // any frame with FLG.BC set
    w.zeroed = c.off;
    w.wbase = c.take<unsigned long long>(ticket_table_bytes(nframes));
    w.slot_cnt = c.take<uint64_t>(a256(((uint64_t)nframes + 1) * 8));
    w.first_slot = c.take<uint64_t>(a256(((uint64_t)nframes + 1) * 8));
    w.tab = c.take<LzBlk>(a256((uint64_t)nslots * sizeof(LzBlk)));
    w.prog = c.take<uint32_t>(a256((uint64_t)nslots * 4));
    w.rec = c.take<unsigned long long>(a256((in_bytes / 3 + 8) * 8));   // a match record per 3 input bytes at most: a token and an offset take 3
    return c.off + 1024;
}

extern "C" size_t zmt_lz4d_workspace_bytes(uint32_t nframes, uint32_t nslots, uint64_t in_bytes) { Lz4dWs w; return (size_t)lz4d_layout(nullptr, nframes, nslots, in_bytes, w); }

// seg = nullptr: whole frames (zmt_lz4_decompress_device); else every frame of the batch is a segment
static int lz4_decompress_launch(const void* d_in, uint64_t in_bytes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, uint32_t nframes,
                                 uint32_t nslots, void* d_out, const uint64_t* d_out_off, uint64_t* d_out_size,
                                 uint32_t* d_status, zmt_lz4_segment* seg, void* d_work, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    if (nframes == 0) return ZMT_ST_OK;
    if (nslots < nframes) return ZMT_ST_BAD_ARG;
    Lz4dWs w;
    lz4d_layout((uint8_t*)d_work, nframes, nslots, in_bytes, w);
    cudaMemsetAsync(d_status, 0, (size_t)nframes * 4, stream);
    cudaMemsetAsync(d_out_size, 0, (size_t)nframes * 8, stream);
    cudaMemsetAsync(w.stored, 0, w.zeroed, stream);
    const uint8_t* in = (const uint8_t*)d_in;
    lz4_slot_counts_kernel<<<(nframes + 255) / 256, 256, 0, stream>>>(d_out_off, nframes, w.slot_cnt);
    scan_u64_kernel<<<1, 1024, 0, stream>>>(w.slot_cnt, w.first_slot, nframes);
    ticket_windows_kernel<<<1, 256, 0, stream>>>(w.first_slot, nframes, w.wbase);
    lz4_scan_frames_kernel<<<(nframes + 127) / 128, 128, 0, stream>>>(in, d_frame_off, d_frame_csize, d_out_off, w.first_slot, nslots, w.tab, w.prog, d_status,
                                                                      w.stored, w.needs_seq, w.any_bchk, seg, nframes);
    zmt_dbg_check(stream, "lz4_scan_frames_kernel");
    {
        const uint32_t maxg = (uint32_t)(zmt_sm_count() * 8), need = (nslots + X_WARPS - 1) / X_WARPS;
        lz4_block_checksum_kernel<<<need < maxg ? need : maxg, 32 * X_WARPS, 0, stream>>>(in, d_frame_off, w.first_slot, w.tab, d_status, w.any_bchk, nframes, nslots);
    }
    zmt_dbg_check(stream, "lz4_block_checksum_kernel");
    { ZmtProfScope ps(ZMT_K_LZ4_DECODE, stream);
    lz4_parse_blocks_kernel<<<(nslots + LZD_WARPS - 1) / LZD_WARPS, 32 * LZD_WARPS, 0, stream>>>(
        in, in + in_bytes, d_frame_off, (uint8_t*)d_out, d_out_off, w.first_slot, w.tab, w.rec, (unsigned long long*)d_out_size, d_status, w.needs_seq, seg, nframes,
        nslots); }
    zmt_dbg_check(stream, "lz4_parse_blocks_kernel");
    {
        const uint32_t maxg = (uint32_t)(zmt_sm_count() * 8);
        const uint32_t need = (nslots + LZD_WARPS - 1) / LZD_WARPS;
        ZmtProfScope ps(ZMT_K_LZ4_DEXEC, stream);
        // the shared-memory step window turns a chain of matches feeding each other into SMEM round trips instead of L2 ones
        // (DESIGN.md §3.2)
        lz4_exec_blocks_kernel<<<need < maxg ? need : maxg, 32 * LZD_WARPS, 0, stream>>>(
            (uint8_t*)d_out, d_out_off, d_frame_off, w.first_slot, w.tab, w.rec, w.prog, d_status, w.needs_seq, w.ticket, w.wbase, nframes, nslots);
    }
    zmt_dbg_check(stream, "lz4_exec_blocks_kernel");
    lz4_decode_frames_seq_kernel<<<(nframes + LZD_WARPS - 1) / LZD_WARPS, 32 * LZD_WARPS, 0, stream>>>(
        in, in + in_bytes, d_frame_off, d_frame_csize, (uint8_t*)d_out, d_out_off, (unsigned long long*)d_out_size, d_status, w.needs_seq, seg, nframes);
    zmt_dbg_check(stream, "lz4_decode_frames_seq_kernel");
    { ZmtProfScope ps(ZMT_K_XXH32_DEC, stream);
    if (seg) lz4_segment_xxh32_kernel<<<(nframes + X_WARPS - 1) / X_WARPS, 32 * X_WARPS, 0, stream>>>((const uint8_t*)d_out, d_out_off,
                                                                                                     (const unsigned long long*)d_out_size, d_status, seg, w.computed, nframes);
    else xxh32_kernel<<<(nframes + X_WARPS - 1) / X_WARPS, 32 * X_WARPS, 0, stream>>>((const uint8_t*)d_out, d_out_off, d_out_size, nullptr, 0, 0, w.computed, nframes); }
    lz4_verify_kernel<<<(nframes + 255) / 256, 256, 0, stream>>>(in, d_frame_off, d_frame_csize, d_status,
                                                                (const unsigned long long*)d_out_size, w.stored, w.computed, seg, nframes);
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

extern "C" int zmt_lz4_decompress_device(const void* d_in, uint64_t in_bytes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, uint32_t nframes,
                                         uint32_t nslots, void* d_out, const uint64_t* d_out_off, uint64_t* d_out_size,
                                         uint32_t* d_status, void* d_work, void* stream)
{
    return lz4_decompress_launch(d_in, in_bytes, d_frame_off, d_frame_csize, nframes, nslots, d_out, d_out_off, d_out_size, d_status, nullptr, d_work, stream);
}

extern "C" int zmt_lz4_decompress_segments_device(const void* d_in, uint64_t in_bytes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                                                  uint32_t nframes, uint32_t nslots, void* d_out, const uint64_t* d_out_off, uint64_t* d_out_size,
                                                  uint32_t* d_status, zmt_lz4_segment* d_seg, void* d_work, void* stream)
{
    if (!d_seg && nframes) return ZMT_ST_BAD_ARG;
    return lz4_decompress_launch(d_in, in_bytes, d_frame_off, d_frame_csize, nframes, nslots, d_out, d_out_off, d_out_size, d_status, d_seg, d_work, stream);
}

extern "C" int zmt_lz4f_segment_host(const uint8_t* seg, size_t n, size_t start, uint32_t flg, uint32_t bd, size_t max_in, uint64_t max_out,
                                     size_t* end, uint64_t* room, uint32_t* last)
{
    Lz4fWalk w; w.pos = start; w.bound = 0; w.nblk = 0; w.done = 0;
    const size_t stop = max_in > start ? max_in : start + 1;                  // at least one block (or the end mark)
    if (!lz4f_walk_blocks(seg, n, flg, bd, &w, stop, max_out > 0 ? max_out : 1) || w.pos > n) return ZMT_ST_TRUNCATED;
    *end = w.pos; *room = w.bound; *last = w.done;
    return ZMT_ST_OK;
}
