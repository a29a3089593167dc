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
    uint32_t V[C_TILE / 32];              // visited-by-own-chain bits
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
    uint8_t  len[C_TILE];                 // piece length per selected piece start (written by the marking walk)
    uint16_t piece[C_MAXPIECE];           // tile-relative start of the r-th selected piece
    union {                               // segprev is read by head detection, before the heads are written
        uint16_t hidx[C_TILE / 4];        // heads: one per sequence, sequences hold a match of >= 4 bytes
        uint16_t segprev[C_CHAINS];       // per segment: 1 + start of the last non-Cont piece before it (0: none)
    };
    uint32_t longl[2 * (C_TILE / (C_LONGLIT + 1) + 2)];   // jobs: literal runs > C_LONGLIT (start | length << 16, output offset) -- at most
                                                           // 4096/37 + 1 pending per tile -- and 255-runs of match lengths >= 1290 (count, offset | 1<<31)
};

// number of bytes (<= cap) for which s[p + i] == s[p + i - d].  Word compares only: the last, partial word gets a
// sentinel bit at byte `cap` (reads run at most 3 bytes past p + cap: LzStage::in carries 32 pad bytes).
__device__ __forceinline__ uint32_t c_extend(const uint8_t* s, uint32_t p, uint32_t d, uint32_t cap)
{
    uint32_t L = 0;
    for (;;) {
        uint32_t x = lds32u(s, p + L) ^ lds32u(s, p + L - d);
        const uint32_t rem = cap - L;
        if (rem < 4) x |= 1u << (8 * rem);
        if (x) return L + ((__ffs(x) - 1) >> 3);
        L += 4;
    }
}

// Walk one speculative chain through the tile.  The greedy parse is evaluated piecewise: a match is cut at
// the first segment boundary that leaves it >= 4 bytes, and continues ("inside", din = its offset) into the
// next segment, so no lane ever compares more than 19 bytes per step.  Pieces are merged again at emission.
//   MODE 0: own segment only (sets V, exit state -> X.xfree/X.xdin)                      X: LzFront
//   MODE 1: continuation until it merges into another chain or leaves the tile (-> X.link/X.mpos)
//   MODE 2: re-walk of a chain that is on the true path: marks X.Sel/X.Cont and the piece lengths X.len
//           (same steps as MODE 0 + 1)                                                    X: LzBack
template <int MODE, class OUT>
__device__ __forceinline__ void c_walk(const uint8_t* in, PipeTile& T, OUT& X, uint32_t k, uint32_t p, uint32_t din, uint32_t t0, uint32_t limit)
{
    const uint32_t t1 = t0 + C_TILE;
    uint32_t lk = 0xFFFFFFFFu, mp = 0;
    bool done = false;
    while (!done) {                                  // single exit: the warp reconverges before the next barrier
        if (p >= t1) { lk = C_END; mp = p; done = true; continue; }
        const uint32_t rel = p - t0, j = rel / C_SEG;
        if (MODE == 0 && j != k) { mp = p; done = true; continue; }
        if (din) {
            // inside a match with offset din that covered everything up to the boundary p
            if (MODE != 0 && j != k && ((T.M[rel >> 5] >> (rel & 31)) & 1) && T.off[rel] == din) {
                lk = j; mp = p; done = true; continue;          // chain j's own first step is this very match
            }
            uint32_t cap = p < limit ? limit - p : 0; if (cap > C_SEG) cap = C_SEG;
            const uint32_t E = c_extend(in, p, din, cap);
            if constexpr (MODE == 2) {
                if (E) { atomicOr(&X.Sel[rel >> 5], 1u << (rel & 31)); atomicOr(&X.Cont[rel >> 5], 1u << (rel & 31)); X.len[rel] = (uint8_t)E; }
            }
            p += E;
            if (E != C_SEG) din = 0;
            continue;
        }
        if (MODE != 0 && j != k && (rel & (C_SEG - 1)) == 0) { lk = j; mp = p; done = true; continue; }
        uint32_t bits = (T.M[rel >> 5] >> (rel & 16)) & 0xFFFFu;     // this segment's 16 candidate bits
        bits &= 0xFFFFu << (rel & 15);
        if (!bits) {                                                   // segment exhausted: free at its end
            const uint32_t nx = t0 + (j + 1) * C_SEG;
            if (MODE == 0) { mp = nx; done = true; }
            else if (j + 1 == C_CHAINS) { lk = C_END; mp = t1; done = true; }
            else if (j != k) { lk = j + 1; mp = nx; done = true; }
            else p = nx;
            continue;
        }
        const uint32_t qr = (rel & ~15u) + (__ffs(bits) - 1), q = t0 + qr;
        if (MODE != 0 && j != k && ((T.V[qr >> 5] >> (qr & 31)) & 1)) { lk = j; mp = q; done = true; continue; }
        const uint32_t d = T.off[qr];
        uint32_t B = (q & ~(C_SEG - 1)) + C_SEG;                     // cut at the first boundary leaving >= 4 bytes
        if (B - q < 4) B += C_SEG;
        const uint32_t end = B < limit ? B : limit;
        const uint32_t L = 4 + c_extend(in, q + 4, d, end - (q + 4));  // first 4 bytes are known equal; q + 4 <= limit always
        if constexpr (MODE == 2) { atomicOr(&X.Sel[qr >> 5], 1u << (qr & 31)); X.len[qr] = (uint8_t)L; }
        if constexpr (MODE == 0) atomicOr(&T.V[qr >> 5], 1u << (qr & 31));
        p = q + L;
        if (p == B) din = d;                                          // reached the boundary: still inside the match
    }
    if constexpr (MODE == 0) { X.xfree[k] = mp; X.xdin[k] = (uint16_t)din; }
    if constexpr (MODE == 1) { X.link[k] = (uint16_t)lk; X.mpos[k] = mp; if (lk == C_END) X.xdin[k] = (uint16_t)din; }
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
                   uint32_t bpc, uint8_t* __restrict__ tmp, uint32_t* __restrict__ blk_csize, uint32_t nblocks, uint32_t flags,
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
        lz_stage<NT>(S.stage, S.tab, &S.mbar, in + cbase + boff, n, flags, tid);

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
// XXH32 (seed 0) of p[0, n) by one warp; tile = the warp's 1 KiB of shared memory.  The hash is valid on lane 0.
__device__ __forceinline__ uint32_t warp_xxh32(const uint8_t* p, uint64_t n, uint4 (*tile)[32], uint32_t lane)
{
    const uint32_t j = lane & 3;
    uint32_t acc = j == 0 ? XXP1 + XXP2 : j == 1 ? XXP2 : j == 2 ? 0u : 0u - XXP1;
    const uint64_t ns = n >> 4;                              // 16-byte stripes
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

__global__ void zstd_frame_sizes_kernel(const uint32_t* __restrict__ blk_csize, uint64_t in_bytes, uint32_t chunk_size,
                                        const uint32_t* __restrict__ chunk_bytes, uint32_t bpc, uint32_t nchunks, uint64_t* __restrict__ frame_size)
{
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const uint64_t cbytes = zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size);
    uint64_t sz = 12 + 4 + 1 + zstd_fcs_bytes(cbytes);
    if (cbytes == 0) sz += 3;
    for (uint32_t b = 0; b < bpc; b++) sz += blk_csize[c * bpc + b];
    frame_size[c] = sz;
}

__global__ void __launch_bounds__(256)
zstd_frame_pack_kernel(uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes, uint32_t bpc,
                       const uint8_t* __restrict__ tmp, const uint32_t* __restrict__ blk_csize, const uint64_t* __restrict__ frame_off,
                       uint8_t* __restrict__ out, uint32_t nblocks)
{
    for (uint32_t blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const uint32_t c = blk / bpc, b = blk % bpc;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, c, in_bytes, chunk_size);
        const uint32_t fl = zstd_fcs_bytes(cbytes), hdr = 12 + 4 + 1 + fl;
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
            if (fl == 1) f[17] = (uint8_t)cbytes;
            else if (fl == 2) { const uint32_t v = (uint32_t)cbytes - 256; f[17] = (uint8_t)v; f[18] = (uint8_t)(v >> 8); }
            else stg_le32(f + 17, (uint32_t)cbytes);
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
    static const int16_t LLn[36] = { 4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1 };
    static const int16_t MLn[53] = { 1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1 };
    static const int16_t OFn[29] = { 1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1 };
    static const uint32_t LLb[36] = { 0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,18,20,22,24,28,32,40,48,64,128,256,512,1024,2048,4096,8192,16384,32768,65536 };
    static const uint8_t  LLx[36] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16 };
    static const uint32_t MLb[53] = { 3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,35,37,39,41,43,47,51,59,67,83,99,131,259,515,1027,2051,4099,8195,16387,32771,65539 };
    static const uint8_t  MLx[53] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16 };
    ZFseCTable t;
    zstd_build_ctable(t, LLn, 36, 6); if (cudaMemcpyToSymbol(c_fse_ll, &t, sizeof(t)) != cudaSuccess) return ZMT_ST_CUDA;
    zstd_build_ctable(t, OFn, 29, 5); if (cudaMemcpyToSymbol(c_fse_of, &t, sizeof(t)) != cudaSuccess) return ZMT_ST_CUDA;
    zstd_build_ctable(t, MLn, 53, 6); if (cudaMemcpyToSymbol(c_fse_ml, &t, sizeof(t)) != cudaSuccess) return ZMT_ST_CUDA;
    uint8_t llc[64], mlc[128];
    for (int v = 0; v < 64; v++) { int c = 0; while (c + 1 < 36 && LLb[c + 1] <= (uint32_t)v) c++; llc[v] = (uint8_t)c; }
    for (int v = 0; v < 128; v++) { int c = 0; while (c + 1 < 53 && MLb[c + 1] <= (uint32_t)v + 3) c++; mlc[v] = (uint8_t)c; }
    cudaMemcpyToSymbol(c_ll_code, llc, sizeof(llc)); cudaMemcpyToSymbol(c_ml_code, mlc, sizeof(mlc));
    cudaMemcpyToSymbol(c_ll_base, LLb, sizeof(LLb)); cudaMemcpyToSymbol(c_ml_base, MLb, sizeof(MLb));
    cudaMemcpyToSymbol(c_ll_bits, LLx, sizeof(LLx)); cudaMemcpyToSymbol(c_ml_bits, MLx, sizeof(MLx));
    if (cudaGetLastError() != cudaSuccess) return ZMT_ST_CUDA;
    if (cudaDeviceSynchronize() != cudaSuccess) return ZMT_ST_CUDA;    // the kernels run on non-blocking streams: nothing else orders the table copies before them
    done[dev] = true;
    return ZMT_ST_OK;
}

// ============================================================================ host launchers
// ZSTDMT_B200_DEBUG_SYNC=1: synchronise after every kernel and name the one that failed (debug only)
// ---- optional per-kernel timing (zmt_prof_begin / zmt_prof_end): CUDA events recorded on the launching
// stream around every kernel while enabled; used by bench.py for the roofline of the dominant kernel.
struct ZmtProfRec { int id; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::vector<ZmtProfRec> g_prof;
struct ZmtProfScope {
    cudaStream_t st; cudaEvent_t a = nullptr, b = nullptr; int id;
    ZmtProfScope(int id_, cudaStream_t s) : st(s), id(id_) { if (g_prof_on) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, st); } }
    ~ZmtProfScope() { if (a) { cudaEventRecord(b, st); g_prof.push_back({id, a, b}); } }
};
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

// begin / end marks for code outside this file (zstd_decode.cu): same records as ZmtProfScope
static cudaEvent_t g_mark_a[ZMT_K_COUNT];
extern "C" void zmt_prof_mark(int id, void* stream, int end)
{
    if (!g_prof_on || id < 0 || id >= ZMT_K_COUNT) return;
    cudaStream_t st = (cudaStream_t)stream;
    if (!end) { cudaEventCreate(&g_mark_a[id]); cudaEventRecord(g_mark_a[id], st); }
    else { cudaEvent_t b; cudaEventCreate(&b); cudaEventRecord(b, st); g_prof.push_back({id, g_mark_a[id], b}); }
}

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

static std::mutex g_dev_mu;                     // guards the per-device lazy state below (contexts may run on several host threads)
static inline int zmt_sm_count()
{
    static int n[64];
    int dev = 0; cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return 132;
    std::lock_guard<std::mutex> g(g_dev_mu);
    if (!n[dev]) { cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev); if (n[dev] <= 0) n[dev] = 132; }
    return n[dev];
}

// side stream + fork / join events, one set per (device, host thread): a set must not be shared by two launch sequences
// that interleave, and every host thread enqueues its own sequences in order
struct ZmtSide { cudaStream_t stream = nullptr; cudaEvent_t fork = nullptr, join = nullptr; bool ok = false; };
static ZmtSide zmt_side_stream()
{
    static const bool off = getenv("ZSTDMT_B200_NO_SIDE_STREAM") != nullptr;
    thread_local ZmtSide side[64];
    int dev = 0;
    if (off || cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return ZmtSide();
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

extern "C" size_t zmt_lz4c_workspace_bytes(uint32_t nchunks, uint32_t chunk_size)
{
    if (chunk_size == 0) return 0;
    const uint64_t bpc = ((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK;
    const uint64_t nblocks = (uint64_t)nchunks * bpc;
    uint64_t sz = 0;
    sz += nblocks * ZMT_LZ4_TMP_STRIDE;                  // per-block temp slots
    sz += ((nblocks * 4 + 255) & ~255ull);               // blk_csize
    sz += (((uint64_t)nchunks * 4 + 255) & ~255ull);     // chk
    sz += ((((uint64_t)nchunks + 1) * 8 + 255) & ~255ull); // frame_size
    return (size_t)sz + 1024;
}

extern "C" uint64_t zmt_lz4c_out_bound(uint32_t nchunks, uint32_t chunk_size)
{
    if (chunk_size == 0) return 0;
    const uint64_t bpc = ((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK;
    return (uint64_t)nchunks * ((uint64_t)chunk_size + 12 + 15 + 8 + 4 * bpc) + 256;
}

extern "C" int zmt_lz4_compress_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                       uint32_t nchunks, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    if (chunk_size == 0 || nchunks == 0) return ZMT_ST_BAD_ARG;
    if (!d_chunk_bytes && nchunks != zmt_chunk_count(in_bytes, chunk_size)) return ZMT_ST_BAD_ARG;
    const uint32_t bpc = (uint32_t)(((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK);
    if ((uint64_t)nchunks * bpc > 0x7FFFFFFFull) return ZMT_ST_BAD_ARG;
    const uint32_t nblocks = nchunks * bpc;
    uint8_t* w = (uint8_t*)d_work;
    uint8_t* tmp = w; w += (uint64_t)nblocks * ZMT_LZ4_TMP_STRIDE;
    uint32_t* blk_csize = (uint32_t*)w; w += (((uint64_t)nblocks * 4 + 255) & ~255ull);
    uint32_t* chk = (uint32_t*)w; w += (((uint64_t)nchunks * 4 + 255) & ~255ull);
    uint64_t* frame_size = (uint64_t*)w;

    // 2 CTAs x 16 warps per SM: throughput scales ~linearly with resident warps (DESIGN.md §3)
    cudaFuncSetAttribute(lz4_blocks_pipe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PipeSmem));
    const uint32_t maxc = (uint32_t)(zmt_sm_count() * 2 * 8);
    uint32_t gridc = nblocks < maxc ? nblocks : maxc;
    static bool occ_shown = false;
    if (!occ_shown && getenv("ZSTDMT_B200_SHOW_OCC")) {
        int nb = 0; occ_shown = true;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, lz4_blocks_pipe_kernel, 2 * P_TEAM, sizeof(PipeSmem));
        fprintf(stderr, "[zstdmt_b200] lz4_blocks_pipe_kernel: %d CTAs/SM, %zu B smem\n", nb, sizeof(PipeSmem));
    }
    const ZmtSide side = zmt_side_stream();
    if (side.ok) cudaEventRecord(side.fork, stream);
    { ZmtProfScope ps(ZMT_K_LZ4_COMPRESS, stream);
    lz4_blocks_pipe_kernel<<<gridc, 2 * P_TEAM, sizeof(PipeSmem), stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, nblocks, getenv("ZSTDMT_B200_NO_TMA") ? 1u : 0u); }
    zmt_dbg_check(stream, "lz4 block compressor");
    // The content checksum only reads the input.  It cannot share an SM with the compressor (two compressor CTAs hold every
    // register of an SM), but enqueued on a side stream BEHIND the compressor's launch it fills the SMs the compressor's last,
    // ragged wave leaves idle, instead of starting when the last CTA has retired; the pack kernel joins both.
    if (side.ok) {
        cudaStreamWaitEvent(side.stream, side.fork, 0);          // fork = everything before the compressor launch (the input is ready)
        { ZmtProfScope ps(ZMT_K_XXH32, side.stream);
        xxh32_kernel<<<(nchunks + X_WARPS - 1) / X_WARPS, 32 * X_WARPS, 0, side.stream>>>((const uint8_t*)d_in, nullptr, nullptr, d_chunk_bytes, chunk_size, in_bytes, chk, nchunks); }
        cudaEventRecord(side.join, side.stream);
        cudaStreamWaitEvent(stream, side.join, 0);
    } else {
        ZmtProfScope ps(ZMT_K_XXH32, stream);
        xxh32_kernel<<<(nchunks + X_WARPS - 1) / X_WARPS, 32 * X_WARPS, 0, stream>>>((const uint8_t*)d_in, nullptr, nullptr, d_chunk_bytes, chunk_size, in_bytes, chk, nchunks);
    }
    zmt_dbg_check(stream, "xxh32_kernel");
    { ZmtProfScope ps(ZMT_K_LZ4_SIZES, stream);
    lz4_frame_sizes_kernel<<<(nchunks + 255) / 256, 256, 0, stream>>>(blk_csize, in_bytes, chunk_size, d_chunk_bytes, bpc, nchunks, frame_size); }
    zmt_dbg_check(stream, "lz4_frame_sizes_kernel");
    { ZmtProfScope ps(ZMT_K_SCAN, stream);
    scan_u64_kernel<<<1, 1024, 0, stream>>>(frame_size, d_frame_off, nchunks); }
    zmt_dbg_check(stream, "scan_u64_kernel");
    const uint32_t maxp = (uint32_t)(zmt_sm_count() * 16);
    const uint32_t gridp = nblocks < maxp ? nblocks : maxp;
    { ZmtProfScope ps(ZMT_K_LZ4_PACK, stream);
    lz4_frame_pack_kernel<<<gridp, 256, 0, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, chk, d_frame_off, (uint8_t*)d_out, nblocks, 0x20u); }
    zmt_dbg_check(stream, "lz4_frame_pack_kernel");
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

// ---------------------------------------------------------------- zstd compress
#define ZSTD_MAX_GRID (132u * 2u * 4u)       // the workspace holds one ZScratch per CTA of the largest grid (H100 SXM: 132 SMs)
static inline uint32_t zstd_grid(uint32_t nblocks) { uint32_t m = (uint32_t)(zmt_sm_count() * 2 * 4); if (m > ZSTD_MAX_GRID) m = ZSTD_MAX_GRID; return nblocks < m ? nblocks : m; }

extern "C" size_t zmt_zstdc_workspace_bytes(uint32_t nchunks, uint32_t chunk_size)
{
    if (chunk_size == 0) return 0;
    const uint64_t bpc = ((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK;
    const uint64_t nblocks = (uint64_t)nchunks * bpc;
    uint64_t sz = nblocks * ZMT_LZ4_TMP_STRIDE;
    sz += ((nblocks * 4 + 255) & ~255ull);
    sz += ((((uint64_t)nchunks + 1) * 8 + 255) & ~255ull);
    sz += (uint64_t)(ZSTD_MAX_GRID + 8) * ((sizeof(ZScratch) + 255) & ~255ull);    // per-CTA scratch, sized for the largest grid we launch
    return (size_t)sz + 1024;
}

extern "C" uint64_t zmt_zstdc_out_bound(uint32_t nchunks, uint32_t chunk_size)
{
    if (chunk_size == 0) return 0;
    const uint64_t bpc = ((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK;
    return (uint64_t)nchunks * ((uint64_t)chunk_size + 12 + 9 + 3 + 32 * bpc) + 256;     // <= 5 blocks x 3-byte headers per 64 KiB window
}

extern "C" int zmt_zstd_compress_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                        uint32_t nchunks, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    if (chunk_size == 0 || nchunks == 0) return ZMT_ST_BAD_ARG;
    if (!d_chunk_bytes && nchunks != zmt_chunk_count(in_bytes, chunk_size)) return ZMT_ST_BAD_ARG;
    const uint32_t bpc = (uint32_t)(((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK);
    if ((uint64_t)nchunks * bpc > 0x7FFFFFFFull) return ZMT_ST_BAD_ARG;
    const int ti = zstd_tables_init(); if (ti != ZMT_ST_OK) return ti;
    const uint32_t nblocks = nchunks * bpc;
    uint8_t* w = (uint8_t*)d_work;
    uint8_t* tmp = w; w += (uint64_t)nblocks * ZMT_LZ4_TMP_STRIDE;
    uint32_t* blk_csize = (uint32_t*)w; w += (((uint64_t)nblocks * 4 + 255) & ~255ull);
    uint64_t* frame_size = (uint64_t*)w; w += ((((uint64_t)nchunks + 1) * 8 + 255) & ~255ull);
    ZScratch* zsc = (ZScratch*)w;
    static_assert(sizeof(ZScratch) % 8 == 0, "scratch stride");
    cudaFuncSetAttribute(zstd_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ZstdSmem));
    const uint32_t gridc = zstd_grid(nblocks);
    { ZmtProfScope ps(ZMT_K_ZSTD_COMPRESS, stream);
    zstd_blocks_kernel<<<gridc, P_TEAM, sizeof(ZstdSmem), stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, nblocks, getenv("ZSTDMT_B200_NO_TMA") ? 1u : 0u, zsc); }
    zmt_dbg_check(stream, "zstd_blocks_kernel");
    zstd_frame_sizes_kernel<<<(nchunks + 255) / 256, 256, 0, stream>>>(blk_csize, in_bytes, chunk_size, d_chunk_bytes, bpc, nchunks, frame_size);
    scan_u64_kernel<<<1, 1024, 0, stream>>>(frame_size, d_frame_off, nchunks);
    const uint32_t maxp = (uint32_t)(zmt_sm_count() * 16);
    const uint32_t gridp = nblocks < maxp ? nblocks : maxp;
    { ZmtProfScope ps(ZMT_K_ZSTD_PACK, stream);
    zstd_frame_pack_kernel<<<gridp, 256, 0, stream>>>(in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, d_frame_off, (uint8_t*)d_out, nblocks); }
    zmt_dbg_check(stream, "zstd_frame_pack_kernel");
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

static inline uint64_t a256(uint64_t x) { return (x + 255) & ~255ull; }

// ---------------------------------------------------------------- zstd compress, levels 6-22 (zstd_lazy.cuh)
// chunks per group: the per-position arrays (keys, values, prev, best: 16 bytes per position) cover one group at a time
static inline uint32_t zl_group_chunks(uint32_t nchunks, uint32_t chunk_size)
{
    uint32_t g = ZL_GROUP_BYTES / chunk_size;
    if (g == 0) g = 1;
    return g < nchunks ? g : nchunks;
}
static size_t zl_sort_temp_bytes(uint32_t npos)
{
    size_t t = 0;
    cub::DoubleBuffer<uint32_t> k(nullptr, nullptr), v(nullptr, nullptr);
    if (cub::DeviceRadixSort::SortPairs(nullptr, t, k, v, (int)npos, 0, ZL_HASHLOG) != cudaSuccess) { cudaGetLastError(); return 0; }
    return t;
}

extern "C" size_t zmt_zstdc_level_workspace_bytes(uint32_t nchunks, uint32_t chunk_size, int level)
{
    const size_t base = zmt_zstdc_workspace_bytes(nchunks, chunk_size);
    if (level < ZL_MIN_LEVEL || base == 0 || nchunks == 0) return base;
    const uint64_t npos = (uint64_t)zl_group_chunks(nchunks, chunk_size) * chunk_size;
    if (npos > 0xFFFFFFFFull) return 0;
    return base + 4 * a256(npos * 4) + a256(zl_sort_temp_bytes((uint32_t)npos));
}

extern "C" int zmt_zstd_compress_level_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                              uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    if (level < ZL_MIN_LEVEL) return zmt_zstd_compress_device(d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, d_work, d_out, d_frame_off, stream_);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (chunk_size == 0 || nchunks == 0) return ZMT_ST_BAD_ARG;
    if (!d_chunk_bytes && nchunks != zmt_chunk_count(in_bytes, chunk_size)) return ZMT_ST_BAD_ARG;
    const uint32_t bpc = (uint32_t)(((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK);
    if ((uint64_t)nchunks * bpc > 0x7FFFFFFFull) return ZMT_ST_BAD_ARG;
    const uint32_t G = zl_group_chunks(nchunks, chunk_size);
    const uint64_t npos_max = (uint64_t)G * chunk_size;
    if (npos_max > 0xFFFFFFFFull) return ZMT_ST_BAD_ARG;
    const int ti = zstd_tables_init(); if (ti != ZMT_ST_OK) return ti;
    const uint32_t nblocks = nchunks * bpc;
    uint8_t* w = (uint8_t*)d_work;
    uint8_t* tmp = w; w += (uint64_t)nblocks * ZMT_LZ4_TMP_STRIDE;
    uint32_t* blk_csize = (uint32_t*)w; w += a256((uint64_t)nblocks * 4);
    uint64_t* frame_size = (uint64_t*)w; w += a256(((uint64_t)nchunks + 1) * 8);
    ZScratch* zsc = (ZScratch*)w;
    w = (uint8_t*)d_work + zmt_zstdc_workspace_bytes(nchunks, chunk_size);        // the level-3 layout ends here
    uint32_t* arr[4];
    for (int k = 0; k < 4; k++) { arr[k] = (uint32_t*)w; w += a256(npos_max * 4); }
    void* sort_tmp = w;
    const size_t sort_cap = zl_sort_temp_bytes((uint32_t)npos_max);
    const ZlParams P = zl_params(level);
    const uint32_t W = zl_window(level);
    cudaFuncSetAttribute(zstd_lazy_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ZlSmem));

    for (uint32_t c0 = 0; c0 < nchunks; c0 += G) {
        const uint32_t ng = nchunks - c0 < G ? nchunks - c0 : G;
        uint64_t npos = (uint64_t)ng * chunk_size;
        if (!d_chunk_bytes) { const uint64_t b = (uint64_t)c0 * chunk_size; npos = in_bytes > b ? (in_bytes - b < npos ? in_bytes - b : npos) : 0; }
        cub::DoubleBuffer<uint32_t> K(arr[0], arr[1]), V(arr[2], arr[3]);
        if (npos) {
            const uint32_t np = (uint32_t)npos, g = (np + 255) / 256;
            { ZmtProfScope ps(ZMT_K_ZL_HASH, stream);
            zstd_lazy_hash_kernel<<<g, 256, 0, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, c0, np, P.min_match, K.Current(), V.Current()); }
            zmt_dbg_check(stream, "zstd_lazy_hash_kernel");
            {
                ZmtProfScope ps(ZMT_K_ZL_SORT, stream);
                size_t tb = 0;
                if (cub::DeviceRadixSort::SortPairs(nullptr, tb, K, V, (int)np, 0, ZL_HASHLOG, stream) != cudaSuccess || tb > sort_cap) return ZMT_ST_CUDA;
                if (cub::DeviceRadixSort::SortPairs(sort_tmp, tb, K, V, (int)np, 0, ZL_HASHLOG, stream) != cudaSuccess) return ZMT_ST_CUDA;
                zstd_lazy_prev_kernel<<<g, 256, 0, stream>>>(K.Current(), V.Current(), np, V.Alternate());
            }
            zmt_dbg_check(stream, "zstd_lazy sort + prev");
            { ZmtProfScope ps(ZMT_K_ZL_SEARCH, stream);
            zstd_lazy_search_kernel<ZL_BLOCK, 0, 0><<<g, 256, 0, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, c0, np, P.min_match, P.depth, W, V.Alternate(), K.Alternate()); }
            zmt_dbg_check(stream, "zstd_lazy_search_kernel");
        }
        const uint32_t nwin = ng * bpc;
        { ZmtProfScope ps(ZMT_K_ZL_BLOCKS, stream);
        zstd_lazy_blocks_kernel<<<zstd_grid(nwin), 256, sizeof(ZlSmem), stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, c0, nwin, P.lazy,
                                                                                   K.Alternate(), tmp, blk_csize, zsc); }
        zmt_dbg_check(stream, "zstd_lazy_blocks_kernel");
    }
    zstd_frame_sizes_kernel<<<(nchunks + 255) / 256, 256, 0, stream>>>(blk_csize, in_bytes, chunk_size, d_chunk_bytes, bpc, nchunks, frame_size);
    scan_u64_kernel<<<1, 1024, 0, stream>>>(frame_size, d_frame_off, nchunks);
    const uint32_t maxp = (uint32_t)(zmt_sm_count() * 16);
    const uint32_t gridp = nblocks < maxp ? nblocks : maxp;
    { ZmtProfScope ps(ZMT_K_ZSTD_PACK, stream);
    zstd_frame_pack_kernel<<<gridp, 256, 0, stream>>>(in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, d_frame_off, (uint8_t*)d_out, nblocks); }
    zmt_dbg_check(stream, "zstd_frame_pack_kernel");
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

// ---------------------------------------------------------------- LZ4 compress, levels 1-12 (levels 10-12: lz4_hc.cuh)
// The level-1 layout, then the four per-position arrays (keys, values, prev, best) of one group and the sort's temp.
extern "C" size_t zmt_lz4c_level_workspace_bytes(uint32_t nchunks, uint32_t chunk_size, int level)
{
    if (level < 1 || level > L4H_MAX_LEVEL) return 0;
    const size_t base = zmt_lz4c_workspace_bytes(nchunks, chunk_size);
    if (level < L4H_MIN_LEVEL || base == 0 || nchunks == 0) return base;
    const uint64_t npos = (uint64_t)zl_group_chunks(nchunks, chunk_size) * chunk_size;
    if (npos > 0xFFFFFFFFull) return 0;
    return base + 4 * a256(npos * 4) + a256(zl_sort_temp_bytes((uint32_t)npos));
}

extern "C" int zmt_lz4_compress_level_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                             uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream_)
{
    if (level < 1 || level > L4H_MAX_LEVEL) return ZMT_ST_BAD_ARG;
    if (level < L4H_MIN_LEVEL) return zmt_lz4_compress_device(d_in, in_bytes, chunk_size, d_chunk_bytes, nchunks, d_work, d_out, d_frame_off, stream_);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (chunk_size == 0 || nchunks == 0) return ZMT_ST_BAD_ARG;
    if (!d_chunk_bytes && nchunks != zmt_chunk_count(in_bytes, chunk_size)) return ZMT_ST_BAD_ARG;
    const uint32_t bpc = (uint32_t)(((uint64_t)chunk_size + LZ4_BLK - 1) / LZ4_BLK);
    if ((uint64_t)nchunks * bpc > 0x7FFFFFFFull) return ZMT_ST_BAD_ARG;
    const uint32_t G = zl_group_chunks(nchunks, chunk_size);
    const uint64_t npos_max = (uint64_t)G * chunk_size;
    if (npos_max > 0xFFFFFFFFull) return ZMT_ST_BAD_ARG;
    const uint32_t nblocks = nchunks * bpc;
    uint8_t* w = (uint8_t*)d_work;
    uint8_t* tmp = w; w += (uint64_t)nblocks * ZMT_LZ4_TMP_STRIDE;
    uint32_t* blk_csize = (uint32_t*)w; w += a256((uint64_t)nblocks * 4);
    uint32_t* chk = (uint32_t*)w; w += a256((uint64_t)nchunks * 4);
    uint64_t* frame_size = (uint64_t*)w;
    w = (uint8_t*)d_work + zmt_lz4c_workspace_bytes(nchunks, chunk_size);         // the level-1 layout ends here
    uint32_t* arr[4];
    for (int k = 0; k < 4; k++) { arr[k] = (uint32_t*)w; w += a256(npos_max * 4); }
    void* sort_tmp = w;
    const size_t sort_cap = zl_sort_temp_bytes((uint32_t)npos_max);
    const L4hParams P = l4h_params(level);
    cudaFuncSetAttribute(lz4_hc_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(L4hSmem));

    // the content checksum only reads the input: on the side stream it runs beside the search
    const ZmtSide side = zmt_side_stream();
    cudaStream_t xs = side.ok ? side.stream : stream;
    if (side.ok) { cudaEventRecord(side.fork, stream); cudaStreamWaitEvent(side.stream, side.fork, 0); }
    { ZmtProfScope ps(ZMT_K_XXH32, xs);
    xxh32_kernel<<<(nchunks + X_WARPS - 1) / X_WARPS, 32 * X_WARPS, 0, xs>>>((const uint8_t*)d_in, nullptr, nullptr, d_chunk_bytes, chunk_size, in_bytes, chk, nchunks); }
    if (side.ok) cudaEventRecord(side.join, side.stream);
    zmt_dbg_check(xs, "xxh32_kernel");

    for (uint32_t c0 = 0; c0 < nchunks; c0 += G) {
        const uint32_t ng = nchunks - c0 < G ? nchunks - c0 : G;
        uint64_t npos = (uint64_t)ng * chunk_size;
        if (!d_chunk_bytes) { const uint64_t b = (uint64_t)c0 * chunk_size; npos = in_bytes > b ? (in_bytes - b < npos ? in_bytes - b : npos) : 0; }
        cub::DoubleBuffer<uint32_t> K(arr[0], arr[1]), V(arr[2], arr[3]);
        if (npos) {
            const uint32_t np = (uint32_t)npos, g = (np + 255) / 256;
            { ZmtProfScope ps(ZMT_K_ZL_HASH, stream);
            zstd_lazy_hash_kernel<<<g, 256, 0, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, c0, np, L4H_MINMATCH, K.Current(), V.Current()); }
            zmt_dbg_check(stream, "zstd_lazy_hash_kernel");
            {
                ZmtProfScope ps(ZMT_K_ZL_SORT, stream);
                size_t tb = 0;
                if (cub::DeviceRadixSort::SortPairs(nullptr, tb, K, V, (int)np, 0, ZL_HASHLOG, stream) != cudaSuccess || tb > sort_cap) return ZMT_ST_CUDA;
                if (cub::DeviceRadixSort::SortPairs(sort_tmp, tb, K, V, (int)np, 0, ZL_HASHLOG, stream) != cudaSuccess) return ZMT_ST_CUDA;
                zstd_lazy_prev_kernel<<<g, 256, 0, stream>>>(K.Current(), V.Current(), np, V.Alternate());
            }
            zmt_dbg_check(stream, "zstd_lazy sort + prev");
            { ZmtProfScope ps(ZMT_K_ZL_SEARCH, stream);
            zstd_lazy_search_kernel<L4H_BLOCK, L4H_MFLIMIT, L4H_LASTLIT><<<g, 256, 0, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, c0, np,
                                                                                              L4H_MINMATCH, P.depth, L4H_WINDOW, V.Alternate(), K.Alternate()); }
            zmt_dbg_check(stream, "zstd_lazy_search_kernel");
        }
        const uint32_t nblk = ng * bpc;
        { ZmtProfScope ps(ZMT_K_L4H_BLOCKS, stream);
        lz4_hc_blocks_kernel<<<zstd_grid(nblk), 256, sizeof(L4hSmem), stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, c0, nblk, P.lazy,
                                                                                 K.Alternate(), tmp, blk_csize); }
        zmt_dbg_check(stream, "lz4_hc_blocks_kernel");
    }
    if (side.ok) cudaStreamWaitEvent(stream, side.join, 0);
    { ZmtProfScope ps(ZMT_K_LZ4_SIZES, stream);
    lz4_frame_sizes_kernel<<<(nchunks + 255) / 256, 256, 0, stream>>>(blk_csize, in_bytes, chunk_size, d_chunk_bytes, bpc, nchunks, frame_size); }
    { ZmtProfScope ps(ZMT_K_SCAN, stream);
    scan_u64_kernel<<<1, 1024, 0, stream>>>(frame_size, d_frame_off, nchunks); }
    const uint32_t maxp = (uint32_t)(zmt_sm_count() * 16);
    const uint32_t gridp = nblocks < maxp ? nblocks : maxp;
    { ZmtProfScope ps(ZMT_K_LZ4_PACK, stream);
    lz4_frame_pack_kernel<<<gridp, 256, 0, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, chk, d_frame_off, (uint8_t*)d_out, nblocks, 0u); }
    zmt_dbg_check(stream, "lz4_frame_pack_kernel");
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

// workspace: stored[] | computed[] | needs_seq[] | ticket, any-FLG.BC flag | slot counts | first_slot | block table | progress | match records
extern "C" size_t zmt_lz4d_workspace_bytes(uint32_t nframes, uint32_t nslots, uint64_t in_bytes)
{
    uint64_t sz = 3 * a256((uint64_t)nframes * 4) + 256 + 2 * a256(((uint64_t)nframes + 1) * 8) + a256(((uint64_t)nframes / LZX_WIN + 2) * 8);
    sz += a256((uint64_t)nslots * sizeof(LzBlk)) + a256((uint64_t)nslots * 4);
    sz += a256((in_bytes / 3 + 8) * 8);
    return (size_t)sz + 1024;
}

extern "C" int zmt_lz4_decompress_device(const void* d_in, uint64_t in_bytes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, uint32_t nframes,
                                         uint32_t nslots, void* d_out, const uint64_t* d_out_off, uint64_t* d_out_size,
                                         uint32_t* d_status, void* d_work, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    if (nframes == 0) return ZMT_ST_OK;
    if (nslots < nframes) return ZMT_ST_BAD_ARG;
    uint8_t* w = (uint8_t*)d_work;
    uint32_t* stored = (uint32_t*)w; w += a256((uint64_t)nframes * 4);
    uint32_t* computed = (uint32_t*)w; w += a256((uint64_t)nframes * 4);
    uint32_t* needs_seq = (uint32_t*)w; w += a256((uint64_t)nframes * 4);
    unsigned long long* ticket = (unsigned long long*)w;
    uint32_t* any_bchk = (uint32_t*)(ticket + 1); w += 256;
    unsigned long long* wbase = (unsigned long long*)w; w += a256(((uint64_t)nframes / LZX_WIN + 2) * 8);
    uint64_t* slot_cnt = (uint64_t*)w; w += a256(((uint64_t)nframes + 1) * 8);
    uint64_t* first_slot = (uint64_t*)w; w += a256(((uint64_t)nframes + 1) * 8);
    LzBlk* tab = (LzBlk*)w; w += a256((uint64_t)nslots * sizeof(LzBlk));
    uint32_t* prog = (uint32_t*)w; w += a256((uint64_t)nslots * 4);
    unsigned long long* rec = (unsigned long long*)w;
    cudaMemsetAsync(d_status, 0, (size_t)nframes * 4, stream);
    cudaMemsetAsync(d_out_size, 0, (size_t)nframes * 8, stream);
    cudaMemsetAsync(stored, 0, 3 * a256((uint64_t)nframes * 4) + 256, stream);      // stored, computed, needs_seq, ticket
    const uint8_t* in = (const uint8_t*)d_in;
    lz4_slot_counts_kernel<<<(nframes + 255) / 256, 256, 0, stream>>>(d_out_off, nframes, slot_cnt);
    scan_u64_kernel<<<1, 1024, 0, stream>>>(slot_cnt, first_slot, nframes);
    lz4_ticket_windows_kernel<<<1, 256, 0, stream>>>(first_slot, nframes, wbase);
    lz4_scan_frames_kernel<<<(nframes + 127) / 128, 128, 0, stream>>>(in, d_frame_off, d_frame_csize, d_out_off, first_slot, nslots, tab, prog, d_status, stored, needs_seq, any_bchk, nframes);
    zmt_dbg_check(stream, "lz4_scan_frames_kernel");
    {
        const uint32_t maxg = (uint32_t)(zmt_sm_count() * 8), need = (nslots + X_WARPS - 1) / X_WARPS;
        lz4_block_checksum_kernel<<<need < maxg ? need : maxg, 32 * X_WARPS, 0, stream>>>(in, d_frame_off, first_slot, tab, d_status, any_bchk, nframes, nslots);
    }
    zmt_dbg_check(stream, "lz4_block_checksum_kernel");
    { ZmtProfScope ps(ZMT_K_LZ4_DECODE, stream);
    lz4_parse_blocks_kernel<<<(nslots + LZD_WARPS - 1) / LZD_WARPS, 32 * LZD_WARPS, 0, stream>>>(
        in, in + in_bytes, d_frame_off, (uint8_t*)d_out, d_out_off, first_slot, tab, rec, (unsigned long long*)d_out_size, d_status, needs_seq, nframes, nslots); }
    zmt_dbg_check(stream, "lz4_parse_blocks_kernel");
    {
        const uint32_t maxg = (uint32_t)(zmt_sm_count() * 8);
        const uint32_t need = (nslots + LZD_WARPS - 1) / LZD_WARPS;
        ZmtProfScope ps(ZMT_K_LZ4_DEXEC, stream);
        // the shared-memory step window turns a chain of matches feeding each other into SMEM round trips instead of L2 ones
        // (DESIGN.md §3.2); ZSTDMT_B200_LZ4_STAGED=0 keeps the plain variant for A/B
        static const char* force = getenv("ZSTDMT_B200_LZ4_STAGED");
        const bool staged = force ? (*force == '1') : true;
        if (staged)
            lz4_exec_blocks_kernel<true><<<need < maxg ? need : maxg, 32 * LZD_WARPS, 0, stream>>>(
                (uint8_t*)d_out, d_out_off, d_frame_off, first_slot, tab, rec, prog, d_status, needs_seq, ticket, wbase, nframes, nslots);
        else
            lz4_exec_blocks_kernel<false><<<need < maxg ? need : maxg, 32 * LZD_WARPS, 0, stream>>>(
                (uint8_t*)d_out, d_out_off, d_frame_off, first_slot, tab, rec, prog, d_status, needs_seq, ticket, wbase, nframes, nslots);
    }
    zmt_dbg_check(stream, "lz4_exec_blocks_kernel");
    lz4_decode_frames_seq_kernel<<<(nframes + LZD_WARPS - 1) / LZD_WARPS, 32 * LZD_WARPS, 0, stream>>>(
        in, in + in_bytes, d_frame_off, d_frame_csize, (uint8_t*)d_out, d_out_off, (unsigned long long*)d_out_size, d_status, needs_seq, nframes);
    zmt_dbg_check(stream, "lz4_decode_frames_seq_kernel");
    { ZmtProfScope ps(ZMT_K_XXH32_DEC, stream);
    xxh32_kernel<<<(nframes + X_WARPS - 1) / X_WARPS, 32 * X_WARPS, 0, stream>>>((const uint8_t*)d_out, d_out_off, d_out_size, nullptr, 0, 0, computed, nframes); }
    lz4_verify_kernel<<<(nframes + 255) / 256, 256, 0, stream>>>(in, d_frame_off, d_frame_csize, d_status,
                                                                (const unsigned long long*)d_out_size, stored, computed, nframes);
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}
