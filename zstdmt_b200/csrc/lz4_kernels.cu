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
//   lz77_blocks_kernel<codec,NT> one CTA per 64 KiB block (LZ4F block / zstd match window); block staged in SMEM by the TMA
//                               unit (cp.async.bulk); round-synchronous hash candidates,
//                               speculative-chain parallel greedy parse, scan-based emission.
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
#define C_NT         C_CHAINS      // smem arrays below are per chain
#define C_TILE       4096u         // positions parsed per tile
#define C_SEG        16u           // C_TILE / C_NT : positions owned by one speculative chain
#define C_ROUND      1024u         // hash-table update granularity
#define C_HASHLOG    12
#define C_MAXPIECE   1536u         // >= max pieces per tile (4096/4 match pieces + 256 continuation pieces), multiple of 512
#define C_LONGLIT    32u           // literal runs longer than this are copied cooperatively
#define C_END        0xFFFFu       // link: chain leaves the tile

struct __align__(16) CompressSmem {
    static constexpr bool relen = false;   // chain walks cache piece lengths in len[] for the marking walk
    uint8_t  pad0[16];                    // bytes "before" the block (read by the 8-byte window of phase 1, never matched)
    uint8_t  in[LZ4_BLK + 32];            // block bytes + zero pad
    uint32_t tab[1 << C_HASHLOG];         // hash -> 1 + position
    // ---- tile arrays (dead between tiles: the zstd entropy stage aliases them, see ZEnt)
    uint16_t off[C_TILE];                 // per tile position: candidate offset (0 = none)
    uint8_t  len[C_TILE];                 // per piece start: piece length (<= 19)
    uint32_t M[C_TILE / 32];              // has-candidate bits
    uint32_t V[C_TILE / 32];              // visited-by-own-chain bits
    uint32_t Sel[C_TILE / 32];            // pieces on the true greedy chain
    uint32_t Cont[C_TILE / 32];           // ... that continue the previous piece's match across a segment boundary
    uint32_t xfree[C_NT];                 // own-walk exit position (absolute)
    uint16_t xdin[C_NT];                  // own-walk exit: offset of the match we are still inside (0 = free)
    uint32_t mpos[C_NT];                  // merge position / tile exit (absolute)
    uint32_t min_[C_NT];                  // entry (free) position of a reachable chain
    uint16_t link[C_NT];                  // chain this chain merges into (C_END: leaves the tile)
    uint16_t jump[C_NT];
    uint16_t entry[8];                    // per warp: first chain of the true path inside it (0xFFFF: none)
    uint16_t piece[C_MAXPIECE];           // tile-relative start of the r-th selected piece
    uint16_t hidx[C_MAXPIECE];            // piece index of the h-th head
    uint32_t longl[3 * (C_TILE / C_LONGLIT + 2)];
    // ---- end of tile arrays
    ZFseShared fse;                       // zstd: predefined FSE encoding tables (unused by the LZ4 instantiation)
    uint32_t scanws[40];                  // block_exscan / block_exscan1 scratch (two 16-word halves + total)
    uint32_t nlong;
    uint32_t e_next;                      // chain state entering the next tile: position ...
    uint32_t d_next;                      // ... and offset of the match still open there (0 = free)
    uint64_t mbar;
};

static_assert(offsetof(CompressSmem, fse) - offsetof(CompressSmem, off) >= sizeof(ZEnt), "entropy scratch must fit in the tile arrays");

// number of bytes (<= cap) for which s[p + i] == s[p + i - d].  Word compares only: the last, partial word gets a
// sentinel bit at byte `cap` (reads run at most 3 bytes past p + cap: S.in carries 32 pad bytes).
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
//   MODE 0: own segment only (sets V, caches len, exit state -> xfree/xdin)
//   MODE 1: continuation until it merges into another chain or leaves the tile (-> link/mpos)
//   MODE 2: re-walk of a chain that is on the true path: marks Sel/Cont (same steps as MODE 0 + 1)
template <int MODE, class SM>
__device__ __forceinline__ void c_walk(SM& S, uint32_t k, uint32_t p, uint32_t din, uint32_t t0, uint32_t limit)
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
            if (MODE != 0 && j != k && ((S.M[rel >> 5] >> (rel & 31)) & 1) && S.off[rel] == din) {
                lk = j; mp = p; done = true; continue;          // chain j's own first step is this very match
            }
            uint32_t cap = p < limit ? limit - p : 0; if (cap > C_SEG) cap = C_SEG;
            const uint32_t E = c_extend(S.in, p, din, cap);
            if (MODE == 2 && E) { atomicOr(&S.Sel[rel >> 5], 1u << (rel & 31)); atomicOr(&S.Cont[rel >> 5], 1u << (rel & 31)); S.len[rel] = (uint8_t)E; }
            p += E;
            if (E != C_SEG) din = 0;
            continue;
        }
        if (MODE != 0 && j != k && (rel & (C_SEG - 1)) == 0) { lk = j; mp = p; done = true; continue; }
        uint32_t bits = (S.M[rel >> 5] >> (rel & 16)) & 0xFFFFu;     // this segment's 16 candidate bits
        bits &= 0xFFFFu << (rel & 15);
        if (!bits) {                                                   // segment exhausted: free at its end
            const uint32_t nx = t0 + (j + 1) * C_SEG;
            if (MODE == 0) { mp = nx; done = true; }
            else if (j + 1 == C_NT) { lk = C_END; mp = t1; done = true; }
            else if (j != k) { lk = j + 1; mp = nx; done = true; }
            else p = nx;
            continue;
        }
        const uint32_t qr = (rel & ~15u) + (__ffs(bits) - 1), q = t0 + qr;
        if (MODE != 0 && j != k && ((S.V[qr >> 5] >> (qr & 31)) & 1)) { lk = j; mp = q; done = true; continue; }
        const uint32_t d = S.off[qr];
        uint32_t B = (q & ~(C_SEG - 1)) + C_SEG;                     // cut at the first boundary leaving >= 4 bytes
        if (B - q < 4) B += C_SEG;
        uint32_t L;
        if (MODE == 2 && !SM::relen) { atomicOr(&S.Sel[qr >> 5], 1u << (qr & 31)); L = S.len[qr]; }
        else {
            const uint32_t end = B < limit ? B : limit;
            L = 4 + c_extend(S.in, q + 4, d, end - (q + 4));        // first 4 bytes are known equal; q + 4 <= limit always
            if (MODE == 2) { atomicOr(&S.Sel[qr >> 5], 1u << (qr & 31)); S.len[qr] = (uint8_t)L; }   // relen: len[] belongs to the marking team
            else {
                if (!SM::relen) S.len[qr] = (uint8_t)L;
                if (MODE == 0) atomicOr(&S.V[qr >> 5], 1u << (qr & 31));
            }
        }
        p = q + L;
        if (p == B) din = d;                                          // reached the boundary: still inside the match
    }
    if (MODE == 0) { S.xfree[k] = mp; S.xdin[k] = (uint16_t)din; }
    if (MODE == 1) { S.link[k] = (uint16_t)lk; S.mpos[k] = mp; if (lk == C_END) S.xdin[k] = (uint16_t)din; }
}

__device__ __forceinline__ uint32_t c_seq_size(uint32_t lit, uint32_t L)
{
    uint32_t s = 1 + lit + 2;
    if (lit >= 15) s += 1 + (lit - 15) / 255;
    if (L - 4 >= 15) s += 1 + (L - 19) / 255;
    return s;
}

// writes one LZ4 sequence at op (token, lengths, offset); literals longer than C_LONGLIT are queued for a
// warp-cooperative copy.  Returns the encoded size.
template <class SM>
__device__ __forceinline__ uint32_t c_emit_seq(SM& S, uint8_t* dst, uint32_t o, uint32_t lit_start, uint32_t lit, uint32_t off, uint32_t mlen)
{
    uint8_t* op = dst + o;
    const uint32_t ml = mlen - 4;
    *op++ = (uint8_t)(((lit >= 15 ? 15u : lit) << 4) | (ml >= 15 ? 15u : ml));
    if (SM::relen) {
        // pipelined kernel: no serial 255-runs.  The 255 bytes of a literal length exist only when lit >= 270 > C_LONGLIT
        // and are written by the warp that copies that literal run; long match-length runs become a fill job.
        static_assert(C_LONGLIT < 15 + 255, "literal-length 255 runs must imply the cooperative path");
        if (lit >= 15) { const uint32_t x = lit - 15, nf = x / 255; op += nf; *op++ = (uint8_t)(x - nf * 255); }
        if (lit <= C_LONGLIT) { for (uint32_t i = 0; i < lit; i++) op[i] = S.in[lit_start + i]; }
        else { const uint32_t s = atomicAdd(&S.nlong, 1u); S.longl[2 * s] = lit_start | (lit << 16); S.longl[2 * s + 1] = (uint32_t)(op - dst); }
        op += lit;
        *op++ = (uint8_t)off; *op++ = (uint8_t)(off >> 8);
        if (ml >= 15) {
            const uint32_t x = ml - 15, nf = x / 255;
            if (nf > 4) { const uint32_t s = atomicAdd(&S.nlong, 1u); S.longl[2 * s] = nf; S.longl[2 * s + 1] = (uint32_t)(op - dst) | 0x80000000u; op += nf; }
            else for (uint32_t i = 0; i < nf; i++) *op++ = 255;
            *op++ = (uint8_t)(x - nf * 255);
        }
        return (uint32_t)(op - (dst + o));
    }
    if (lit >= 15) { uint32_t x = lit - 15; while (x >= 255) { *op++ = 255; x -= 255; } *op++ = (uint8_t)x; }
    if (lit <= C_LONGLIT) { for (uint32_t i = 0; i < lit; i++) op[i] = S.in[lit_start + i]; }
    else { const uint32_t s = atomicAdd(&S.nlong, 1u); S.longl[3 * s] = lit_start; S.longl[3 * s + 1] = (uint32_t)(op - dst); S.longl[3 * s + 2] = lit; }
    op += lit;
    *op++ = (uint8_t)off; *op++ = (uint8_t)(off >> 8);
    if (ml >= 15) { uint32_t x = ml - 15; while (x >= 255) { *op++ = 255; x -= 255; } *op++ = (uint8_t)x; }
    return (uint32_t)(op - (dst + o));
}

// pipelined kernel: one job of the long list, done by `nthr` threads (thread index t): a literal run with the 255 bytes
// of its length field, or a run of 255 bytes of a match length
template <class SM>
__device__ __forceinline__ void c_long_job(SM& S, uint8_t* dst, uint32_t s, uint32_t t, uint32_t nthr)
{
    const uint32_t a = S.longl[2 * s], dp = S.longl[2 * s + 1];
    if (dp & 0x80000000u) { uint8_t* q = dst + (dp & 0x7FFFFFFFu); for (uint32_t i = t; i < a; i += nthr) q[i] = 255; return; }
    const uint32_t sp = a & 0xFFFFu, ln = a >> 16;
    for (uint32_t i = t; i < ln; i += nthr) dst[dp + i] = S.in[sp + i];
    const uint32_t nf = (ln - 15) / 255;                       // ln > C_LONGLIT >= 15
    uint8_t* q = dst + dp - 1 - nf;
    for (uint32_t i = t; i < nf; i += nthr) q[i] = 255;
}

// CODEC 0: LZ4 block format out.  CODEC 1: Zstandard blocks out (same candidates + parse, entropy stage per ~16 KiB).
template <int CODEC, int NTHREADS>
__global__ void __launch_bounds__(NTHREADS, 2)
lz77_blocks_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                   uint32_t bpc, uint8_t* __restrict__ tmp, uint32_t* __restrict__ blk_csize, uint32_t nblocks, uint32_t flags,
                   ZScratch* __restrict__ zscratch)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    CompressSmem& S = *reinterpret_cast<CompressSmem*>(smem_raw);
    constexpr uint32_t NT = NTHREADS;                         // threads per CTA (chains stay C_CHAINS = 256)
    static_assert(NT == 256 || NT == 512, "NT");
    static_assert(CODEC == 0 || NT == 256, "the zstd entropy stage is written for 256 threads");
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (CODEC == 1) z_load_fse_shared(S.fse, tid, NT);

    for (uint32_t blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const uint32_t chunk = blk / bpc, bic = blk % bpc;
        const uint64_t cbase = (uint64_t)chunk * chunk_size;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, chunk, in_bytes, chunk_size);
        const uint64_t boff = (uint64_t)bic * LZ4_BLK;
        uint32_t n = 0;
        if (boff < cbytes) n = (uint32_t)((cbytes - boff) < LZ4_BLK ? (cbytes - boff) : LZ4_BLK);
        if (n == 0) { if (tid == 0) blk_csize[blk] = 0; continue; }
        const uint8_t* src = in + cbase + boff;
        uint8_t* dst = tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE;

        // ---- stage the block into shared memory (TMA bulk copy when 16-byte aligned)
        CTA_SYNC();                                       // previous block fully consumed
        const uint32_t nb16 = ((((uintptr_t)src & 15) == 0) && !(flags & 1)) ? (n & ~15u) : 0;
        if (tid == 0) { if (nb16) mbar_init(&S.mbar, 1); S.nlong = 0; }
        CTA_SYNC();
        if (tid == 0 && nb16) { mbar_expect_tx(&S.mbar, nb16); bulk_g2s(S.in, src, nb16, &S.mbar); }
        for (uint32_t i = nb16 + tid; i < n; i += NT) S.in[i] = src[i];
        for (uint32_t i = n + tid; i < ((n + 3) & ~3u) + 32 && i < LZ4_BLK + 32; i += NT) S.in[i] = 0;
        if (tid < 16) S.pad0[tid] = 0;
        for (uint32_t i = tid; i < (1u << C_HASHLOG); i += NT) S.tab[i] = 0;
        // one thread observes the TMA completion; the CTA barrier publishes the staged bytes to everyone
        if (tid == 0 && nb16) { mbar_wait(&S.mbar, 0); asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(&S.mbar))); }
        CTA_SYNC();

        const uint32_t limit = n >= 5 ? n - 5 : 0;        // matches end at or before n-5
        uint32_t e = 0, e_din = 0, out_pos = 0;           // CTA-uniform parse state (position, offset of the open match)
        // pending sequence: its match may still grow in the next tile, so it is emitted one tile late
        uint32_t pd_valid = 0, pd_lit = 0, pd_start = 0, pd_off = 0, pd_end = 0;
        // zstd: sequences / literals gathered for the current sub-block, content already emitted into blocks
        ZScratch* const zs = CODEC == 1 ? zscratch + blockIdx.x : nullptr;
        ZEnt& ZE = *reinterpret_cast<ZEnt*>(&S.off[0]);
        uint32_t z_nseq = 0, z_nlit = 0, z_pos = 0, z_tiles = 0;
        const bool z_last_of_chunk = (boff + n == cbytes);
        auto cta_sync = [] () { CTA_SYNC(); };

        for (uint32_t t0 = 0; t0 < n; t0 += C_TILE) {
            // ---------------- phase 1: candidates (4 rounds of 1024 positions)
            if (tid < C_TILE / 32) { S.V[tid] = 0; S.Sel[tid] = 0; S.Cont[tid] = 0; }
            uint32_t anyM = 0;
#pragma unroll 1
            for (uint32_t r = 0; r < C_TILE / C_ROUND; r++) {
                constexpr uint32_t KPR = C_ROUND / NT;       // positions per thread per round
                uint32_t hreg[KPR];
#pragma unroll
                for (uint32_t k = 0; k < KPR; k++) {
                    const uint32_t rel = r * C_ROUND + k * NT + tid, i = t0 + rel;
                    const bool ok = (i + 12 <= n);
                    // 8-byte window: bytes i-4 .. i+3  (S.in is preceded by 16 pad bytes, so word -1 exists)
                    const uint32_t* w = reinterpret_cast<const uint32_t*>(S.in) + (i >> 2);
                    const uint32_t sh = (i & 3) * 8;
                    const uint32_t w0 = w[-1], w1 = w[0], w2 = w[1];
                    const uint32_t v = __funnelshift_r(w1, w2, sh), pv = __funnelshift_r(w0, w1, sh);
                    const uint32_t h = (v * 2654435761u) >> (32 - C_HASHLOG);
                    hreg[k] = ok ? h : 0xFFFFFFFFu;
                    uint32_t o = 0;
                    if (ok) {
                        // short-period candidates d = 1..4: v(i-d) is a byte-shift of the window
                        if (i >= 1 && __funnelshift_r(pv, v, 24) == v) o = 1;
                        else if (i >= 2 && __funnelshift_r(pv, v, 16) == v) o = 2;
                        else if (i >= 3 && __funnelshift_r(pv, v, 8) == v) o = 3;
                        else if (i >= 4 && pv == v) o = 4;
                        else {
                            const uint32_t t = S.tab[h];
                            if (t && lds32u(S.in, t - 1) == v) o = i - (t - 1);
                        }
                    }
                    S.off[rel] = (uint16_t)o;
                    const uint32_t mw = __ballot_sync(ZMT_FULL_MASK, o != 0);
                    if (lane == 0) S.M[rel >> 5] = mw;
                    anyM |= mw;
                }
                CTA_SYNC();
#pragma unroll
                for (uint32_t k = 0; k < KPR; k++)
                    if (hreg[k] != 0xFFFFFFFFu) atomicMax(&S.tab[hreg[k]], t0 + r * C_ROUND + k * NT + tid + 1);
                CTA_SYNC();
            }
            const uint32_t t1 = t0 + C_TILE;
            __syncwarp();
            const int tile_has_match = __syncthreads_or(anyM != 0);
            const bool do_parse = !((!tile_has_match && !e_din) || e >= t1);
            if (!do_parse) { if (e < t1) e = t1; }         // nothing to parse in this tile
            else do {
            // ---------------- phase 2: speculative chains (own segment, then continuation)
            const uint32_t k0 = (e - t0) / C_SEG;
            const uint32_t seg0 = t0 + tid * C_SEG;
            const bool is_chain = tid < C_CHAINS;          // threads beyond the chains only help in the data-parallel phases
            const bool alive = is_chain && tid >= k0;
            if (alive) c_walk<0>(S, tid, tid == k0 ? e : seg0, tid == k0 ? e_din : 0u, t0, limit);
            else if (is_chain) S.link[tid] = (uint16_t)tid;   // dead: self link, never reached
            CTA_SYNC();
            if (alive) c_walk<1>(S, tid, S.xfree[tid], S.xdin[tid], t0, limit);
            CTA_SYNC();
            // ---------------- phase 3: which chains lie on the true path (entry k0, follow the links)
            // Links only go forward.  Each warp resolves its own 32 chains with shuffles (pointer doubling on lane
            // indices: terminal chain + bitmask of the lanes on the way), one thread then hops from warp to warp
            // (<= 8 hops), and each warp reads its path mask back: 2 CTA barriers instead of 18.
            bool on_path;
            {
                const uint32_t lk = is_chain ? S.link[tid] : tid;
                const bool inwarp = is_chain && (lk != C_END) && (lk != tid) && ((lk >> 5) == wid);
                uint32_t jmp = inwarp ? (lk & 31) : lane;                 // next lane inside this warp (self = terminal)
                uint32_t pm = (1u << lane) | (1u << jmp);
#pragma unroll
                for (int r = 0; r < 5; r++) { pm |= __shfl_sync(ZMT_FULL_MASK, pm, jmp); jmp = __shfl_sync(ZMT_FULL_MASK, jmp, jmp); }
                if (is_chain) {
                    S.jump[tid] = (uint16_t)(32 * wid + jmp);              // terminal chain reached from tid without leaving the warp
                    S.xfree[tid] = pm;                                     // lanes on that way (xfree is dead after the continuation walk)
                }
                if (tid < 8) S.entry[tid] = 0xFFFFu;
                CTA_SYNC();
                if (tid == 0) {
                    uint32_t cur = k0;
                    S.min_[k0] = e;
                    for (;;) {
                        S.entry[cur >> 5] = (uint16_t)cur;
                        const uint32_t t = S.jump[cur], tl = S.link[t];
                        if (tl == C_END) { S.e_next = S.mpos[t]; S.d_next = S.xdin[t]; break; }
                        S.min_[tl] = S.mpos[t];                            // entry position of the next warp's first chain on the path
                        cur = tl;
                    }
                }
                CTA_SYNC();
                const uint32_t a = is_chain ? S.entry[wid] : 0xFFFFu;
                on_path = (a != 0xFFFFu) && ((S.xfree[a] >> lane) & 1u);
                if (on_path && inwarp) S.min_[lk] = S.mpos[tid];           // in-warp successor: entry position = my merge position
                __syncwarp();
            }
            // ---------------- phase 4: mark the pieces of the true chain
            if (on_path) c_walk<2>(S, tid, S.min_[tid], tid == k0 ? e_din : 0u, t0, limit);
            CTA_SYNC();
            e = S.e_next; e_din = S.d_next;

            // ---------------- phase 5: merge pieces into sequences, emit all but the last (it may still grow)
            uint32_t np;
            {
                uint32_t w = tid < C_TILE / 32 ? S.Sel[tid] : 0;
                uint32_t base = block_exscan1(__popc(w), S.scanws, 0, &np);
                while (w) { const uint32_t b = __ffs(w) - 1; w &= w - 1; S.piece[base++] = (uint16_t)(tid * 32 + b); }
            }
            CTA_SYNC();
            if (np == 0) break;
            // piece r is a HEAD unless it continues the previous piece's match: flagged continuation, or contiguous with the
            // same offset (the effective offset of a flagged piece is that of the nearest unflagged piece before it)
            uint32_t nh_local = 0, headmask = 0;
            constexpr uint32_t PPT = C_MAXPIECE / NT;     // pieces per thread
#pragma unroll
            for (uint32_t k = 0; k < PPT; k++) {
                const uint32_t r = tid * PPT + k;
                if (r < np) {
                    const uint32_t pr = S.piece[r];
                    bool head = !((S.Cont[pr >> 5] >> (pr & 31)) & 1);
                    if (head) {
                        uint32_t pend, poff;                         // end and effective offset of what precedes piece r
                        if (r == 0) { pend = pd_valid ? pd_end : 0xFFFFFFFFu; poff = pd_off; }
                        else {
                            uint32_t b = r - 1, pb = S.piece[b];
                            pend = t0 + pb + S.len[pb];
                            while (((S.Cont[pb >> 5] >> (pb & 31)) & 1) && b > 0) { b--; pb = S.piece[b]; }
                            poff = ((S.Cont[pb >> 5] >> (pb & 31)) & 1) ? pd_off : S.off[pb];
                        }
                        if (pend == t0 + pr && poff == S.off[pr]) head = false;
                    }
                    if (head) { headmask |= 1u << k; nh_local++; }
                }
            }
            uint32_t nh;
            {
                uint32_t hb = block_exscan1(nh_local, S.scanws, 1, &nh);
#pragma unroll
                for (uint32_t k = 0; k < PPT; k++) if (headmask & (1u << k)) S.hidx[hb++] = (uint16_t)(tid * PPT + k);
            }
            CTA_SYNC();
            const uint32_t lastp = S.piece[np - 1];
            const uint32_t tile_end = t0 + lastp + S.len[lastp];     // end of the last piece of this tile
            if (nh == 0) { pd_end = tile_end; break; }               // every piece extends the pending sequence
            if (pd_valid && S.hidx[0] > 0) { const uint32_t pb = S.piece[S.hidx[0] - 1]; pd_end = t0 + pb + S.len[pb]; }
            // sequences to emit now: [pending] + heads 0 .. nh-2 ; head nh-1 becomes the new pending sequence
            const uint32_t nemit = pd_valid + nh - 1;
            constexpr uint32_t SPT = 1024 / NT;           // sequences per thread (at most 1024 per tile)
            uint32_t sz = 0, e_lit0[SPT], e_lit[SPT], e_off[SPT], e_len[SPT], cnt = 0;
#pragma unroll
            for (uint32_t k = 0; k < SPT; k++) {
                const uint32_t sidx = tid * SPT + k;
                if (sidx < nemit) {
                    uint32_t ls, st, of, en;
                    if (pd_valid && sidx == 0) { ls = pd_lit; st = pd_start; of = pd_off; en = pd_end; }
                    else {
                        const uint32_t h = sidx - pd_valid;          // head index, h <= nh-2
                        const uint32_t pi = S.hidx[h], pr = S.piece[pi];
                        const uint32_t pl = S.piece[S.hidx[h + 1] - 1];
                        st = t0 + pr; of = S.off[pr]; en = t0 + pl + S.len[pl];
                        if (h == 0) ls = pd_valid ? pd_end : pd_lit;     // pd_lit doubles as "end of everything emitted so far"
                        else { const uint32_t pp = S.piece[pi - 1]; ls = t0 + pp + S.len[pp]; }
                    }
                    e_lit0[k] = ls; e_lit[k] = st - ls; e_off[k] = of; e_len[k] = en - st;
                    sz += CODEC == 0 ? c_seq_size(e_lit[k], e_len[k]) : ((1u << 18) | e_lit[k]); cnt++;   // zstd: (count, literal bytes) packed
                }
            }
            uint32_t total;
            uint32_t o = block_exscan1(sz, S.scanws, 0, &total);
            if (CODEC == 0) {
                o += out_pos;
#pragma unroll
                for (uint32_t k = 0; k < SPT; k++) {
                    if (k >= cnt) break;
                    o += c_emit_seq(S, dst, o, e_lit0[k], e_lit[k], e_off[k], e_len[k]);
                }
            } else {
                uint32_t si = z_nseq + (o >> 18), li = z_nlit + (o & 0x3FFFF);
#pragma unroll
                for (uint32_t k = 0; k < SPT; k++) {
                    if (k >= cnt) break;
                    ZSeq q; q.litlen = e_lit[k]; q.off = (uint16_t)e_off[k]; q.mlen = (uint16_t)e_len[k];
                    zs->seq[si++] = q;
                    if (e_lit[k] <= C_LONGLIT) { for (uint32_t i = 0; i < e_lit[k]; i++) zs->lit[li + i] = S.in[e_lit0[k] + i]; }
                    else { const uint32_t s = atomicAdd(&S.nlong, 1u); S.longl[3 * s] = e_lit0[k]; S.longl[3 * s + 1] = li; S.longl[3 * s + 2] = e_lit[k]; }
                    li += e_lit[k];
                }
            }
            CTA_SYNC();
            {   // cooperative copies of long literal runs: one warp per run
                const uint32_t nl = S.nlong;
                uint8_t* const ldst = CODEC == 0 ? dst : zs->lit;
                for (uint32_t s = wid; s < nl; s += NT / 32) {
                    const uint32_t sp = S.longl[3 * s], dp = S.longl[3 * s + 1], ln = S.longl[3 * s + 2];
                    for (uint32_t i = lane; i < ln; i += 32) ldst[dp + i] = S.in[sp + i];
                }
                if (CODEC == 0) out_pos += total; else { z_nseq += total >> 18; z_nlit += total & 0x3FFFF; }
                // new pending = last head of this tile
                const uint32_t pi = S.hidx[nh - 1], pr = S.piece[pi];
                uint32_t ls;
                if (nh >= 2 || pd_valid) { if (pi > 0) { const uint32_t pp = S.piece[pi - 1]; ls = t0 + pp + S.len[pp]; } else ls = pd_end; }
                else ls = pd_lit;                          // first sequence of the block: literals start where emission stands (0)
                pd_valid = 1; pd_lit = ls; pd_start = t0 + pr; pd_off = S.off[pr]; pd_end = tile_end;
                CTA_SYNC();
                if (tid == 0) S.nlong = 0;
            }
            } while (0);

            if (CODEC == 1) {
                // ---------------- zstd: close a block every 4 tiles (not at the end of the window: the final flush does that)
                z_tiles++;
                if ((z_tiles & 3) == 0 && t1 < n) {
                    CTA_SYNC();
                    // trailing literals up to C: everything before the pending match (or all parsed bytes when nothing is pending)
                    const uint32_t cover = pd_valid ? pd_lit : z_pos;
                    const uint32_t C = pd_valid ? pd_start : t1;
                    for (uint32_t i = tid; i < C - cover; i += NT) zs->lit[z_nlit + i] = S.in[cover + i];
                    const uint32_t nl = z_nlit + (C - cover);
                    CTA_SYNC();
                    if (C > z_pos) out_pos += z_encode_block(ZE, S.fse, zs, z_nseq, nl, S.in + z_pos, C - z_pos, false, dst + out_pos, S.scanws, cta_sync);
                    z_pos = C; pd_lit = C;                  // literals before C are emitted: the next sequence's literal run starts here
                    z_nseq = 0; z_nlit = 0;
                }
            }
        }

        // ---------------- flush the pending sequence + last literals
        if (CODEC == 1) {
            CTA_SYNC();
            uint32_t anchor = z_pos;
            if (pd_valid) {
                anchor = pd_end;
                const uint32_t ll = pd_start - pd_lit;
                if (tid == 0) { ZSeq q; q.litlen = ll; q.off = (uint16_t)pd_off; q.mlen = (uint16_t)(pd_end - pd_start); zs->seq[z_nseq] = q; }
                for (uint32_t i = tid; i < ll; i += NT) zs->lit[z_nlit + i] = S.in[pd_lit + i];
                z_nseq++; z_nlit += ll;
            }
            for (uint32_t i = tid; i < n - anchor; i += NT) zs->lit[z_nlit + i] = S.in[anchor + i];
            z_nlit += n - anchor;
            CTA_SYNC();
            // the frame's last block carries the Last_Block bit; an empty raw block does when nothing is left
            out_pos += z_encode_block(ZE, S.fse, zs, z_nseq, z_nlit, S.in + z_pos, n - z_pos, z_last_of_chunk, dst + out_pos, S.scanws, cta_sync);
            if (tid == 0) blk_csize[blk] = out_pos;
        } else {
            uint32_t anchor = 0;
            if (pd_valid) {
                anchor = pd_end;
                if (tid == 0) (void)c_emit_seq(S, dst, out_pos, pd_lit, pd_start - pd_lit, pd_off, pd_end - pd_start);
                out_pos += c_seq_size(pd_start - pd_lit, pd_end - pd_start);
                CTA_SYNC();
                if (S.nlong) {                              // its literal run was long: copy it with the whole CTA
                    const uint32_t sp = S.longl[0], dp = S.longl[1], ln = S.longl[2];
                    for (uint32_t i = tid; i < ln; i += NT) dst[dp + i] = S.in[sp + i];
                }
            }
            const uint32_t lit = n - anchor;
            const uint32_t fin = out_pos + 1 + lit + (lit >= 15 ? 1 + (lit - 15) / 255 : 0);
            if (fin >= n) { if (tid == 0) blk_csize[blk] = n | 0x80000000u; }   // stored block (LZ4F rule)
            else {
                uint8_t* op = dst + out_pos;
                uint32_t hl = 1;
                if (lit >= 15) hl += 1 + (lit - 15) / 255;
                if (tid == 0) {
                    uint8_t* q = op;
                    *q++ = (uint8_t)((lit >= 15 ? 15u : lit) << 4);
                    if (lit >= 15) { uint32_t x = lit - 15; while (x >= 255) { *q++ = 255; x -= 255; } *q++ = (uint8_t)x; }
                    blk_csize[blk] = fin;
                }
                for (uint32_t i = tid; i < lit; i += NT) op[hl + i] = S.in[anchor + i];
            }
        }
    }
}

#include "lz4_pipe.cuh"

// ============================================================================ XXH32 (content checksum)
// One warp per buffer.  XXH32 is four serial accumulator chains (one per 32-bit word of every 16-byte
// stripe), so the latency floor per buffer is (len/16) * ~12 cycles; everything else is about keeping the
// four chain lanes fed: all 32 lanes stream the buffer with 16-byte loads (X_DEPTH tiles of 512 B in flight
// per warp), park each tile in a per-warp shared-memory slot, and lanes 0..3 walk the slot word by word.
#define X_WARPS 8
#define X_DEPTH 4
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
    const uint8_t* p = base + off;
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
                    uint4* slot = tile[wid][d & 1];
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
    if (lane == 0) {
        uint32_t h = n >= 16 ? rotl32(a1, 1) + rotl32(a2, 7) + rotl32(a3, 12) + rotl32(a4, 18) : XXP5;
        h += (uint32_t)n;
        const uint8_t* q = p + (ns << 4);
        const uint8_t* end = p + n;
        while (q + 4 <= end) { h = rotl32(h + ldg_le32(q) * XXP3, 17) * XXP4; q += 4; }
        while (q < end) { h = rotl32(h + (*q) * XXP5, 11) * XXP1; q++; }
        h ^= h >> 15; h *= XXP2; h ^= h >> 13; h *= XXP3; h ^= h >> 16;
        out[g] = h;
    }
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
// the headers, the last block the end mark + checksum.
__global__ void __launch_bounds__(256)
lz4_frame_pack_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes, uint32_t bpc,
                      const uint8_t* __restrict__ tmp, const uint32_t* __restrict__ blk_csize,
                      const uint32_t* __restrict__ chk, const uint64_t* __restrict__ frame_off,
                      uint8_t* __restrict__ out, uint32_t nblocks)
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
                h[0] = cbytes ? 0x6C : 0x64; h[1] = 0x40;
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

    constexpr int LZ4_NT = 512;                    // 2 CTAs x 16 warps per SM: throughput scales ~linearly with resident warps (DESIGN.md §3)
    cudaFuncSetAttribute(lz77_blocks_kernel<0, LZ4_NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CompressSmem));
    const uint32_t maxc = (uint32_t)(zmt_sm_count() * 2 * 8);
    uint32_t gridc = nblocks < maxc ? nblocks : maxc;
    size_t smem_bytes = sizeof(CompressSmem);
    if (getenv("ZSTDMT_B200_OCC1")) {          // experiment knob: pad shared memory so that only one CTA fits per SM
        smem_bytes = 200 * 1024;
        cudaFuncSetAttribute(lz77_blocks_kernel<0, LZ4_NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    }
    static const bool no_pipe = getenv("ZSTDMT_B200_NOPIPE") != nullptr;   // A/B knob: single-team schedule (same output bytes)
    const ZmtSide side = zmt_side_stream();
    if (side.ok) cudaEventRecord(side.fork, stream);
    { ZmtProfScope ps(ZMT_K_LZ4_COMPRESS, stream);
    if (no_pipe || smem_bytes != sizeof(CompressSmem))
        lz77_blocks_kernel<0, LZ4_NT><<<gridc, LZ4_NT, smem_bytes, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, nblocks, getenv("ZSTDMT_B200_NO_TMA") ? 1u : 0u, nullptr);
    else {
        cudaFuncSetAttribute(lz4_blocks_pipe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PipeSmem));
        static bool occ_shown = false;
        if (!occ_shown && getenv("ZSTDMT_B200_SHOW_OCC")) {
            int nb = 0; occ_shown = true;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, lz4_blocks_pipe_kernel, 2 * P_TEAM, sizeof(PipeSmem));
            fprintf(stderr, "[zstdmt_b200] lz4_blocks_pipe_kernel: %d CTAs/SM, %zu B smem\n", nb, sizeof(PipeSmem));
        }
        lz4_blocks_pipe_kernel<<<gridc, 2 * P_TEAM, sizeof(PipeSmem), stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, nblocks, getenv("ZSTDMT_B200_NO_TMA") ? 1u : 0u);
    } }
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
    lz4_frame_pack_kernel<<<gridp, 256, 0, stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, chk, d_frame_off, (uint8_t*)d_out, nblocks); }
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
    cudaFuncSetAttribute(lz77_blocks_kernel<1, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CompressSmem));
    const uint32_t gridc = zstd_grid(nblocks);
    { ZmtProfScope ps(ZMT_K_ZSTD_COMPRESS, stream);
    lz77_blocks_kernel<1, 256><<<gridc, 256, sizeof(CompressSmem), stream>>>((const uint8_t*)d_in, in_bytes, chunk_size, d_chunk_bytes, bpc, tmp, blk_csize, nblocks, getenv("ZSTDMT_B200_NO_TMA") ? 1u : 0u, zsc); }
    zmt_dbg_check(stream, "lz77_blocks_kernel<zstd>");
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

// workspace: stored[] | computed[] | needs_seq[] | ticket | slot counts | first_slot | block table | progress | match records
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
    unsigned long long* ticket = (unsigned long long*)w; w += 256;
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
    lz4_scan_frames_kernel<<<(nframes + 127) / 128, 128, 0, stream>>>(in, d_frame_off, d_frame_csize, d_out_off, first_slot, nslots, tab, prog, d_status, stored, needs_seq, nframes);
    zmt_dbg_check(stream, "lz4_scan_frames_kernel");
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
