// lz4_hc.cuh — the LZ4 high-compression class of levels 10-12: hash chains over the whole chunk, a lazy parse and
// linked 64 KiB blocks (rule: lz4_hc_rule.h; CPU twin: oracle/lz4_hc_twin.c).  Included by lz4_kernels.cu after
// zstd_lazy.cuh, whose hash, sort, prev[] and search kernels it runs with the LZ4 block and margins; the block kernel
// below writes the same per-block slots as lz4_blocks_pipe_kernel, so the LZ4 frame kernels take it from there.
//
//   lz4_hc_blocks_kernel  one CTA per 64 KiB LZ4 block.  The block is parsed in four 16 KiB quarters, in order, each by
//                         the range scheme of zstd_lazy_blocks_kernel (nx[] / ex[] over 64-position ranges, chained
//                         entries, fold flags); the parse position is carried from one quarter into the next.  Each
//                         quarter's sequences are sized, scanned and written with c_emit_seq; the last one stays open,
//                         since a match of the next quarter may still fold into it.
#pragma once
#include "lz4_hc_rule.h"

#define L4H_Q       16384u                                   // quarter: 256 threads x ZL_RANGE positions
#define L4H_MAXSEQ  (L4H_Q / L4H_MINMATCH + 2)               // sequences held: one quarter's + the open one before it
#define L4H_MAXLONG (L4H_Q / (C_LONGLIT + 1) + L4H_Q / 1290 + 8)   // literal runs > C_LONGLIT + match lengths >= 1290

struct L4hLong { uint32_t longl[2 * L4H_MAXLONG]; };         // c_emit_seq's job list

struct __align__(16) L4hSmem {
    uint16_t nx[ZL_PAD(L4H_Q)];           // next free position of the parse from p (quarter-relative)
    uint16_t ex[ZL_PAD(L4H_Q)];           // first position at or past the end of p's range that the parse reaches from p
    uint16_t entry[256];                  // first position of the true parse in each range (0xFFFF: none)
    uint32_t fold[256];                   // the range's entry match folds into the sequence before it
    uint32_t sq[L4H_MAXSEQ];              // sequence: match start (block-relative) | offset << 16
    uint32_t sl[L4H_MAXSEQ];              //           merged match length
    L4hLong  K;
    __align__(16) uint32_t scanws[40];    // block_exscan (33 words)
    uint32_t nlong, pos;                  // queued long jobs; parse position entering the next quarter (block-relative)
};
static_assert(sizeof(L4hSmem) + 1024 <= (228 * 1024) / 2, "two CTAs per SM");

__global__ void __launch_bounds__(256, 2)
lz4_hc_blocks_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                     uint32_t bpc, uint32_t c0, uint32_t nblk, uint32_t lazy, const uint32_t* __restrict__ best,
                     uint8_t* __restrict__ tmp, uint32_t* __restrict__ blk_csize)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    L4hSmem& S = *reinterpret_cast<L4hSmem*>(smem_raw);
    constexpr uint32_t NT = 256;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

    for (uint32_t w = blockIdx.x; w < nblk; w += gridDim.x) {
        const uint32_t blk = c0 * bpc + w, chunk = blk / bpc, bic = blk % bpc;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, chunk, in_bytes, chunk_size);
        const uint64_t boff = (uint64_t)bic * L4H_BLOCK;
        uint32_t n = 0;
        if (boff < cbytes) n = (uint32_t)((cbytes - boff) < L4H_BLOCK ? (cbytes - boff) : L4H_BLOCK);
        if (n == 0) { if (tid == 0) blk_csize[blk] = 0; continue; }
        uint8_t* dst = tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE;
        const uint8_t* src = in + (uint64_t)chunk * chunk_size + boff;
        const uint32_t* bb = best + (uint64_t)(chunk - c0) * chunk_size + boff;
        uint32_t out_pos = 0, pos = 0, anchor = 0;       // bytes written; parse position; end of the last written match
        uint32_t open = 0;                               // 1: sq[0] / sl[0] hold the sequence the last quarter left open

        CTA_SYNC();                                      // the previous block is done with the shared memory
        if (tid == 0) S.nlong = 0;
        for (uint32_t q0 = 0; q0 < n; q0 += L4H_Q) {
            const uint32_t nb = n - q0 < L4H_Q ? n - q0 : L4H_Q;
            const uint32_t* qb = bb + q0;
            for (uint32_t p = tid; p < nb; p += NT) {
                const uint32_t m = qb[p];
                uint32_t x = p + 1;
                if (m && !l4h_defer(m, qb[p + 1], qb[p + 2], lazy)) x = p + l4h_len(m);   // a match implies p + 12 <= n
                S.nx[ZL_PAD(p)] = (uint16_t)x;
            }
            S.entry[tid] = 0xFFFF; S.fold[tid] = 0;
            CTA_SYNC();
            const uint32_t r0 = tid * ZL_RANGE, r1 = r0 + ZL_RANGE < nb ? r0 + ZL_RANGE : nb;
            for (uint32_t p = r1; p > r0;) { p--; const uint32_t x = S.nx[ZL_PAD(p)]; S.ex[ZL_PAD(p)] = (uint16_t)(x >= r1 ? x : S.ex[ZL_PAD(x)]); }
            CTA_SYNC();
            if (tid == 0) {
                uint32_t p = pos - q0;                   // < nb: a carried position ends a match, so it is <= n - 5
                if (open && S.nx[ZL_PAD(p)] != p + 1 && (S.sq[0] & 0xFFFFu) + S.sl[0] == pos && (S.sq[0] >> 16) == (qb[p] >> ZL_LEN_BITS))
                    S.fold[p / ZL_RANGE] = 1;            // the entry match continues the sequence left open
                for (; p < nb; p = S.ex[ZL_PAD(p)]) S.entry[p / ZL_RANGE] = (uint16_t)p;
                S.pos = q0 + p;
            }
            CTA_SYNC();

            // ---- walk 1: new sequences of the range; flag a fold at the next range's entry
            const uint32_t e = S.entry[tid];
            uint32_t nseq = 0;
            bool ematch = false;
            if (e != 0xFFFFu) {
                uint32_t poff = 0;
                for (uint32_t p = e; p < r1;) {
                    const uint32_t x = S.nx[ZL_PAD(p)];
                    if (x == p + 1) poff = 0;
                    else {
                        const uint32_t off = qb[p] >> ZL_LEN_BITS;
                        if (p == e) ematch = true;
                        if (off != poff) nseq++;
                        poff = off;
                        if (x >= r1 && x < nb && S.nx[ZL_PAD(x)] != x + 1 && (qb[x] >> ZL_LEN_BITS) == off) S.fold[x / ZL_RANGE] = 1;
                    }
                    p = x;
                }
            }
            pos = S.pos;
            CTA_SYNC();
            const bool efold = ematch && S.fold[tid];
            if (efold) nseq--;
            uint32_t tot;
            const uint32_t pre = open + block_exscan(nseq, S.scanws, &tot);

            // ---- walk 2: write the sequences (a fold at the entry, and folds before the range's first new sequence, go
            // to the sequence of an earlier range or quarter: added once its owner has written it)
            uint32_t si = pre, carry = 0;
            if (e != 0xFFFFu) {
                uint32_t poff = 0, qs = 0, ql = 0;
                bool own = false;
                for (uint32_t p = e; p < r1;) {
                    const uint32_t x = S.nx[ZL_PAD(p)];
                    if (x == p + 1) poff = 0;
                    else {
                        const uint32_t off = qb[p] >> ZL_LEN_BITS, len = x - p;
                        if (p == e ? efold : off == poff) { if (own) ql += len; else carry += len; }
                        else {
                            if (own) { S.sq[si] = qs; S.sl[si] = ql; si++; }
                            qs = (q0 + p) | (off << 16); ql = len; own = true;
                        }
                        poff = off;
                    }
                    p = x;
                }
                if (own) { S.sq[si] = qs; S.sl[si] = ql; }
            }
            CTA_SYNC();
            if (carry) atomicAdd(&S.sl[pre - 1], carry);
            CTA_SYNC();

            // ---- emit every sequence but the last, which stays open unless this is the block's last quarter
            const uint32_t held = open + tot, last_q = q0 + nb == n;
            const uint32_t ne = last_q ? held : (held ? held - 1 : 0);
            const uint32_t per = (ne + NT - 1) / NT, i0 = tid * per < ne ? tid * per : ne, i1 = i0 + per < ne ? i0 + per : ne;
            uint32_t sz = 0;
            for (uint32_t i = i0; i < i1; i++) {
                const uint32_t a = i ? (S.sq[i - 1] & 0xFFFFu) + S.sl[i - 1] : anchor;
                sz += c_seq_size((S.sq[i] & 0xFFFFu) - a, S.sl[i]);
            }
            uint32_t qbytes;
            uint32_t o = out_pos + block_exscan(sz, S.scanws, &qbytes);
            for (uint32_t i = i0; i < i1; i++) {
                const uint32_t a = i ? (S.sq[i - 1] & 0xFFFFu) + S.sl[i - 1] : anchor, st = S.sq[i] & 0xFFFFu;
                o += c_emit_seq(src, S.K, S.nlong, dst, o, a, st - a, S.sq[i] >> 16, S.sl[i]);
            }
            if (ne) anchor = (S.sq[ne - 1] & 0xFFFFu) + S.sl[ne - 1];
            out_pos += qbytes;
            CTA_SYNC();
            const uint32_t nl = S.nlong;
            for (uint32_t s = wid; s < nl; s += NT / 32) c_long_job(src, S.K, dst, s, lane, 32);
            if (tid == 0) {
                S.nlong = 0;
                if (!last_q && held) { S.sq[0] = S.sq[held - 1]; S.sl[0] = S.sl[held - 1]; }
            }
            open = !last_q && held;
            CTA_SYNC();
        }

        // ---- last literals, or the whole block stored raw when the encoding does not shrink it (LZ4F rule)
        const uint32_t lit = n - anchor;
        const uint32_t hl = 1 + (lit >= 15 ? 1 + (lit - 15) / 255 : 0), fin = out_pos + hl + lit;
        if (fin >= n) { if (tid == 0) blk_csize[blk] = n | 0x80000000u; }
        else {
            uint8_t* op = dst + out_pos;
            for (uint32_t i = tid; i + 2 < hl; i += NT) op[1 + i] = 255;
            if (tid == 0) {
                op[0] = (uint8_t)((lit >= 15 ? 15u : lit) << 4);
                if (lit >= 15) op[hl - 1] = (uint8_t)(lit - 15 - (hl - 2) * 255);
                blk_csize[blk] = fin;
            }
            for (uint32_t i = tid; i < lit; i += NT) op[hl + i] = src[anchor + i];
        }
    }
}
