/* chain_twin.c — TEST INFRASTRUCTURE ONLY: the CPU twin of the GPU chain-search encoders, the zstd class of levels
 * 6-12 (zstdmt_b200/csrc/zstd_lazy.cuh) and the LZ4 high-compression class of levels 10-12 (lz4_hc.cuh).  It applies
 * the rules of zstd_lazy_rule.h and lz4_hc_rule.h serially — hash chains by a head table, best[] by walking them, the
 * lazy parse and the merge block by block — and returns each block's sequences, which the tests compare with the
 * sequences traced out of the GPU's frames; for LZ4 it also writes the whole framed stream (12-byte container headers,
 * LZ4F frames with linked blocks, raw blocks where the encoding does not shrink), which the tests compare byte for
 * byte with what the GPU writes. */
#include <stdlib.h>
#include <string.h>
#include "../zstdmt_b200/csrc/lz4_hc_rule.h"

#define NONE 0xFFFFFFFFu

/* best[] of one chunk of n bytes (hash of mm bytes, window W, blocks of B bytes); best must hold n + 3 zeroed words.
 * start / end are the margins of the GPU search kernel: a match starts at p only if p + (start ? start : mm) <= blockEnd
 * and ends at or before blockEnd - end (zstd: 0, 0; LZ4: 12, 5).  So the parse of a block never reads best[] past it. */
static int chunk_best(const uint8_t* src, size_t n, uint32_t mm, uint32_t start, uint32_t end, uint32_t depth, uint32_t W,
                      uint32_t B, uint32_t* best)
{
    const uint32_t first = start ? start : mm;
    uint32_t* head = (uint32_t*)malloc(sizeof(uint32_t) << ZL_HASHLOG);
    uint32_t* prev = (uint32_t*)malloc(sizeof(uint32_t) * (n + 1));
    if (!head || !prev) { free(head); free(prev); return -1; }
    memset(head, 0xFF, sizeof(uint32_t) << ZL_HASHLOG);
    for (size_t p = 0; p + mm <= n; p++) {
        uint64_t v = 0;
        for (uint32_t k = 0; k < mm; k++) v |= (uint64_t)src[p + k] << (8 * k);
        const uint32_t h = zl_hash(v, mm);
        prev[p] = head[h]; head[h] = (uint32_t)p;
    }
    for (size_t b0 = 0; b0 < n; b0 += B) {
        const size_t b1 = b0 + B < n ? b0 + B : n;
        for (size_t p = b0; p + first <= b1; p++) {
            const uint32_t cap = (uint32_t)(b1 - end - p < ZL_LCAP ? b1 - end - p : ZL_LCAP);
            uint32_t bl = 0, bo = 0, q = prev[p];
            for (uint32_t step = 0; step < depth && q != NONE && p - q <= W; step++, q = prev[q]) {
                uint32_t l = 0;
                while (l < cap && src[q + l] == src[p + l]) l++;
                if (l >= mm && l > bl) { bl = l; bo = (uint32_t)(p - q); if (l == cap) break; }
            }
            best[p] = bl ? bl | (bo << ZL_LEN_BITS) : 0;
        }
    }
    free(head); free(prev);
    return 0;
}

/* the class's lazy decision: zl_defer or l4h_defer */
typedef int (*Defer)(uint32_t m, uint32_t m1, uint32_t m2, uint32_t lazy);

/* the parse of block [b0, b1): appends 3 words per sequence (literal length, offset, match length) to seq */
static long block_parse(const uint32_t* best, size_t b0, size_t b1, uint32_t lazy, Defer defer, uint32_t* seq, size_t max_seqs)
{
    long ns = 0;
    uint32_t last_off = 0;
    size_t anchor = b0;
    for (size_t p = b0; p < b1;) {
        const uint32_t m = best[p];
        if (!m || defer(m, best[p + 1], best[p + 2], lazy)) { p++; continue; }
        const uint32_t len = zl_len(m), off = zl_off(m);
        if (p == anchor && ns && off == last_off) seq[3 * (ns - 1) + 2] += len;
        else {
            if ((size_t)ns >= max_seqs) return -1;
            seq[3 * ns] = (uint32_t)(p - anchor); seq[3 * ns + 1] = off; seq[3 * ns + 2] = len;
            ns++;
        }
        last_off = off; p += len; anchor = p;
    }
    return ns;
}

/* best[] of one chunk into best[0 .. n): length | offset << ZL_LEN_BITS, 0 where there is no match */
static int chunk_best_out(const uint8_t* src, size_t n, uint32_t mm, uint32_t start, uint32_t end, uint32_t depth,
                          uint32_t W, uint32_t B, uint32_t* best)
{
    uint32_t* b = (uint32_t*)calloc(n + 3, sizeof(uint32_t));
    if (!b || chunk_best(src, n, mm, start, end, depth, W, B, b)) { free(b); return -1; }
    memcpy(best, b, sizeof(uint32_t) * n);
    free(b);
    return 0;
}

/* the sequences of one chunk, block by block: 3 words per sequence, all blocks back to back; blk_nseq[b]: sequences
 * of block b */
static long chunk_sequences(const uint8_t* src, size_t n, uint32_t mm, uint32_t start, uint32_t end, uint32_t depth,
                            uint32_t lazy, Defer defer, uint32_t W, uint32_t B,
                            uint32_t* seq, size_t max_seqs, uint32_t* blk_nseq, size_t max_blocks)
{
    const size_t nblocks = (n + B - 1) / B;
    if (nblocks > max_blocks) return -1;
    uint32_t* best = (uint32_t*)calloc(n + 3, sizeof(uint32_t));
    long ns = 0;
    if (!best || chunk_best(src, n, mm, start, end, depth, W, B, best)) { free(best); return -1; }
    for (size_t b = 0; b < nblocks; b++) {
        const size_t b0 = b * B, b1 = b0 + B < n ? b0 + B : n;
        const long k = block_parse(best, b0, b1, lazy, defer, seq + 3 * ns, max_seqs - (size_t)ns);
        if (k < 0) { ns = -1; break; }
        blk_nseq[b] = (uint32_t)k; ns += k;
    }
    free(best);
    return ns;
}

/* ---- zstd levels 6-12: window / block 0 for the level's window and 16 KiB blocks; other values shrink them so that
 * small inputs reach their edges */

/* best[] of one chunk of n bytes at `level`.  Returns 0, or -1 when memory runs out. */
int orc_zstd_lazy_best(const uint8_t* src, size_t n, int level, uint32_t window, uint32_t block, uint32_t* best)
{
    const ZlParams P = zl_params(level);
    return chunk_best_out(src, n, P.min_match, 0, 0, P.depth, window ? window : zl_window(level), block ? block : ZL_BLOCK, best);
}

/* One chunk (= one frame) of n bytes at `level`.  seq: 3 words per sequence (literal length, offset, match length),
 * all blocks back to back; blk_nseq[b]: sequences of block b.  Returns the number of sequences, or -1 when max_seqs /
 * max_blocks is too small or memory runs out. */
long orc_zstd_lazy_sequences(const uint8_t* src, size_t n, int level, uint32_t window, uint32_t block,
                             uint32_t* seq, size_t max_seqs, uint32_t* blk_nseq, size_t max_blocks)
{
    const ZlParams P = zl_params(level);
    return chunk_sequences(src, n, P.min_match, 0, 0, P.depth, P.lazy, zl_defer, window ? window : zl_window(level),
                           block ? block : ZL_BLOCK, seq, max_seqs, blk_nseq, max_blocks);
}

/* ---- LZ4 levels 10-12: window / block 0 for 65535 and 64 KiB blocks; other values shrink them */

/* best[] of one chunk of n bytes at `level`.  Returns 0, or -1 when memory runs out. */
int orc_lz4_hc_best(const uint8_t* src, size_t n, int level, uint32_t window, uint32_t block, uint32_t* best)
{
    const L4hParams P = l4h_params(level);
    return chunk_best_out(src, n, L4H_MINMATCH, L4H_MFLIMIT, L4H_LASTLIT, P.depth, window ? window : L4H_WINDOW,
                          block ? block : L4H_BLOCK, best);
}

/* One chunk of n bytes at `level`, returned as for orc_zstd_lazy_sequences */
long orc_lz4_hc_sequences(const uint8_t* src, size_t n, int level, uint32_t window, uint32_t block,
                          uint32_t* seq, size_t max_seqs, uint32_t* blk_nseq, size_t max_blocks)
{
    const L4hParams P = l4h_params(level);
    return chunk_sequences(src, n, L4H_MINMATCH, L4H_MFLIMIT, L4H_LASTLIT, P.depth, P.lazy, l4h_defer,
                           window ? window : L4H_WINDOW, block ? block : L4H_BLOCK, seq, max_seqs, blk_nseq, max_blocks);
}

/* ---- LZ4 framing */
static uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static void wr32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

static uint32_t xxh32(const uint8_t* p, size_t len)
{
    const uint32_t P1 = 0x9E3779B1u, P2 = 0x85EBCA77u, P3 = 0xC2B2AE3Du, P4 = 0x27D4EB2Fu, P5 = 0x165667B1u;
    const uint8_t* end = p + len;
    uint32_t h;
    if (len >= 16) {
        uint32_t a[4] = { P1 + P2, P2, 0, 0u - P1 };
        for (; p + 16 <= end; p += 16)
            for (int j = 0; j < 4; j++) a[j] = rotl32(a[j] + rd32(p + 4 * j) * P2, 13) * P1;
        h = rotl32(a[0], 1) + rotl32(a[1], 7) + rotl32(a[2], 12) + rotl32(a[3], 18);
    } else h = P5;
    h += (uint32_t)len;
    for (; p + 4 <= end; p += 4) h = rotl32(h + rd32(p) * P3, 17) * P4;
    for (; p < end; p++) h = rotl32(h + (*p) * P5, 11) * P1;
    h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
    return h;
}

static uint8_t* put_len(uint8_t* op, uint32_t x) { for (; x >= 255; x -= 255) *op++ = 255; *op++ = (uint8_t)x; return op; }

/* the LZ4 block of [src, src + bn) from its sequences; returns its size */
static size_t block_encode(const uint8_t* src, size_t bn, const uint32_t* seq, long ns, uint8_t* op0)
{
    uint8_t* op = op0;
    size_t pos = 0;
    for (long i = 0; i < ns; i++) {
        const uint32_t ll = seq[3 * i], off = seq[3 * i + 1], ml = seq[3 * i + 2] - L4H_MINMATCH;
        *op++ = (uint8_t)(((ll >= 15 ? 15u : ll) << 4) | (ml >= 15 ? 15u : ml));
        if (ll >= 15) op = put_len(op, ll - 15);
        memcpy(op, src + pos, ll); op += ll; pos += ll;
        *op++ = (uint8_t)off; *op++ = (uint8_t)(off >> 8);
        if (ml >= 15) op = put_len(op, ml - 15);
        pos += ml + L4H_MINMATCH;
    }
    const size_t ll = bn - pos;
    *op++ = (uint8_t)((ll >= 15 ? 15u : ll) << 4);
    if (ll >= 15) op = put_len(op, (uint32_t)(ll - 15));
    memcpy(op, src + pos, ll); op += ll;
    return (size_t)(op - op0);
}

/* room for one chunk's frame: an encoded block is written before it is known to shrink, and may exceed its input by
 * bn / 255 + 2 bytes */
static size_t frame_bound(size_t n) { return 12 + 4 + 2 + 8 + 1 + n + ((n + 65535) / 65536) * (4 + 300) + 4 + 4; }

/* The framed stream of src cut every `chunk` bytes at `level`, as zmt_lz4_compress_level_device writes it: per chunk
 * a 12-byte container header and an LZ4F frame (FLG 0x4C, or 0x44 when the chunk is empty; BD 0x40; content size;
 * linked 64 KiB blocks; end mark; XXH32 of the content).  An empty input gives one empty frame.  Returns the bytes
 * written, or 0 when dst_cap is too small or memory runs out. */
size_t orc_lz4_hc_compress(const uint8_t* src, size_t n, size_t chunk, int level, uint8_t* dst, size_t dst_cap)
{
    const L4hParams P = l4h_params(level);
    size_t pos = 0, out = 0;
    uint32_t* best = (uint32_t*)calloc((chunk < n ? chunk : n) + 3, sizeof(uint32_t));
    uint32_t* seq = (uint32_t*)malloc(sizeof(uint32_t) * 3 * (L4H_BLOCK / L4H_MINMATCH + 1));
    if (!best || !seq || !chunk) { out = 0; goto done; }
    do {
        const size_t cn = n - pos < chunk ? n - pos : chunk;
        const uint8_t* s = src + pos;
        if (dst_cap - out < frame_bound(cn)) { out = 0; goto done; }
        memset(best, 0, sizeof(uint32_t) * (cn + 3));
        if (chunk_best(s, cn, L4H_MINMATCH, L4H_MFLIMIT, L4H_LASTLIT, P.depth, L4H_WINDOW, L4H_BLOCK, best)) { out = 0; goto done; }
        uint8_t* f = dst + out;
        uint8_t* op = f + 12;
        wr32(op, 0x184D2204u);
        op[4] = cn ? 0x4C : 0x44; op[5] = 0x40;
        size_t hl = 2;
        if (cn) { wr32(op + 6, (uint32_t)cn); wr32(op + 10, (uint32_t)((uint64_t)cn >> 32)); hl = 10; }
        op[4 + hl] = (uint8_t)(xxh32(op + 4, hl) >> 8);
        op += 4 + hl + 1;
        for (size_t b0 = 0; b0 < cn; b0 += L4H_BLOCK) {
            const size_t b1 = b0 + L4H_BLOCK < cn ? b0 + L4H_BLOCK : cn, bn = b1 - b0;
            const long ns = block_parse(best, b0, b1, P.lazy, l4h_defer, seq, L4H_BLOCK / L4H_MINMATCH + 1);
            if (ns < 0) { out = 0; goto done; }
            const size_t cs = block_encode(s + b0, bn, seq, ns, op + 4);
            if (cs >= bn) { wr32(op, (uint32_t)bn | 0x80000000u); memcpy(op + 4, s + b0, bn); op += 4 + bn; }
            else { wr32(op, (uint32_t)cs); op += 4 + cs; }
        }
        wr32(op, 0); wr32(op + 4, xxh32(s, cn)); op += 8;
        wr32(f, 0x184D2A50u); wr32(f + 4, 4); wr32(f + 8, (uint32_t)(op - f - 12));
        out += (size_t)(op - f); pos += cn;
    } while (pos < n);
done:
    free(best); free(seq);
    return out;
}
