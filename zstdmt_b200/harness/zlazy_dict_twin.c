/* zlazy_dict_twin.c — TEST INFRASTRUCTURE ONLY: the CPU twin of the zstd search class of levels 6-12 compressing against
 * a dictionary (zmt_zstd_compress_dict_device; rule: zstdmt_b200/csrc/zstd_lazy_rule.h).  It applies the rule serially:
 * one head table over the dictionary's content D followed by the chunk, so a chunk position's chain runs through the
 * chunk and then through the linked positions of D; best[] by walking it with the dictionary's distance and length
 * caps; the lazy parse and the merge block by block.  With an empty D it is the twin of the call without a dictionary
 * (orc_zstd_lazy_sequences).  It also counts the edges of the walk a test corpus has to reach (ZDT_*). */
#include <stdlib.h>
#include <string.h>
#include "../csrc/zstd_lazy_rule.h"

#define NONE 0xFFFFFFFFu

/* stats[] counters (per position of the chunk, or per candidate) */
enum {
    ZDT_SWITCH0 = 0,        /* the walk reaches the dictionary after 0 chunk steps */
    ZDT_SWITCH_LAST,        /* ... after depth - 1 chunk steps */
    ZDT_DEPTH_IN_CHUNK,     /* depth used up in the chunk while the dictionary holds a candidate with that hash in the window */
    ZDT_DIST_W,             /* a dictionary candidate at distance exactly W is measured */
    ZDT_DIST_W1,            /* the walk stops at a dictionary candidate at distance W + 1 */
    ZDT_CAPPED_THEN_LONGER, /* a dictionary match cut at the content's end, then a longer candidate later in the walk */
    ZDT_SKIP_DICT_END,      /* a dictionary candidate skipped because bl >= dlen - q */
    ZDT_COUNT
};

static uint32_t hash_at(const uint8_t* s, uint32_t mm)
{
    uint64_t v = 0;
    for (uint32_t k = 0; k < mm; k++) v |= (uint64_t)s[k] << (8 * k);
    return zl_hash(v, mm);
}

/* best[] of chunk src[0, n) behind dictionary content d[0, dlen); best must hold n + 3 zeroed words */
static int dict_best(const uint8_t* d, size_t dlen, const uint8_t* src, size_t n, uint32_t mm, uint32_t depth, uint32_t W,
                     uint32_t B, uint32_t* best, uint64_t* stats)
{
    const size_t T = dlen + n;
    uint8_t* buf = (uint8_t*)malloc(T + 1);
    uint32_t* head = (uint32_t*)malloc(sizeof(uint32_t) << ZL_HASHLOG);
    uint32_t* prev = (uint32_t*)malloc(sizeof(uint32_t) * (T + 1));
    if (!buf || !head || !prev) { free(buf); free(head); free(prev); return -1; }
    if (dlen) memcpy(buf, d, dlen);
    if (n) memcpy(buf + dlen, src, n);
    memset(head, 0xFF, sizeof(uint32_t) << ZL_HASHLOG);
    for (size_t q = 0; q + mm <= dlen; q++) { const uint32_t h = hash_at(buf + q, mm); prev[q] = head[h]; head[h] = (uint32_t)q; }
    for (size_t p = 0; p + mm <= n; p++) {
        const size_t g = dlen + p;
        const uint32_t h = hash_at(buf + g, mm);
        prev[g] = head[h]; head[h] = (uint32_t)g;
    }
    for (size_t b0 = 0; b0 < n; b0 += B) {
        const size_t b1 = b0 + B < n ? b0 + B : n;
        for (size_t p = b0; p + mm <= b1; p++) {
            const size_t g = dlen + p;
            const uint32_t cap = (uint32_t)(b1 - p < ZL_LCAP ? b1 - p : ZL_LCAP);
            uint32_t bl = 0, bo = 0, step = 0, q = prev[g], chunk_steps = 0, capped = 0;
            int in_dict = 0;
            for (; step < depth && q != NONE; step++, q = prev[q]) {
                const size_t dist = g - q;
                if (q < dlen && !in_dict) {
                    in_dict = 1;
                    if (stats && chunk_steps == 0) stats[ZDT_SWITCH0]++;
                    if (stats && depth > 1 && chunk_steps == depth - 1) stats[ZDT_SWITCH_LAST]++;
                }
                if (dist > W) { if (stats && q < dlen && dist == (size_t)W + 1) stats[ZDT_DIST_W1]++; break; }
                if (q >= dlen) chunk_steps++;
                const uint32_t qcap = q < dlen && dlen - q < cap ? (uint32_t)(dlen - q) : cap;
                if (q < dlen && bl && bl >= qcap) { if (stats) stats[ZDT_SKIP_DICT_END]++; continue; }
                if (stats && q < dlen && dist == W) stats[ZDT_DIST_W]++;
                uint32_t l = 0;
                while (l < qcap && buf[q + l] == buf[g + l]) l++;
                if (l >= mm && l > bl) {
                    if (stats && capped) stats[ZDT_CAPPED_THEN_LONGER]++;
                    capped = q < dlen && l == qcap && qcap < cap;
                    bl = l; bo = (uint32_t)dist;
                    if (l == cap) break;
                }
            }
            if (stats && step == depth && !in_dict && q != NONE && q < dlen && g - q <= W) stats[ZDT_DEPTH_IN_CHUNK]++;
            best[p] = bl ? bl | (bo << ZL_LEN_BITS) : 0;
        }
    }
    free(buf); free(head); free(prev);
    return 0;
}

/* the parse of block [b0, b1): appends 3 words per sequence (literal length, offset, match length) to seq */
static long block_parse(const uint32_t* best, size_t b0, size_t b1, uint32_t lazy, uint32_t* seq, size_t max_seqs)
{
    long ns = 0;
    uint32_t last_off = 0;
    size_t anchor = b0;
    for (size_t p = b0; p < b1;) {
        const uint32_t m = best[p];
        if (!m || zl_defer(m, best[p + 1], best[p + 2], lazy)) { p++; continue; }
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

/* best[] of one chunk of n bytes at `level` against content d[0, dlen) (window / block 0: the level's window and
 * 16 KiB blocks); stats: NULL or ZDT_COUNT counters, added to.  Returns 0, or -1 when memory runs out. */
int orc_zstd_lazy_best_dict(const uint8_t* d, size_t dlen, const uint8_t* src, size_t n, int level, uint32_t window, uint32_t block,
                            uint32_t* best, uint64_t* stats)
{
    const ZlParams P = zl_params(level);
    uint32_t* b = (uint32_t*)calloc(n + 3, sizeof(uint32_t));
    if (!b || dict_best(d, dlen, src, n, P.min_match, P.depth, window ? window : zl_window(level), block ? block : ZL_BLOCK, b, stats)) {
        free(b); return -1;
    }
    memcpy(best, b, sizeof(uint32_t) * n);
    free(b);
    return 0;
}

/* One chunk (= one frame) of n bytes at `level` against content d[0, dlen), returned as orc_zstd_lazy_sequences returns
 * it: 3 words per sequence, all blocks back to back; blk_nseq[b]: sequences of block b.  Returns the number of
 * sequences, or -1 when max_seqs / max_blocks is too small or memory runs out. */
long orc_zstd_lazy_sequences_dict(const uint8_t* d, size_t dlen, const uint8_t* src, size_t n, int level, uint32_t window,
                                  uint32_t block, uint32_t* seq, size_t max_seqs, uint32_t* blk_nseq, size_t max_blocks, uint64_t* stats)
{
    const ZlParams P = zl_params(level);
    const uint32_t B = block ? block : ZL_BLOCK;
    const size_t nblocks = (n + B - 1) / B;
    if (nblocks > max_blocks) return -1;
    uint32_t* best = (uint32_t*)calloc(n + 3, sizeof(uint32_t));
    long ns = 0;
    if (!best || dict_best(d, dlen, src, n, P.min_match, P.depth, window ? window : zl_window(level), B, best, stats)) { free(best); return -1; }
    for (size_t b = 0; b < nblocks; b++) {
        const size_t b0 = b * B, b1 = b0 + B < n ? b0 + B : n;
        const long k = block_parse(best, b0, b1, P.lazy, seq + 3 * ns, max_seqs - (size_t)ns);
        if (k < 0) { ns = -1; break; }
        blk_nseq[b] = (uint32_t)k; ns += k;
    }
    free(best);
    return ns;
}
