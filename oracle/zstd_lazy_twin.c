/* zstd_lazy_twin.c — TEST INFRASTRUCTURE ONLY: the CPU twin of the GPU zstd search class for levels 6-12
 * (zstdmt_b200/csrc/zstd_lazy.cuh).  It applies the rule of zstd_lazy_rule.h serially — hash chains by a head table,
 * best[] by walking them, the lazy parse and the merge block by block — and returns each block's sequences, which the
 * tests compare with the sequences traced out of the GPU's frames. */
#include <stdlib.h>
#include <string.h>
#include "../zstdmt_b200/csrc/zstd_lazy_rule.h"

#define NONE 0xFFFFFFFFu

/* best[] of one chunk of n bytes (window W, blocks of B bytes); best must hold n + 3 zeroed words.  A match starts at
 * p only if p + minMatch <= blockEnd, so the parse of a block never reads best[] of the next one. */
static int chunk_best(const uint8_t* src, size_t n, ZlParams P, uint32_t W, uint32_t B, uint32_t* best)
{
    const uint32_t mm = P.min_match;
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
        for (size_t p = b0; p + mm <= b1; p++) {
            const uint32_t cap = (uint32_t)(b1 - p < ZL_LCAP ? b1 - p : ZL_LCAP);
            uint32_t bl = 0, bo = 0, q = prev[p];
            for (uint32_t step = 0; step < P.depth && q != NONE && p - q <= W; step++, q = prev[q]) {
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

/* best[] of one chunk of n bytes at `level` (window / block as for orc_zstd_lazy_sequences) into best[0 .. n):
 * length | offset << ZL_LEN_BITS, 0 where there is no match.  Returns 0, or -1 when memory runs out. */
int orc_zstd_lazy_best(const uint8_t* src, size_t n, int level, uint32_t window, uint32_t block, uint32_t* best)
{
    const ZlParams P = zl_params(level);
    uint32_t* b = (uint32_t*)calloc(n + 3, sizeof(uint32_t));
    if (!b || chunk_best(src, n, P, window ? window : zl_window(level), block ? block : ZL_BLOCK, b)) { free(b); return -1; }
    memcpy(best, b, sizeof(uint32_t) * n);
    free(b);
    return 0;
}

/* One chunk (= one frame) of n bytes at `level`.  window / block: 0 for the level's window and 16 KiB blocks; other
 * values shrink them so that small inputs reach their edges.  seq: 3 words per sequence (literal length, offset, match
 * length), all blocks back to back; blk_nseq[b]: sequences of block b.  Returns the number of sequences, or -1 when
 * max_seqs / max_blocks is too small or memory runs out. */
long orc_zstd_lazy_sequences(const uint8_t* src, size_t n, int level, uint32_t window, uint32_t block,
                             uint32_t* seq, size_t max_seqs, uint32_t* blk_nseq, size_t max_blocks)
{
    const ZlParams P = zl_params(level);
    const uint32_t W = window ? window : zl_window(level), B = block ? block : ZL_BLOCK;
    const size_t nblocks = (n + B - 1) / B;
    if (nblocks > max_blocks) return -1;
    uint32_t* best = (uint32_t*)calloc(n + 3, sizeof(uint32_t));
    long ns = 0;
    if (!best || chunk_best(src, n, P, W, B, best)) { ns = -1; goto done; }
    for (size_t b = 0; b < nblocks; b++) {
        const size_t b0 = b * B, b1 = b0 + B < n ? b0 + B : n;
        uint32_t nb = 0, last_off = 0;
        size_t anchor = b0;
        for (size_t p = b0; p < b1;) {
            const uint32_t m = best[p];
            if (!m) { p++; continue; }
            const int32_t g = zl_gain(m);
            if (best[p + 1] && zl_gain(best[p + 1]) > g + 4) { p++; continue; }
            if (P.lazy >= 2 && best[p + 2] && zl_gain(best[p + 2]) > g + 7) { p++; continue; }
            const uint32_t len = m & ((1u << ZL_LEN_BITS) - 1), off = m >> ZL_LEN_BITS;
            if (p == anchor && nb && off == last_off) seq[3 * (ns - 1) + 2] += len;
            else {
                if ((size_t)ns >= max_seqs) { ns = -1; goto done; }
                seq[3 * ns] = (uint32_t)(p - anchor); seq[3 * ns + 1] = off; seq[3 * ns + 2] = len;
                ns++; nb++;
            }
            last_off = off; p += len; anchor = p;
        }
        blk_nseq[b] = nb;
    }
done:
    free(best);
    return ns;
}
