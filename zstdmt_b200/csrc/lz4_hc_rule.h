/* lz4_hc_rule.h — the parse rule of the LZ4 high-compression class for levels 10-12.
 *
 * One definition shared by the GPU pipeline (lz4_hc.cuh) and its CPU twin (oracle/chain_twin.c); plain C so both
 * compilers take it.  The rule, per chunk (= one LZ4F frame with linked 64 KiB blocks, FLG 0x4C, 0x44 when empty):
 *   blocks  : 64 KiB, the chunk's last one may be short; the parse of each block starts at its first byte.  A match
 *             starts at p only if p + 12 <= blockEnd (MFLIMIT) and ends at or before blockEnd - 5 (LASTLITERALS), so a
 *             block of fewer than 13 bytes is all literals.
 *   chains  : h(p) = zl_hash of the 4 bytes at p (zstd_lazy_rule.h, 22-bit keys);
 *             prev[p] = the largest q < p of the chunk with h(q) == h(p).
 *   best[p] : walk prev from p, at most `depth` steps, while p - q <= 65535 (q may lie in an earlier block of the chunk:
 *             that is what linked blocks allow); length = equal bytes, capped at min(L4H_LCAP, blockEnd - 5 - p); the
 *             longest of at least 4 bytes, the first met (smallest offset) on a tie; none where p + 12 > blockEnd.
 *   parse   : every offset costs 2 bytes, so only lengths are compared.  At a free position p with a match m = best[p]:
 *             a literal if len(best[p+1]) > len(m) + 1, or, at lazy depth 2, len(best[p+2]) > len(m) + 2; else take m.
 *   merge   : a match with no literals before it and the offset of the match before it (in the same block) is folded
 *             into that one; this undoes the length cap.
 *   encode  : canonical LZ4 sequences, the last one literals only; a block whose encoding does not shrink it is stored
 *             raw (high bit of the block size), and is still history for the next block.
 */
#ifndef LZ4_HC_RULE_H
#define LZ4_HC_RULE_H
#include <stdint.h>
#include "zstd_lazy_rule.h"

#define L4H_BLOCK     65536u        /* LZ4F block = parse unit */
#define L4H_MINMATCH  4u
#define L4H_MFLIMIT   12u           /* a match starts at p only if p + 12 <= blockEnd */
#define L4H_LASTLIT   5u            /* ... and ends at or before blockEnd - 5 */
#define L4H_WINDOW    65535u        /* largest LZ4 offset */
#define L4H_LCAP      ZL_LCAP       /* match length cap of best[] (256; the search kernel is shared with the zstd class) */
#define L4H_MIN_LEVEL 10
#define L4H_MAX_LEVEL 12

typedef struct { uint32_t depth, lazy; } L4hParams;

/* (chain depth, lazy depth) of levels 10..12 */
ZL_HD L4hParams l4h_params(int level)
{
    const uint32_t dp[3] = { 64, 128, 256 }, lz[3] = { 2, 2, 2 };
    const int i = (level > L4H_MAX_LEVEL ? L4H_MAX_LEVEL : level < L4H_MIN_LEVEL ? L4H_MIN_LEVEL : level) - L4H_MIN_LEVEL;
    L4hParams p; p.depth = dp[i]; p.lazy = lz[i];
    return p;
}

/* the lazy decision at a free position whose match is m (nonzero; best[] packed as in the zstd class): 1 = emit a
 * literal, 0 = take m */
ZL_HD int l4h_defer(uint32_t m, uint32_t m1, uint32_t m2, uint32_t lazy)
{
    const uint32_t l = zl_len(m);
    return zl_len(m1) > l + 1 || (lazy >= 2 && zl_len(m2) > l + 2);
}

#endif
