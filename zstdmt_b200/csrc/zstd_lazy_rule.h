/* zstd_lazy_rule.h — the parse rule of the zstd search class for levels 6-12 (and 13-22, which use level 12's row).
 *
 * One definition shared by the GPU pipeline (zstd_lazy.cuh) and its CPU twin (oracle/chain_twin.c); plain C so
 * both compilers take it.  The rule, per chunk (= one single-segment frame):
 *   blocks  : 16 KiB zstd blocks, the last one may be short; the parse of each block starts at its first byte and no
 *             match crosses its end.
 *   chains  : h(p) = multiplicative hash of the minMatch bytes at p (p + minMatch <= chunk length);
 *             prev[p] = the largest q < p of the chunk with h(q) == h(p).
 *   best[p] : walk prev from p, at most `depth` steps, while p - q <= W; length = equal bytes, capped at
 *             min(ZL_LCAP, blockEnd - p); the longest of at least minMatch bytes, the first met on a tie; none where
 *             p + minMatch > blockEnd.
 *   parse   : at a free position p with a match m = best[p]: a literal if gain(best[p+1]) > gain(m) + 4, or, at lazy
 *             depth 2, gain(best[p+2]) > gain(m) + 7; else take m.  gain(m) = 4 len - highbit32(off + 3).
 *   merge   : a sequence with literal length 0 and the offset of the sequence before it is folded into that one.
 */
#ifndef ZSTD_LAZY_RULE_H
#define ZSTD_LAZY_RULE_H
#include <stdint.h>

#ifdef __CUDACC__
#define ZL_HD __host__ __device__ __forceinline__
#else
#define ZL_HD static inline
#endif

#define ZL_BLOCK     16384u         /* zstd block = parse unit */
#define ZL_LCAP      256u           /* match length cap of best[] (the merge undoes the cut) */
#define ZL_HASHLOG   22
#define ZL_LEN_BITS  9              /* best[] packing: length (<= 256) | offset << 9, offset < 2^23 */
#define ZL_MIN_LEVEL 6
#define ZL_MAX_LEVEL 12             /* levels above use this row */

typedef struct { uint32_t min_match, depth, lazy; } ZlParams;

/* (minMatch, chain depth, lazy depth) of levels 6..12 */
ZL_HD ZlParams zl_params(int level)
{
    const uint32_t mm[7] = { 5, 5, 5, 5, 5, 5, 5 }, dp[7] = { 8, 16, 16, 32, 48, 56, 64 }, lz[7] = { 1, 1, 2, 2, 2, 2, 2 };
    const int i = (level > ZL_MAX_LEVEL ? ZL_MAX_LEVEL : level < ZL_MIN_LEVEL ? ZL_MIN_LEVEL : level) - ZL_MIN_LEVEL;
    ZlParams p; p.min_match = mm[i]; p.depth = dp[i]; p.lazy = lz[i];
    return p;
}

/* match window: 1 << windowLog of the reference's table at the index that also picks the default chunk
 * (levels 6-9: 2 MiB, 10-12: 4 MiB) */
ZL_HD uint32_t zl_window(int level) { return (level > ZL_MAX_LEVEL ? ZL_MAX_LEVEL : level) >= 10 ? (1u << 22) : (1u << 21); }

/* h of the min_match (4 or 5) little-endian bytes held in the low bits of v */
ZL_HD uint32_t zl_hash(uint64_t v, uint32_t min_match)
{
    if (min_match == 4) return ((uint32_t)v * 2654435761u) >> (32 - ZL_HASHLOG);
    return (uint32_t)(((v << 24) * 889523592379ull) >> (64 - ZL_HASHLOG));
}

ZL_HD uint32_t zl_highbit(uint32_t v)
{
#ifdef __CUDA_ARCH__
    return 31 - __clz(v);
#else
    return 31 - __builtin_clz(v);
#endif
}

/* best[] packs length | offset << ZL_LEN_BITS */
ZL_HD uint32_t zl_len(uint32_t m) { return m & ((1u << ZL_LEN_BITS) - 1); }
ZL_HD uint32_t zl_off(uint32_t m) { return m >> ZL_LEN_BITS; }
ZL_HD int32_t zl_gain(uint32_t m) { return (int32_t)(4 * zl_len(m)) - (int32_t)zl_highbit(zl_off(m) + 3); }

/* the lazy decision at a free position whose match is m (nonzero): 1 = emit a literal, 0 = take m */
ZL_HD int zl_defer(uint32_t m, uint32_t m1, uint32_t m2, uint32_t lazy)
{
    const int32_t g = zl_gain(m);
    return (m1 && zl_gain(m1) > g + 4) || (lazy >= 2 && m2 && zl_gain(m2) > g + 7);
}

#endif
