/* oracle/lz4_oracle.c — TEST INFRASTRUCTURE ONLY (see oracle.h).
 *
 * CPU restatement of the LZ4 side of zstdmt's per-chunk hot path:
 *   - XXH32                      (content + header checksum inside LZ4F; liblz4 v1.9.4 xxhash.c [ext])
 *   - LZ4 block decode           (what LZ4F_decompress does per block; call site
 *                                 lib/lz4-mt_decompress.c:349-351)
 *   - LZ4 frame decode / encode  (LZ4F_compressFrame call site lib/lz4-mt_compress.c:280-283;
 *                                 preferences lib/lz4-mt_compress.c:141-146)
 *   - the 12-byte skippable container (lib/lz4-mt_compress.c:293-298 write,
 *                                 lib/lz4-mt_decompress.c:192-281 read)
 *   - orc_lz4_block_compress_b200: the bit-exact CPU twin of OUR sm_90a
 *     compressor (the reference's compressed bytes are not a parity target;
 *     BASELINE.json north_star: "produces a stream the reference CPU path
 *     decompresses to the identical input").
 * Pinned by tests/test_oracle.py against SURVEY.md Appendix A vectors and the
 * real reference build (oracle/_ref).
 */
#include "oracle.h"
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ helpers */
static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static uint64_t rd64(const uint8_t* p) { return (uint64_t)rd32(p) | ((uint64_t)rd32(p + 4) << 32); }
static void wr32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
static void wr64(uint8_t* p, uint64_t v) { wr32(p, (uint32_t)v); wr32(p + 4, (uint32_t)(v >> 32)); }

/* -------------------------------------------------------------------- XXH32 */
#define XP1 0x9E3779B1u
#define XP2 0x85EBCA77u
#define XP3 0xC2B2AE3Du
#define XP4 0x27D4EB2Fu
#define XP5 0x165667B1u
static uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
static uint32_t xround(uint32_t acc, uint32_t lane) { return rotl32(acc + lane * XP2, 13) * XP1; }

uint32_t orc_xxh32(const void* data, size_t len, uint32_t seed)
{
    const uint8_t* p = (const uint8_t*)data;
    const uint8_t* end = p + len;
    uint32_t h;
    if (len >= 16) {
        uint32_t a1 = seed + XP1 + XP2, a2 = seed + XP2, a3 = seed, a4 = seed - XP1;
        const uint8_t* lim = end - 16;
        do {
            a1 = xround(a1, rd32(p));
            a2 = xround(a2, rd32(p + 4));
            a3 = xround(a3, rd32(p + 8));
            a4 = xround(a4, rd32(p + 12));
            p += 16;
        } while (p <= lim);
        h = rotl32(a1, 1) + rotl32(a2, 7) + rotl32(a3, 12) + rotl32(a4, 18);
    } else {
        h = seed + XP5;
    }
    h += (uint32_t)len;
    while (p + 4 <= end) { h = rotl32(h + rd32(p) * XP3, 17) * XP4; p += 4; }
    while (p < end)      { h = rotl32(h + (*p) * XP5, 11) * XP1; p++; }
    h ^= h >> 15; h *= XP2; h ^= h >> 13; h *= XP3; h ^= h >> 16;
    return h;
}

/* --------------------------------------------------------- LZ4 block decode */
/* tr != NULL: one ORC_L4S_* row per sequence; token positions are counted from src - base (the frame start) */
static long block_decode(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t prefix,
                         orc_lz4f_trace_t* tr, size_t base)
{
    const uint8_t* ip = src;
    const uint8_t* const iend = src + srcSize;
    uint8_t* op = dst;
    uint8_t* const oend = dst + dstCap;
    if (srcSize == 0) return ORC_ERR_BLOCK;
    for (;;) {
        size_t lit, ml, off, tokpos = (size_t)(ip - src), llext, mlext, mdst;
        unsigned token;
        int64_t* row;
        if (ip >= iend) return ORC_ERR_BLOCK;
        token = *ip++;
        lit = token >> 4;
        if (lit == 15) {
            unsigned b;
            do { if (ip >= iend) return ORC_ERR_BLOCK; b = *ip++; lit += b; } while (b == 255);
        }
        llext = (size_t)(ip - src) - tokpos - 1;
        if (lit > (size_t)(iend - ip)) return ORC_ERR_BLOCK;
        if (lit > (size_t)(oend - op)) return ORC_ERR_DST_SMALL;
        memcpy(op, ip, lit); ip += lit; op += lit;
        off = ml = mlext = 0; mdst = (size_t)(op - dst);
        if (ip != iend) {
            const uint8_t* e;
            if ((size_t)(iend - ip) < 2) return ORC_ERR_BLOCK;
            off = (size_t)ip[0] | ((size_t)ip[1] << 8); ip += 2;
            if (off == 0 || off > (size_t)(op - dst) + prefix) return ORC_ERR_BLOCK;
            ml = token & 15; e = ip;
            if (ml == 15) {
                unsigned b;
                do { if (ip >= iend) return ORC_ERR_BLOCK; b = *ip++; ml += b; } while (b == 255);
            }
            mlext = (size_t)(ip - e);
            ml += 4;
            if (ml > (size_t)(oend - op)) return ORC_ERR_DST_SMALL;
            { const uint8_t* m = op - off; size_t i; for (i = 0; i < ml; i++) op[i] = m[i]; }
            op += ml;
        }
        if (tr) {
            if (tr->nseqs >= tr->max_seqs) return ORC_ERR_DST_SMALL;
            row = tr->seq + tr->nseqs++ * ORC_L4S_NF;
            row[ORC_L4S_TOKPOS] = (int64_t)(base + tokpos); row[ORC_L4S_LLEXT] = (int64_t)llext; row[ORC_L4S_MLEXT] = (int64_t)mlext;
            row[ORC_L4S_LL] = (int64_t)lit; row[ORC_L4S_OFF] = (int64_t)off; row[ORC_L4S_ML] = (int64_t)ml; row[ORC_L4S_DST] = (int64_t)mdst;
        }
        if (!ml) break;                             /* last sequence: literals only; a block ending after a match is malformed */
    }
    return (long)(op - dst);
}

long orc_lz4_block_decode(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t prefix)
{
    return block_decode(src, srcSize, dst, dstCap, prefix, NULL, 0);
}

/* --------------------------------- GPU compressor twin (deterministic spec)
 * Spec shared with zstdmt_b200/csrc/lz4_kernels.cu (DESIGN.md "LZ4 encoder"):
 *   eligible(i)  : i + 12 <= n                (LZ4 MFLIMIT: no match starts in the last 12 bytes)
 *   v(i)         : LE32 at i;  h(i) = (v * 2654435761) >> 20          (12-bit hash)
 *   rounds of 1024 positions; table[h] = 1 + max eligible position with hash h in EARLIER rounds
 *   local cand   : smallest d in 1..4 (d <= i) with v(i-d) == v(i)        (runs / short periods)
 *   table cand   : table[h(i)]-1 if v(cand) == v(i)
 *   off(i)       : d  else  i - table  else 0 (no match)
 *   parse        : greedy — first match start >= p, length extended while
 *                  q+L < n-5 (LASTLITERALS); p = q + L
 */
#define B200_HASHLOG 12
#define B200_ROUND   1024
#define B200_LOCAL   4

size_t orc_lz4_block_bound(size_t n) { return n + n / 255 + 16; }

static uint8_t* put_len(uint8_t* op, size_t len)   /* len already reduced by 15 */
{
    while (len >= 255) { *op++ = 255; len -= 255; }
    *op++ = (uint8_t)len;
    return op;
}

/* candidate offsets for every position of a block (0 = no match); exported for tests/tools */
void orc_lz4_b200_offsets(const uint8_t* src, size_t n, uint16_t* off)
{
    uint32_t* table = (uint32_t*)calloc((size_t)1 << B200_HASHLOG, sizeof(uint32_t));
    size_t i, r;
    memset(off, 0, n * sizeof(uint16_t));
    for (r = 0; r < n; r += B200_ROUND) {
        size_t rend = r + B200_ROUND < n ? r + B200_ROUND : n;
        for (i = r; i < rend; i++) {
            uint32_t v; size_t d; int found = 0;
            if (i + 12 > n) continue;
            v = rd32(src + i);
            for (d = 1; d <= B200_LOCAL && d <= i; d++) {    /* short-period candidate: smallest d with identical 4 bytes */
                if (rd32(src + i - d) == v) { off[i] = (uint16_t)d; found = 1; break; }
            }
            if (!found) {
                uint32_t t = table[(v * 2654435761u) >> (32 - B200_HASHLOG)];
                if (t && rd32(src + (t - 1)) == v) off[i] = (uint16_t)(i - (t - 1));
            }
        }
        for (i = r; i < rend; i++) {
            if (i + 12 > n) continue;
            table[(rd32(src + i) * 2654435761u) >> (32 - B200_HASHLOG)] = (uint32_t)i + 1;
        }
    }
    free(table);
}

size_t orc_lz4_block_compress_b200(const uint8_t* src, size_t n, uint8_t* dst, size_t dstCap)
{
    uint16_t* off = (uint16_t*)calloc(n ? n : 1, sizeof(uint16_t));
    uint8_t* op = dst;
    size_t anchor = 0, p = 0;
    if (dstCap < orc_lz4_block_bound(n) || n > 65536) { free(off); return 0; }
    orc_lz4_b200_offsets(src, n, off);

    while (p < n) {
        size_t q = p, L, c, lit;
        uint8_t* tok;
        while (q < n && off[q] == 0) q++;
        if (q >= n) break;
        c = q - off[q];
        L = 4;
        while (q + L < n - 5 && src[q + L] == src[c + L]) L++;
        lit = q - anchor;
        tok = op++;
        if (lit >= 15) { *tok = 0xF0; op = put_len(op, lit - 15); } else *tok = (uint8_t)(lit << 4);
        memcpy(op, src + anchor, lit); op += lit;
        *op++ = (uint8_t)off[q]; *op++ = (uint8_t)(off[q] >> 8);
        if (L - 4 >= 15) { *tok |= 15; op = put_len(op, L - 4 - 15); } else *tok |= (uint8_t)(L - 4);
        p = anchor = q + L;
    }
    {   /* last literals */
        size_t lit = n - anchor;
        uint8_t* tok = op++;
        if (lit >= 15) { *tok = 0xF0; op = put_len(op, lit - 15); } else *tok = (uint8_t)(lit << 4);
        memcpy(op, src + anchor, lit); op += lit;
    }
    free(off);
    return (size_t)(op - dst);
}

/* ---------------------------------------------------------------- LZ4 frame */
#define LZ4F_MAGIC 0x184D2204u
static const size_t k_blkmax[8] = { 0, 0, 0, 0, 65536, 262144, 1048576, 4194304 };

static int lz4f_decode(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap,
                       size_t* outSize, size_t* consumed, orc_lz4f_trace_t* tr)
{
    const uint8_t* ip = src;
    const uint8_t* const iend = src + srcSize;
    size_t hdrlen, blkmax, total = 0;
    unsigned flg, bd, indep, bchk, csz, cchk, dictid;
    uint64_t content = 0;
    if (srcSize < 7) return ORC_ERR_TRUNCATED;
    if (rd32(ip) != LZ4F_MAGIC) return ORC_ERR_BAD_MAGIC;
    flg = ip[4]; bd = ip[5];
    if ((flg >> 6) != 1 || (flg & 0x02)) return ORC_ERR_BAD_HEADER;
    indep = (flg >> 5) & 1; bchk = (flg >> 4) & 1; csz = (flg >> 3) & 1; cchk = (flg >> 2) & 1; dictid = flg & 1;
    if ((bd & 0x8F) || ((bd >> 4) & 7) < 4) return ORC_ERR_BAD_HEADER;
    blkmax = k_blkmax[(bd >> 4) & 7];
    hdrlen = 2 + (csz ? 8 : 0) + (dictid ? 4 : 0);
    if (srcSize < 4 + hdrlen + 1) return ORC_ERR_TRUNCATED;
    if (csz) content = rd64(ip + 6);
    if (((orc_xxh32(ip + 4, hdrlen, 0) >> 8) & 0xFF) != ip[4 + hdrlen]) return ORC_ERR_HDR_CHECKSUM;
    ip += 4 + hdrlen + 1;
    if (tr) tr->nblocks = tr->nseqs = 0;
    for (;;) {
        uint32_t bh; size_t bs;
        int64_t* row = NULL;
        if ((size_t)(iend - ip) < 4) return ORC_ERR_TRUNCATED;
        bh = rd32(ip); ip += 4;
        if (bh == 0) break;
        bs = bh & 0x7FFFFFFFu;
        if (bs > blkmax) return ORC_ERR_BLOCK;
        if ((size_t)(iend - ip) < bs + (bchk ? 4 : 0)) return ORC_ERR_TRUNCATED;
        if (tr) {
            if (tr->nblocks >= tr->max_blocks) return ORC_ERR_DST_SMALL;
            row = tr->blk + tr->nblocks++ * ORC_L4B_NF;
            row[ORC_L4B_FOFF] = (int64_t)(ip - src); row[ORC_L4B_BSIZE] = (int64_t)bs; row[ORC_L4B_STORED] = (bh >> 31) != 0;
            row[ORC_L4B_REGEN] = -1; row[ORC_L4B_LINKED] = !indep; row[ORC_L4B_BCHK] = bchk;
            row[ORC_L4B_BCHK_OK] = bchk ? orc_xxh32(ip, bs, 0) == rd32(ip + bs) : -1;
            row[ORC_L4B_SEQ_FIRST] = (int64_t)tr->nseqs; row[ORC_L4B_NSEQ] = 0; row[ORC_L4B_DST] = (int64_t)total;
        }
        if (bh & 0x80000000u) {
            if (bs > dstCap - total) return ORC_ERR_DST_SMALL;
            memcpy(dst + total, ip, bs); total += bs;
            if (row) row[ORC_L4B_REGEN] = (int64_t)bs;
        } else {
            size_t prefix = indep ? 0 : (total < 65536 ? total : 65536);
            size_t cap = dstCap - total < blkmax ? dstCap - total : blkmax;
            long d = block_decode(ip, bs, dst + total, cap, prefix, tr, (size_t)(ip - src));
            if (d < 0) return (int)d;
            total += (size_t)d;
            if (row) { row[ORC_L4B_REGEN] = d; row[ORC_L4B_NSEQ] = (int64_t)tr->nseqs - row[ORC_L4B_SEQ_FIRST]; }
        }
        if (bchk && orc_xxh32(ip, bs, 0) != rd32(ip + bs)) return ORC_ERR_BLOCK;
        ip += bs + (bchk ? 4 : 0);
    }
    if (cchk) {
        if ((size_t)(iend - ip) < 4) return ORC_ERR_TRUNCATED;
        if (orc_xxh32(dst, total, 0) != rd32(ip)) return ORC_ERR_CONTENT_CHECKSUM;
        ip += 4;
    }
    if (csz && content != total) return ORC_ERR_CONTENT_SIZE;
    if (outSize) *outSize = total;
    if (consumed) *consumed = (size_t)(ip - src);
    return ORC_OK;
}

int orc_lz4f_decode(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t* outSize, size_t* consumed)
{
    return lz4f_decode(src, srcSize, dst, dstCap, outSize, consumed, NULL);
}

int orc_lz4f_trace(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t* outSize, size_t* consumed,
                   orc_lz4f_trace_t* tr)
{
    return lz4f_decode(src, srcSize, dst, dstCap, outSize, consumed, tr);
}

size_t orc_lz4f_bound(size_t n)
{
    size_t nblk = (n + 65535) / 65536;
    return 4 + 2 + 8 + 1 + nblk * 4 + n + 4 + 4;
}

size_t orc_lz4f_encode_b200(const uint8_t* src, size_t n, uint8_t* dst, size_t dstCap)
{
    uint8_t* op = dst;
    uint8_t* tmp;
    size_t pos, hl;
    if (dstCap < orc_lz4f_bound(n)) return 0;
    wr32(op, LZ4F_MAGIC);
    op[4] = n ? 0x6C : 0x64;          /* v01 | independent | [contentSize] | contentChecksum */
    op[5] = 0x40;                     /* 64 KiB blocks */
    hl = 2;
    if (n) { wr64(op + 6, (uint64_t)n); hl = 10; }
    op[4 + hl] = (uint8_t)(orc_xxh32(op + 4, hl, 0) >> 8);
    op += 4 + hl + 1;
    tmp = (uint8_t*)malloc(orc_lz4_block_bound(65536));
    for (pos = 0; pos < n; pos += 65536) {
        size_t bn = n - pos < 65536 ? n - pos : 65536;
        size_t cs = orc_lz4_block_compress_b200(src + pos, bn, tmp, orc_lz4_block_bound(65536));
        if (cs >= bn) { wr32(op, (uint32_t)bn | 0x80000000u); memcpy(op + 4, src + pos, bn); op += 4 + bn; }
        else          { wr32(op, (uint32_t)cs); memcpy(op + 4, tmp, cs); op += 4 + cs; }
    }
    free(tmp);
    wr32(op, 0); op += 4;
    wr32(op, orc_xxh32(src, n, 0)); op += 4;
    return (size_t)(op - dst);
}

/* ------------------------------------------------------------- MT container */
#define MT_SKIPPABLE 0x184D2A50u

long orc_mt_scan(const uint8_t* src, size_t srcSize, uint64_t* offsets, uint32_t* csize, size_t maxFrames)
{
    size_t pos = 0; long nf = 0;
    while (pos < srcSize) {
        uint32_t cs;
        if (srcSize - pos < 12) return ORC_ERR_TRUNCATED;
        if (rd32(src + pos) != MT_SKIPPABLE) return ORC_ERR_BAD_MAGIC;
        if (rd32(src + pos + 4) != 4) return ORC_ERR_BAD_HEADER;
        cs = rd32(src + pos + 8);
        if (srcSize - pos - 12 < cs) return ORC_ERR_TRUNCATED;
        if ((size_t)nf < maxFrames) { if (offsets) offsets[nf] = pos; if (csize) csize[nf] = cs; }
        nf++;
        pos += 12 + (size_t)cs;
    }
    return nf;
}

int orc_mt_decode(int codec, const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t* outSize)
{
    size_t pos = 0, total = 0;
    while (pos < srcSize) {
        uint32_t cs; size_t got = 0, used = 0; int rc;
        if (srcSize - pos < 12) return ORC_ERR_TRUNCATED;
        if (rd32(src + pos) != MT_SKIPPABLE) return ORC_ERR_BAD_MAGIC;
        if (rd32(src + pos + 4) != 4) return ORC_ERR_BAD_HEADER;
        cs = rd32(src + pos + 8);
        if (srcSize - pos - 12 < cs) return ORC_ERR_TRUNCATED;
        if (codec == ORC_CODEC_LZ4) rc = orc_lz4f_decode(src + pos + 12, cs, dst + total, dstCap - total, &got, &used);
        else                        rc = orc_zstd_decode(src + pos + 12, cs, dst + total, dstCap - total, &got, &used);
        if (rc != ORC_OK) return rc;
        if (used != cs) return ORC_ERR_CORRUPT;
        total += got;
        pos += 12 + (size_t)cs;
    }
    if (outSize) *outSize = total;
    return ORC_OK;
}

size_t orc_mt_encode_lz4_b200(const uint8_t* src, size_t n, size_t chunk, uint8_t* dst, size_t dstCap)
{
    size_t pos = 0, out = 0;
    do {                                             /* empty input still yields one frame (lz4-mt_compress.c:265) */
        size_t cn = n - pos < chunk ? n - pos : chunk;
        size_t fs;
        if (dstCap - out < 12 + orc_lz4f_bound(cn)) return 0;
        fs = orc_lz4f_encode_b200(src + pos, cn, dst + out + 12, dstCap - out - 12);
        wr32(dst + out, MT_SKIPPABLE); wr32(dst + out + 4, 4); wr32(dst + out + 8, (uint32_t)fs);
        out += 12 + fs; pos += cn;
    } while (pos < n);
    return out;
}
