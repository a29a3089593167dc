/* oracle/zstd_oracle.c — TEST INFRASTRUCTURE ONLY (see oracle.h).
 *
 * CPU restatement of the Zstandard frame decoder (RFC 8878 [ext]) — the
 * arithmetic behind ZSTD_decompressStream at
 * lib/zstd-mt_decompress.c:456,625 (libzstd v1.5.6 is a
 * build-time clone, programs/Makefile:11,245, not in the reference tree).
 * Full format: raw / RLE / compressed blocks; literals raw / RLE / Huffman
 * (1 or 4 streams, direct or FSE-coded weights, treeless reuse); sequences
 * with predefined / RLE / FSE-described / repeat tables; repeat offsets;
 * optional XXH64 content checksum.  No dictionaries, no legacy formats.
 * Pinned by tests/test_oracle.py against frames produced by the real libzstd
 * (through oracle/_ref) and the golden vectors in tests/golden/.
 */
#include "oracle.h"
#include <stdlib.h>
#include <string.h>

static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static uint64_t rd64(const uint8_t* p) { return (uint64_t)rd32(p) | ((uint64_t)rd32(p + 4) << 32); }
static int highbit(uint32_t v) { int r = 0; while (v >>= 1) r++; return r; }

/* -------------------------------------------------------------------- XXH64 */
#define P64_1 0x9E3779B185EBCA87ULL
#define P64_2 0xC2B2AE3D27D4EB4FULL
#define P64_3 0x165667B19E3779F9ULL
#define P64_4 0x85EBCA77C2B2AE63ULL
#define P64_5 0x27D4EB2F165667C5ULL
static uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t x64round(uint64_t acc, uint64_t in) { return rotl64(acc + in * P64_2, 31) * P64_1; }
static uint64_t x64merge(uint64_t acc, uint64_t v) { acc ^= x64round(0, v); return acc * P64_1 + P64_4; }
static uint64_t xxh64(const uint8_t* p, size_t len, uint64_t seed)
{
    const uint8_t* end = p + len; uint64_t h;
    if (len >= 32) {
        uint64_t v1 = seed + P64_1 + P64_2, v2 = seed + P64_2, v3 = seed, v4 = seed - P64_1;
        const uint8_t* lim = end - 32;
        do { v1 = x64round(v1, rd64(p)); v2 = x64round(v2, rd64(p + 8)); v3 = x64round(v3, rd64(p + 16)); v4 = x64round(v4, rd64(p + 24)); p += 32; } while (p <= lim);
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = x64merge(h, v1); h = x64merge(h, v2); h = x64merge(h, v3); h = x64merge(h, v4);
    } else h = seed + P64_5;
    h += (uint64_t)len;
    while (p + 8 <= end) { h ^= x64round(0, rd64(p)); h = rotl64(h, 27) * P64_1 + P64_4; p += 8; }
    if (p + 4 <= end)    { h ^= (uint64_t)rd32(p) * P64_1; h = rotl64(h, 23) * P64_2 + P64_3; p += 4; }
    while (p < end)      { h ^= (*p) * P64_5; h = rotl64(h, 11) * P64_1; p++; }
    h ^= h >> 33; h *= P64_2; h ^= h >> 29; h *= P64_3; h ^= h >> 32;
    return h;
}

/* -------------------------------------------------- backward bit reader
 * RFC 8878 §4.1 / §3.1.1.3.2.1.1: streams are written forward and read from
 * the last byte; the highest set bit of the last byte is a padding marker.
 * `off` is the number of unread bits; reads past the start return zeros and
 * drive `off` negative (how "stream exhausted" is detected). */
typedef struct { const uint8_t* p; long off; } bbits;
static int bb_init(bbits* b, const uint8_t* p, size_t n)
{
    if (n == 0 || p[n - 1] == 0) return -1;
    b->p = p; b->off = (long)n * 8 - (8 - highbit(p[n - 1]));
    return 0;
}
static uint64_t bb_read(bbits* b, int nb)
{
    uint64_t v = 0; long start; int i;
    if (nb == 0) return 0;
    b->off -= nb; start = b->off;
    for (i = 0; i < nb; i++) { long bit = start + i; if (bit >= 0) v |= (uint64_t)((b->p[bit >> 3] >> (bit & 7)) & 1) << i; }
    return v;
}

/* ---------------------------------------------------------------- FSE tables */
#define FSE_MAXLOG 9
#define FSE_MAXSYM 256
typedef struct { uint8_t sym[1 << FSE_MAXLOG]; uint8_t nb[1 << FSE_MAXLOG]; uint16_t base[1 << FSE_MAXLOG]; int log; } fse_dtab;

static int fse_build(fse_dtab* t, const int16_t* norm, int nsym, int log)
{
    int size = 1 << log, high = size - 1, s, i, pos = 0, step = (size >> 1) + (size >> 3) + 3;
    uint16_t next[FSE_MAXSYM];
    if (log > FSE_MAXLOG) return -1;
    t->log = log;
    for (s = 0; s < nsym; s++) {
        if (norm[s] == -1) { t->sym[high--] = (uint8_t)s; next[s] = 1; }
        else next[s] = (uint16_t)norm[s];
    }
    for (s = 0; s < nsym; s++) {
        for (i = 0; i < norm[s]; i++) {
            t->sym[pos] = (uint8_t)s;
            do { pos = (pos + step) & (size - 1); } while (pos > high);
        }
    }
    if (pos != 0) return -1;
    for (i = 0; i < size; i++) {
        uint16_t x = next[t->sym[i]]++;
        t->nb[i] = (uint8_t)(log - highbit(x));
        t->base[i] = (uint16_t)(((uint32_t)x << t->nb[i]) - size);
    }
    return 0;
}
static void fse_build_rle(fse_dtab* t, uint8_t sym) { t->log = 0; t->sym[0] = sym; t->nb[0] = 0; t->base[0] = 0; }

/* normalized-count header (forward bit order); returns bytes consumed or <0 */
static long fse_read_ncount(const uint8_t* src, size_t n, int16_t* norm, int* nsym, int* log, int maxlog, int maxsym)
{
    uint64_t bitpos = 0; int al, remaining, threshold, nbits, sym = 0, prev0 = 0;
#define PEEK(k) ((uint32_t)(((bitpos >> 3) < n ? ( \
        ((uint64_t)src[bitpos >> 3]) | ((bitpos >> 3) + 1 < n ? (uint64_t)src[(bitpos >> 3) + 1] << 8 : 0) | \
        ((bitpos >> 3) + 2 < n ? (uint64_t)src[(bitpos >> 3) + 2] << 16 : 0) | ((bitpos >> 3) + 3 < n ? (uint64_t)src[(bitpos >> 3) + 3] << 24 : 0) | \
        ((bitpos >> 3) + 4 < n ? (uint64_t)src[(bitpos >> 3) + 4] << 32 : 0)) : 0) >> (bitpos & 7)) & ((1u << (k)) - 1))
    if (n < 1) return -1;
    al = (int)PEEK(4) + 5; bitpos += 4;
    if (al > maxlog) return -1;
    remaining = (1 << al) + 1; threshold = 1 << al; nbits = al + 1;
    while (remaining > 1 && sym <= maxsym) {
        int max, count;
        if (prev0) {
            for (;;) { uint32_t rep = PEEK(2); bitpos += 2; sym += (int)rep; if (rep != 3) break; }
            if (sym > maxsym + 1) return -1;
            prev0 = 0;
            /* the zero-run symbols keep norm = 0 (array pre-zeroed) */
            if (sym > maxsym) break;
        }
        max = (2 * threshold - 1) - remaining;
        {
            uint32_t lo = PEEK(nbits - 1);
            if ((int)lo < max) { count = (int)lo; bitpos += (uint64_t)(nbits - 1); }
            else {
                uint32_t full = PEEK(nbits);
                count = (int)full;
                if (count >= threshold) count -= max;
                bitpos += (uint64_t)nbits;
            }
        }
        count--;
        remaining -= count < 0 ? -count : count;
        norm[sym++] = (int16_t)count;
        prev0 = (count == 0);
        while (remaining < threshold) { nbits--; threshold >>= 1; }
    }
#undef PEEK
    if (remaining != 1 || sym > maxsym + 1) return -1;
    if (((bitpos + 7) >> 3) > n) return -1;
    *nsym = sym; *log = al;
    return (long)((bitpos + 7) >> 3);
}

/* ------------------------------------------------------------------ Huffman */
#define HUF_MAXBITS 11
typedef struct { uint8_t sym[1 << HUF_MAXBITS]; uint8_t nb[1 << HUF_MAXBITS]; int maxbits; int valid; } huf_dtab;

/* `full` (may be NULL) receives the weights of all nw + 1 symbols, the implied last one included */
static int huf_build(huf_dtab* h, const uint8_t* weights, int nw /* explicit weights */, uint8_t* full)
{
    uint32_t total = 0, rank[HUF_MAXBITS + 2], left; int i, maxbits, lastw, nsym = nw + 1;
    uint8_t w[256];
    if (nw < 1 || nw > 255) return -1;
    for (i = 0; i < nw; i++) { if (weights[i] > HUF_MAXBITS) return -1; w[i] = weights[i]; if (w[i]) total += 1u << (w[i] - 1); }
    if (total == 0) return -1;
    maxbits = highbit(total) + 1;
    if (maxbits > HUF_MAXBITS) return -1;
    left = (1u << maxbits) - total;
    if (left == 0 || (left & (left - 1))) return -1;           /* must be a power of two */
    lastw = highbit(left) + 1; w[nw] = (uint8_t)lastw;
    memset(rank, 0, sizeof(rank));
    for (i = 0; i < nsym; i++) rank[w[i]]++;
    {   /* start index per weight: ascending weight, then symbol order */
        uint32_t start[HUF_MAXBITS + 2], acc = 0; int wt;
        for (wt = 1; wt <= maxbits; wt++) { start[wt] = acc; acc += rank[wt] << (wt - 1); }
        if (acc != (1u << maxbits)) return -1;
        for (i = 0; i < nsym; i++) {
            uint32_t len, k;
            if (!w[i]) continue;
            len = 1u << (w[i] - 1);
            for (k = 0; k < len; k++) { h->sym[start[w[i]] + k] = (uint8_t)i; h->nb[start[w[i]] + k] = (uint8_t)(maxbits + 1 - w[i]); }
            start[w[i]] += len;
        }
    }
    h->maxbits = maxbits; h->valid = 1;
    if (full) memcpy(full, w, (size_t)nsym);
    return 0;
}

/* *form: 0 direct 4-bit weights, 1 FSE-coded; *nwl: weights listed; full: see huf_build */
static int huf_read_tree(huf_dtab* h, const uint8_t* src, size_t n, size_t* used, int* form, int* nwl, uint8_t* full)
{
    uint8_t weights[256]; int nw = 0; unsigned hb;
    if (n < 1) return -1;
    hb = src[0];
    if (hb >= 128) {
        int cnt = (int)hb - 127, i; size_t bytes = (size_t)(cnt + 1) / 2;
        if (n < 1 + bytes) return -1;
        for (i = 0; i < cnt; i++) weights[i] = (i & 1) ? (src[1 + i / 2] & 15) : (src[1 + i / 2] >> 4);
        nw = cnt; *used = 1 + bytes;
    } else {
        int16_t norm[16]; int nsym = 0, log = 0; long hl; fse_dtab t; bbits b; uint32_t s1, s2;
        if (hb == 0 || n < 1 + (size_t)hb) return -1;
        memset(norm, 0, sizeof(norm));
        hl = fse_read_ncount(src + 1, hb, norm, &nsym, &log, 6, 15);
        if (hl < 0) return -1;
        if (fse_build(&t, norm, nsym, log)) return -1;
        if (bb_init(&b, src + 1 + hl, hb - (size_t)hl)) return -1;
        s1 = (uint32_t)bb_read(&b, log); s2 = (uint32_t)bb_read(&b, log);
        if (b.off < 0) return -1;
        for (;;) {
            if (nw >= 254) return -1;
            weights[nw++] = t.sym[s1]; s1 = t.base[s1] + (uint32_t)bb_read(&b, t.nb[s1]);
            if (b.off < 0) { weights[nw++] = t.sym[s2]; break; }
            if (nw >= 254) return -1;
            weights[nw++] = t.sym[s2]; s2 = t.base[s2] + (uint32_t)bb_read(&b, t.nb[s2]);
            if (b.off < 0) { weights[nw++] = t.sym[s1]; break; }
        }
        *used = 1 + (size_t)hb;
    }
    *form = hb < 128; *nwl = nw;
    return huf_build(h, weights, nw, full);
}

static int huf_decode_stream(const huf_dtab* h, const uint8_t* src, size_t n, uint8_t* dst, size_t count)
{
    bbits b; uint32_t state; size_t i; int mb = h->maxbits;
    if (bb_init(&b, src, n)) return -1;
    state = (uint32_t)bb_read(&b, mb);
    for (i = 0; i < count; i++) {
        int nb = h->nb[state];
        dst[i] = h->sym[state];
        state = ((state << nb) & ((1u << mb) - 1)) | (uint32_t)bb_read(&b, nb);
    }
    /* all bits consumed exactly: after the last symbol we over-read maxbits of look-ahead */
    if (b.off != -(long)mb) return -1;
    return 0;
}

/* ------------------------------------------------------- sequence constants */
static const uint32_t LL_base[36] = { 0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,18,20,22,24,28,32,40,48,64,128,256,512,1024,2048,4096,8192,16384,32768,65536 };
static const uint8_t  LL_bits[36] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16 };
static const uint32_t ML_base[53] = { 3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,35,37,39,41,43,47,51,59,67,83,99,131,259,515,1027,2051,4099,8195,16387,32771,65539 };
static const uint8_t  ML_bits[53] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16 };
static const int16_t LL_defnorm[36] = { 4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1 };
static const int16_t ML_defnorm[53] = { 1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1 };
static const int16_t OF_defnorm[29] = { 1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1 };

typedef struct {
    huf_dtab huf;
    fse_dtab ll, of, ml; int have_ll, have_of, have_ml;
    uint32_t rep[3];
} zctx;

static int read_seq_table(fse_dtab* t, int* have, int mode, const uint8_t** ip, const uint8_t* iend,
                          const int16_t* defnorm, int defsyms, int deflog, int maxlog, int maxsym)
{
    switch (mode) {
    case 0: if (fse_build(t, defnorm, defsyms, deflog)) return -1; *have = 1; return 0;
    case 1: if (*ip >= iend) return -1; if (**ip > maxsym) return -1; fse_build_rle(t, **ip); (*ip)++; *have = 1; return 0;
    case 2: {
        int16_t norm[64]; int nsym = 0, log = 0; long hl;
        memset(norm, 0, sizeof(norm));
        hl = fse_read_ncount(*ip, (size_t)(iend - *ip), norm, &nsym, &log, maxlog, maxsym);
        if (hl < 0) return -1;
        if (fse_build(t, norm, nsym, log)) return -1;
        *ip += hl; *have = 1; return 0; }
    default: return *have ? 0 : -1;             /* repeat */
    }
}

/* tr: trace sink, NULL when decoding normally; tb / tw: this block's record and weights (set up by the caller) */
static int decode_block(zctx* z, const uint8_t* src, size_t n, uint8_t* dstBase, size_t dstPos, size_t dstCap, size_t* produced,
                        orc_zstd_trace_t* tr, int32_t* tb, uint8_t* tw)
{
    const uint8_t* ip = src; const uint8_t* const iend = src + n;
    uint8_t* lit = NULL; size_t litSize = 0; int rc = ORC_ERR_CORRUPT;
    uint8_t* op = dstBase + dstPos; uint8_t* const oend = dstBase + dstCap;
    /* ---- literals section ---- */
    {
        unsigned b0, type, sf; size_t regen, comp = 0, hl; int streams = 1;
        if (n < 1) return ORC_ERR_CORRUPT;
        b0 = ip[0]; type = b0 & 3; sf = (b0 >> 2) & 3;
        if (type < 2) {
            if (sf == 0 || sf == 2) { regen = b0 >> 3; hl = 1; }
            else if (sf == 1) { if (n < 2) return ORC_ERR_CORRUPT; regen = (b0 >> 4) | ((size_t)ip[1] << 4); hl = 2; }
            else { if (n < 3) return ORC_ERR_CORRUPT; regen = (b0 >> 4) | ((size_t)ip[1] << 4) | ((size_t)ip[2] << 12); hl = 3; }
            ip += hl;
            if (tr) { tb[ORC_ZT_LIT_TYPE] = (int32_t)type; tb[ORC_ZT_LIT_SF] = (int32_t)sf; tb[ORC_ZT_LIT_HDR] = (int32_t)hl; tb[ORC_ZT_LIT_REGEN] = (int32_t)regen; }
            lit = (uint8_t*)malloc(regen + 1); litSize = regen;
            if (type == 0) { if ((size_t)(iend - ip) < regen) goto done; memcpy(lit, ip, regen); ip += regen; }
            else { if (iend - ip < 1) goto done; memset(lit, *ip, regen); ip++; }
        } else {
            if (sf == 0 || sf == 1) { if (n < 3) return ORC_ERR_CORRUPT; { uint32_t v = ip[0] | (ip[1] << 8) | ((uint32_t)ip[2] << 16); regen = (v >> 4) & 0x3FF; comp = (v >> 14) & 0x3FF; } hl = 3; streams = sf == 0 ? 1 : 4; }
            else if (sf == 2) { if (n < 4) return ORC_ERR_CORRUPT; { uint32_t v = rd32(ip); regen = (v >> 4) & 0x3FFF; comp = (v >> 18) & 0x3FFF; } hl = 4; streams = 4; }
            else { if (n < 5) return ORC_ERR_CORRUPT; { uint64_t v = (uint64_t)rd32(ip) | ((uint64_t)ip[4] << 32); regen = (size_t)((v >> 4) & 0x3FFFF); comp = (size_t)((v >> 22) & 0x3FFFF); } hl = 5; streams = 4; }
            ip += hl;
            if (tr) {
                tb[ORC_ZT_LIT_TYPE] = (int32_t)type; tb[ORC_ZT_LIT_SF] = (int32_t)sf; tb[ORC_ZT_LIT_HDR] = (int32_t)hl;
                tb[ORC_ZT_LIT_REGEN] = (int32_t)regen; tb[ORC_ZT_LIT_COMP] = (int32_t)comp; tb[ORC_ZT_LIT_STREAMS] = streams;
            }
            if ((size_t)(iend - ip) < comp) return ORC_ERR_CORRUPT;
            lit = (uint8_t*)malloc(regen + 1); litSize = regen;
            {
                const uint8_t* lp = ip; const uint8_t* const lend = ip + comp;
                if (type == 2) {
                    size_t used = 0; int form = 0, nwl = 0;
                    if (huf_read_tree(&z->huf, lp, comp, &used, &form, &nwl, tw)) goto done;
                    lp += used;
                    if (tr) { tb[ORC_ZT_TREE_FORM] = form; tb[ORC_ZT_TREE_BYTES] = (int32_t)used; tb[ORC_ZT_NWEIGHTS] = nwl; tb[ORC_ZT_MAXBITS] = z->huf.maxbits; }
                }
                else if (!z->huf.valid) goto done;
                else if (tr) tb[ORC_ZT_MAXBITS] = z->huf.maxbits;
                if (streams == 1) { if (huf_decode_stream(&z->huf, lp, (size_t)(lend - lp), lit, regen)) goto done; }
                else {
                    size_t s1, s2, s3, s4, per = (regen + 3) / 4;
                    if (lend - lp < 6) goto done;
                    s1 = lp[0] | (lp[1] << 8); s2 = lp[2] | (lp[3] << 8); s3 = lp[4] | (lp[5] << 8); lp += 6;
                    if (s1 + s2 + s3 > (size_t)(lend - lp)) goto done;
                    s4 = (size_t)(lend - lp) - s1 - s2 - s3;
                    if (per * 3 > regen) goto done;
                    if (huf_decode_stream(&z->huf, lp, s1, lit, per)) goto done;
                    if (huf_decode_stream(&z->huf, lp + s1, s2, lit + per, per)) goto done;
                    if (huf_decode_stream(&z->huf, lp + s1 + s2, s3, lit + 2 * per, per)) goto done;
                    if (huf_decode_stream(&z->huf, lp + s1 + s2 + s3, s4, lit + 3 * per, regen - 3 * per)) goto done;
                    if (tr) { tb[ORC_ZT_S1] = (int32_t)s1; tb[ORC_ZT_S2] = (int32_t)s2; tb[ORC_ZT_S3] = (int32_t)s3; tb[ORC_ZT_S4] = (int32_t)s4; }
                }
            }
            ip += comp;
        }
        if (tr) {
            if (litSize > tr->max_lits - tr->nlits) { rc = ORC_ERR_DST_SMALL; goto done; }
            tb[ORC_ZT_LIT_FIRST] = (int32_t)tr->nlits;
            memcpy(tr->lits + tr->nlits, lit, litSize); tr->nlits += litSize;
        }
    }
    /* ---- sequences section ---- */
    {
        size_t nseq, litPos = 0; unsigned b0;
        if (ip >= iend) goto done;
        b0 = *ip++;
        if (b0 == 0) nseq = 0;
        else if (b0 < 128) nseq = b0;
        else if (b0 < 255) { if (ip >= iend) goto done; nseq = ((size_t)(b0 - 128) << 8) + *ip++; }
        else { if (iend - ip < 2) goto done; nseq = (size_t)ip[0] + ((size_t)ip[1] << 8) + 0x7F00; ip += 2; }
        if (tr) {
            tb[ORC_ZT_NSEQ] = (int32_t)nseq; tb[ORC_ZT_NSEQ_BYTES] = b0 < 128 ? 1 : b0 < 255 ? 2 : 3; tb[ORC_ZT_SEQ_FIRST] = (int32_t)tr->nseqs;
            if (nseq > tr->max_seqs - tr->nseqs) { rc = ORC_ERR_DST_SMALL; goto done; }
        }
        if (nseq) {
            unsigned modes; bbits b; uint32_t sLL, sOF, sML; size_t i;
            if (ip >= iend) goto done;
            modes = *ip++;
            if (tr) tb[ORC_ZT_MODES] = (int32_t)modes;
            if (modes & 3) goto done;
            if (read_seq_table(&z->ll, &z->have_ll, (modes >> 6) & 3, &ip, iend, LL_defnorm, 36, 6, 9, 35)) goto done;
            if (read_seq_table(&z->of, &z->have_of, (modes >> 4) & 3, &ip, iend, OF_defnorm, 29, 5, 8, 31)) goto done;
            if (read_seq_table(&z->ml, &z->have_ml, (modes >> 2) & 3, &ip, iend, ML_defnorm, 53, 6, 9, 52)) goto done;
            if (bb_init(&b, ip, (size_t)(iend - ip))) goto done;
            sLL = (uint32_t)bb_read(&b, z->ll.log); sOF = (uint32_t)bb_read(&b, z->of.log); sML = (uint32_t)bb_read(&b, z->ml.log);
            for (i = 0; i < nseq; i++) {
                unsigned ofc = z->of.sym[sOF], mlc = z->ml.sym[sML], llc = z->ll.sym[sLL];
                uint64_t ofv; size_t ml, ll, offset;
                if (llc > 35 || mlc > 52 || ofc > 31) goto done;
                ofv = ((uint64_t)1 << ofc) + bb_read(&b, (int)ofc);
                ml = ML_base[mlc] + (size_t)bb_read(&b, ML_bits[mlc]);
                ll = LL_base[llc] + (size_t)bb_read(&b, LL_bits[llc]);
                if (ofv > 3) { offset = (size_t)(ofv - 3); z->rep[2] = z->rep[1]; z->rep[1] = z->rep[0]; z->rep[0] = (uint32_t)offset; }
                else {
                    unsigned idx = (unsigned)ofv + (ll == 0 ? 1 : 0);
                    if (idx == 1) offset = z->rep[0];
                    else {
                        offset = idx == 4 ? (size_t)z->rep[0] - 1 : z->rep[idx - 1];
                        if (offset == 0) goto done;
                        if (idx > 2) z->rep[2] = z->rep[1];
                        z->rep[1] = z->rep[0]; z->rep[0] = (uint32_t)offset;
                    }
                }
                if (i + 1 < nseq) {
                    sLL = z->ll.base[sLL] + (uint32_t)bb_read(&b, z->ll.nb[sLL]);
                    sML = z->ml.base[sML] + (uint32_t)bb_read(&b, z->ml.nb[sML]);
                    sOF = z->of.base[sOF] + (uint32_t)bb_read(&b, z->of.nb[sOF]);
                }
                if (b.off < 0) goto done;
                if (tr) { uint32_t* t = tr->seq + 4 * tr->nseqs++; t[0] = (uint32_t)ll; t[1] = (uint32_t)ofv; t[2] = (uint32_t)ml; t[3] = (uint32_t)offset; }
                if (ll > litSize - litPos) goto done;
                if (ll + ml > (size_t)(oend - op)) { rc = ORC_ERR_DST_SMALL; goto done; }
                memcpy(op, lit + litPos, ll); op += ll; litPos += ll;
                if (offset > (size_t)(op - dstBase)) goto done;
                { const uint8_t* m = op - offset; size_t k; for (k = 0; k < ml; k++) op[k] = m[k]; }
                op += ml;
            }
            if (b.off != 0) goto done;
        }
        if (litSize - litPos > (size_t)(oend - op)) { rc = ORC_ERR_DST_SMALL; goto done; }
        memcpy(op, lit + litPos, litSize - litPos); op += litSize - litPos;
    }
    *produced = (size_t)(op - (dstBase + dstPos));
    rc = ORC_OK;
done:
    free(lit);
    return rc;
}

static int parse_frame_header(const uint8_t* src, size_t n, size_t* hdrSize, uint64_t* fcs, int* hasFcs, int* hasChk, uint64_t* window)
{
    unsigned fhd, fcsFlag, single, dictFlag; size_t pos = 5, dl, fl;
    if (n < 6) return ORC_ERR_TRUNCATED;
    if (rd32(src) != 0xFD2FB528u) return ORC_ERR_BAD_MAGIC;
    fhd = src[4]; fcsFlag = fhd >> 6; single = (fhd >> 5) & 1; dictFlag = fhd & 3;
    if (fhd & 0x08) return ORC_ERR_BAD_HEADER;
    *hasChk = (fhd >> 2) & 1;
    *window = 0;
    if (!single) { unsigned wd; if (n < pos + 1) return ORC_ERR_TRUNCATED; wd = src[pos++]; { uint64_t base = (uint64_t)1 << (10 + (wd >> 3)); *window = base + (base >> 3) * (wd & 7); } }
    dl = dictFlag == 0 ? 0 : dictFlag == 1 ? 1 : dictFlag == 2 ? 2 : 4;
    fl = fcsFlag == 0 ? (single ? 1 : 0) : fcsFlag == 1 ? 2 : fcsFlag == 2 ? 4 : 8;
    if (n < pos + dl + fl) return ORC_ERR_TRUNCATED;
    if (dl) { uint32_t id = 0; size_t k; for (k = 0; k < dl; k++) id |= (uint32_t)src[pos + k] << (8 * k); if (id) return ORC_ERR_UNSUPPORTED; }
    pos += dl;
    *hasFcs = fl != 0; *fcs = 0;
    if (fl == 1) *fcs = src[pos]; else if (fl == 2) *fcs = (uint64_t)(src[pos] | (src[pos + 1] << 8)) + 256; else if (fl == 4) *fcs = rd32(src + pos); else if (fl == 8) *fcs = rd64(src + pos);
    pos += fl;
    if (single) *window = *fcs;
    *hdrSize = pos;
    return ORC_OK;
}

uint64_t orc_zstd_content_size(const uint8_t* src, size_t srcSize)
{
    size_t hs; uint64_t fcs, win; int hf, hc;
    if (parse_frame_header(src, srcSize, &hs, &fcs, &hf, &hc, &win) != ORC_OK || !hf) return (uint64_t)-1;
    return fcs;
}

static int decode_frame(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t* outSize, size_t* consumed, orc_zstd_trace_t* tr)
{
    size_t hs, pos, total = 0; uint64_t fcs, win; int hasFcs, hasChk, rc, last = 0;
    zctx* z; int32_t* tb = NULL; uint8_t* tw = NULL;
    rc = parse_frame_header(src, srcSize, &hs, &fcs, &hasFcs, &hasChk, &win);
    if (rc != ORC_OK) return rc;
    z = (zctx*)calloc(1, sizeof(zctx));
    z->rep[0] = 1; z->rep[1] = 4; z->rep[2] = 8;
    pos = hs;
    while (!last) {
        uint32_t bh; unsigned type; size_t bs;
        if (srcSize - pos < 3) { rc = ORC_ERR_TRUNCATED; goto out; }
        bh = src[pos] | (src[pos + 1] << 8) | ((uint32_t)src[pos + 2] << 16); pos += 3;
        last = bh & 1; type = (bh >> 1) & 3; bs = bh >> 3;
        if (type == 3 || bs > 128 * 1024) { rc = ORC_ERR_CORRUPT; goto out; }
        if (tr) {
            int k;
            if (tr->nblocks >= tr->max_blocks) { rc = ORC_ERR_DST_SMALL; goto out; }
            tb = tr->blk + tr->nblocks * ORC_ZT_NF; tw = tr->weights + tr->nblocks * 256;
            for (k = 0; k < ORC_ZT_NF; k++) tb[k] = -1;
            memset(tw, 0, 256);
            tb[ORC_ZT_TYPE] = (int32_t)type; tb[ORC_ZT_LAST] = last; tb[ORC_ZT_BSIZE] = (int32_t)bs;
        }
        if (type == 0) {
            if (srcSize - pos < bs) { rc = ORC_ERR_TRUNCATED; goto out; }
            if (bs > dstCap - total) { rc = ORC_ERR_DST_SMALL; goto out; }
            memcpy(dst + total, src + pos, bs); total += bs; pos += bs;
            if (tr) tb[ORC_ZT_REGEN] = (int32_t)bs;
        } else if (type == 1) {
            if (srcSize - pos < 1) { rc = ORC_ERR_TRUNCATED; goto out; }
            if (bs > dstCap - total) { rc = ORC_ERR_DST_SMALL; goto out; }
            memset(dst + total, src[pos], bs); total += bs; pos += 1;
            if (tr) tb[ORC_ZT_REGEN] = (int32_t)bs;
        } else {
            size_t produced = 0;
            if (srcSize - pos < bs) { rc = ORC_ERR_TRUNCATED; goto out; }
            rc = decode_block(z, src + pos, bs, dst, total, dstCap, &produced, tr, tb, tw);
            if (rc != ORC_OK) goto out;
            if (produced > 128 * 1024) { rc = ORC_ERR_CORRUPT; goto out; }
            total += produced; pos += bs;
            if (tr) tb[ORC_ZT_REGEN] = (int32_t)produced;
        }
        if (tr) tr->nblocks++;
    }
    if (hasChk) {
        if (srcSize - pos < 4) { rc = ORC_ERR_TRUNCATED; goto out; }
        if ((uint32_t)xxh64(dst, total, 0) != rd32(src + pos)) { rc = ORC_ERR_CONTENT_CHECKSUM; goto out; }
        pos += 4;
    }
    if (hasFcs && fcs != total) { rc = ORC_ERR_CONTENT_SIZE; goto out; }
    if (outSize) *outSize = total;
    if (consumed) *consumed = pos;
    rc = ORC_OK;
out:
    free(z);
    return rc;
}

int orc_zstd_decode(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t* outSize, size_t* consumed)
{
    return decode_frame(src, srcSize, dst, dstCap, outSize, consumed, NULL);
}

int orc_zstd_trace(const uint8_t* src, size_t srcSize, uint8_t* dst, size_t dstCap, size_t* outSize, size_t* consumed, orc_zstd_trace_t* tr)
{
    if (!tr) return ORC_ERR_UNSUPPORTED;
    tr->nblocks = tr->nseqs = tr->nlits = 0;
    return decode_frame(src, srcSize, dst, dstCap, outSize, consumed, tr);
}
