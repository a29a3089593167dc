/* zstd_enc_twin.c — TEST INFRASTRUCTURE ONLY: the serial CPU twin of the GPU zstd encoder's entropy stage
 * (z_encode_block in zstdmt_b200/csrc/zstd_entropy.cuh), byte for byte.
 *
 * Given one block's sequences, literals and content, orc_zstd_block_b200 writes the block (3-byte header included) that
 * the kernel writes.  It shares no code with the kernel: every rule is restated here from RFC 8878 and from the rules
 * DESIGN §7 gives the encoder:
 *   - literals: RLE iff one distinct byte; Huffman from 64 literals and 2 symbols, else raw; a Huffman section goes raw
 *     again when its tree has no description, when est = ceil(bits / 8) + 4 + tree bytes + 6 >= nlit, or when
 *     est + 64 exceeds the 12 KiB bit buffer;
 *   - the Huffman code: present symbols in ascending (count, symbol) order, a two-queue tree (the leaf taken on ties),
 *     an 11-bit limit; canonical codes in the decoder's table order; direct 4-bit weights iff maxsym <= 128, else
 *     FSE-coded weights (table log 6, the encoder's own normalisation); four streams of ceil(nlit / 4) literals;
 *   - sequences: predefined LL / OF / ML tables, explicit offsets (Offset_Value = offset + 3), per sequence the OF, ML,
 *     LL state bits and then the LL, ML, OF extra bits, the final states flushed ML, OF, LL;
 *   - the block goes raw when it is not smaller than its content, when its sequence bits overflow the 12 KiB bit buffer,
 *     or when it has 0x7F00 sequences or more.
 * FSE encoding is stated from the decoding table (RFC 8878 §4.1.1): encoding symbol s from state X moves to the cell X'
 * of s whose range [baseline, baseline + 2^nbBits) holds X and writes X - baseline in nbBits bits; the first symbol
 * encoded takes the lowest cell of its symbol and writes nothing.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

#define T_BITWORDS   3072u           /* the kernel's bit buffer, in 32-bit words */
#define T_HUF_MAXBITS 11
#define T_MAXSEQ     4352u
#define T_MAXLIT     (64u * 1024u + 256u)
#define T_OVER       0xFFFFFFFFu     /* fse_weights: a buffer of the twin overflowed (a broken invariant, not "no form") */

/* ------------------------------------------------------------------ predefined distributions (RFC 8878 §3.1.1.3.2.2) */
static const int16_t LL_NORM[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1,
                                    -1, -1, -1, -1};
static const int16_t ML_NORM[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                    1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
static const int16_t OF_NORM[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
/* literal-length and match-length codes (RFC 8878 §3.1.1.3.2.1.1) */
static const uint32_t LL_BASE[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64,
                                     128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
static const uint8_t LL_BITS[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11,
                                    12, 13, 14, 15, 16};
static const uint32_t ML_BASE[53] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27,
                                     28, 29, 30, 31, 32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027,
                                     2051, 4099, 8195, 16387, 32771, 65539};
static const uint8_t ML_BITS[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                    1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

static int code_of(const uint32_t* base, int n, uint32_t v)        /* the largest code whose baseline is <= v */
{
    int c = 0;
    while (c + 1 < n && base[c + 1] <= v) c++;
    return c;
}

static int highbit(uint32_t v) { int h = 0; while (v >>= 1) h++; return h; }

/* ------------------------------------------------------------------ FSE decoding tables and encoding from them */
typedef struct {
    int log, nsym;
    uint8_t sym[64], nb[64];
    uint16_t base[64];
    int16_t first[64];               /* lowest cell of each symbol, -1 when absent */
} fse_t;

static void fse_build(fse_t* T, const int16_t* norm, int nsym, int log)
{
    const int size = 1 << log, step = (size >> 1) + (size >> 3) + 3;
    int high = size - 1, pos = 0, next[64];
    T->log = log; T->nsym = nsym;
    for (int s = 0; s < nsym; s++)                                 /* "less than 1" symbols: one cell each, from the top */
        if (norm[s] == -1) { T->sym[high--] = (uint8_t)s; next[s] = 1; }
    for (int s = 0; s < nsym; s++) {
        if (norm[s] <= 0) continue;
        next[s] = norm[s];
        for (int i = 0; i < norm[s]; i++) { T->sym[pos] = (uint8_t)s; do pos = (pos + step) & (size - 1); while (pos > high); }
    }
    for (int s = 0; s < nsym; s++) T->first[s] = -1;
    for (int u = 0; u < size; u++) {                               /* cells in ascending order take the states n .. 2n-1 */
        const int s = T->sym[u], x = next[s]++;
        T->nb[u] = (uint8_t)(log - highbit((uint32_t)x));
        T->base[u] = (uint16_t)((x << T->nb[u]) - size);
        if (T->first[s] < 0) T->first[s] = (int16_t)u;
    }
}

/* encode symbol s leaving cell x: returns the new cell, the bits in *v / *n */
static int fse_enc(const fse_t* T, int x, int s, uint32_t* v, uint32_t* n)
{
    for (int u = 0; u < (1 << T->log); u++)
        if (T->sym[u] == s && x >= T->base[u] && x < T->base[u] + (1 << T->nb[u])) { *v = (uint32_t)(x - T->base[u]); *n = T->nb[u]; return u; }
    return -1;
}

static fse_t g_ll, g_of, g_ml;
static int g_ready;
static void tables(void)
{
    if (g_ready) return;
    fse_build(&g_ll, LL_NORM, 36, 6); fse_build(&g_of, OF_NORM, 29, 5); fse_build(&g_ml, ML_NORM, 53, 6);
    g_ready = 1;
}

int orc_zenc_fse_table(int stream, uint8_t* sym, uint8_t* nb, uint16_t* base)
{
    tables();
    const fse_t* T = stream == 0 ? &g_ll : stream == 1 ? &g_of : &g_ml;
    const int size = 1 << T->log;
    memcpy(sym, T->sym, size); memcpy(nb, T->nb, size);
    for (int u = 0; u < size; u++) base[u] = T->base[u];
    return T->log;
}

/* ------------------------------------------------------------------ little-endian forward bit writer */
typedef struct { uint8_t* p; size_t cap; uint64_t pos; int over; } bw_t;
static void bw_put(bw_t* w, uint32_t v, uint32_t n)
{
    for (uint32_t i = 0; i < n; i++, w->pos++) {
        if ((w->pos >> 3) >= w->cap) { w->over = 1; continue; }
        if ((v >> i) & 1) w->p[w->pos >> 3] |= (uint8_t)(1u << (w->pos & 7));
    }
}

/* ------------------------------------------------------------------ Huffman code lengths */
static uint32_t huf_lengths(const uint32_t* hist, uint8_t* len)
{
    uint32_t order[256], cnt[512], par[512], depth[512], n = 0;
    for (uint32_t s = 0; s < 256; s++) len[s] = 0;
    for (uint32_t s = 0; s < 256; s++) if (hist[s]) order[n++] = s;
    for (uint32_t i = 1; i < n; i++) {                            /* ascending (count, symbol): insertion sort */
        const uint32_t x = order[i]; uint32_t j = i;
        while (j > 0 && hist[order[j - 1]] > hist[x]) { order[j] = order[j - 1]; j--; }
        order[j] = x;
    }
    for (uint32_t i = 0; i < n; i++) cnt[i] = hist[order[i]];
    uint32_t li = 0, ii = n, ni = n;
    for (uint32_t k = 0; k + 1 < n; k++) {
        uint32_t pick[2];
        for (int j = 0; j < 2; j++) pick[j] = (li < n && (ii >= ni || cnt[li] <= cnt[ii])) ? li++ : ii++;
        cnt[ni] = cnt[pick[0]] + cnt[pick[1]]; par[pick[0]] = par[pick[1]] = ni; ni++;
    }
    depth[ni - 1] = 0;
    for (int v = (int)ni - 2; v >= 0; v--) depth[v] = depth[par[v]] + 1;
    uint32_t maxl = 0;
    for (uint32_t i = 0; i < n; i++) if (depth[i] > maxl) maxl = depth[i];
    if (maxl > T_HUF_MAXBITS) {
        int excess = -(1 << T_HUF_MAXBITS);
        for (uint32_t i = 0; i < n; i++) { if (depth[i] > T_HUF_MAXBITS) depth[i] = T_HUF_MAXBITS; excess += 1 << (T_HUF_MAXBITS - depth[i]); }
        while (excess > 0) {                                       /* lengthen the rarest short leaf whose step fits, else the rarest */
            int best = -1;
            for (uint32_t i = 0; i < n; i++)
                if (depth[i] < T_HUF_MAXBITS) {
                    if (best < 0) best = (int)i;
                    if ((1 << (T_HUF_MAXBITS - 1 - depth[i])) <= excess) { best = (int)i; break; }
                }
            if (best < 0) break;
            excess -= 1 << (T_HUF_MAXBITS - 1 - depth[best]); depth[best]++;
        }
        for (uint32_t i = 0; i < n && excess < 0; i++) if (depth[i] == T_HUF_MAXBITS) { depth[i]--; excess++; }
        maxl = T_HUF_MAXBITS;
    }
    for (uint32_t i = 0; i < n; i++) len[order[i]] = (uint8_t)depth[i];
    return maxl;
}

/* ------------------------------------------------------------------ FSE-coded Huffman weights (RFC 8878 §4.2.1.2) */
/* Returns the description's length (header byte included) written to out, 0 when the encoder has no such form, or
 * T_OVER when a bit buffer of the twin overflowed or a state has no cell (neither can happen while the rules hold). */
static uint32_t fse_weights(const uint8_t* len, uint32_t nw, uint32_t maxbits, uint8_t* out)
{
    enum { LOG = 6, SIZE = 64 };
    uint8_t wt[256]; uint32_t count[13] = {0}; int norm[13] = {0};
    if (nw < 2) return 0;
    uint32_t maxw = 0;
    for (uint32_t s = 0; s < nw; s++) { wt[s] = (uint8_t)(len[s] ? maxbits + 1 - len[s] : 0); count[wt[s]]++; if (wt[s] > maxw) maxw = wt[s]; }
    uint32_t maxc = 0;
    for (uint32_t i = 0; i <= maxw; i++) if (count[i] > maxc) maxc = count[i];
    if (maxc == nw || maxc <= 1) return 0;
    /* normalisation: floor(count * 64 / nw), at least 1 when present; a shortfall goes to the first most frequent value,
       an excess is taken from the largest counts (first among equals), never below 1 */
    int sum = 0, big = 0;
    for (uint32_t i = 0; i <= maxw; i++) {
        if (count[i]) { norm[i] = (int)(count[i] * SIZE / nw); if (!norm[i]) norm[i] = 1; }
        sum += norm[i];
        if (count[i] > count[big]) big = (int)i;
    }
    if (sum < SIZE) norm[big] += SIZE - sum;
    while (sum > SIZE) {
        int b = -1;
        for (uint32_t i = 0; i <= maxw; i++) if (norm[i] > 1 && (b < 0 || norm[i] > norm[b])) b = (int)i;
        if (b < 0) return 0;
        const int take = norm[b] - 1 < sum - SIZE ? norm[b] - 1 : sum - SIZE;
        norm[b] -= take; sum -= take;
    }
    /* table description: accuracy log - 5, then each value's probability + 1 in nbBits or nbBits - 1 bits, with 2-bit
       repeat flags after a zero probability */
    uint8_t buf[160]; memset(buf, 0, sizeof buf);
    bw_t w = {buf, sizeof buf, 0, 0};
    bw_put(&w, LOG - 5, 4);
    int remaining = SIZE + 1, threshold = SIZE, nbits = LOG + 1, prev0 = 0;
    uint32_t sym = 0;
    while (sym <= maxw && remaining > 1) {
        if (prev0) {
            uint32_t z = 0;
            while (sym + z <= maxw && norm[sym + z] == 0) z++;
            if (sym + z > maxw) break;
            for (; z >= 3; z -= 3) bw_put(&w, 3, 2);
            bw_put(&w, z, 2);
            while (norm[sym] == 0) sym++;
        }
        const int p = norm[sym++], mx = 2 * threshold - 1 - remaining;
        remaining -= p;
        int v = p + 1;
        if (v >= threshold) v += mx;
        bw_put(&w, (uint32_t)v, (uint32_t)(v < mx ? nbits - 1 : nbits));
        prev0 = p == 0;
        while (remaining < threshold) { nbits--; threshold >>= 1; }
    }
    if (w.over) return T_OVER;
    if (remaining != 1) return 0;
    const uint32_t hdr = (uint32_t)((w.pos + 7) >> 3);
    if (hdr >= 100) return 0;
    /* the weights, last first, on two interleaved states (state 1 decodes the even positions) */
    fse_t T; int16_t nn[13];
    for (uint32_t i = 0; i <= maxw; i++) nn[i] = (int16_t)norm[i];
    fse_build(&T, nn, (int)maxw + 1, LOG);
    uint8_t bits[160]; memset(bits, 0, sizeof bits);
    const uint32_t bcap = (127 - hdr) * 8;
    bw_t b = {bits, sizeof bits, 0, 0};
    int over = 0, s1, s2, ip = (int)nw;
    uint32_t v = 0, n = 0;
#define ENC(st, sy) do { st = fse_enc(&T, st, sy, &v, &n); if (st < 0) return T_OVER; if (b.pos + n > bcap) over = 1; else bw_put(&b, v, n); } while (0)
    if (nw & 1) { s1 = T.first[wt[--ip]]; s2 = T.first[wt[--ip]]; ENC(s1, wt[--ip]); }
    else { s2 = T.first[wt[--ip]]; s1 = T.first[wt[--ip]]; }
    while (ip > 0) { ENC(s2, wt[--ip]); ENC(s1, wt[--ip]); }
#undef ENC
    if (b.pos + LOG > bcap) over = 1; else bw_put(&b, (uint32_t)s2, LOG);
    if (b.pos + LOG > bcap) over = 1; else bw_put(&b, (uint32_t)s1, LOG);
    if (b.pos + 1 > bcap) over = 1; else bw_put(&b, 1, 1);
    if (b.over) return T_OVER;
    const uint32_t total = hdr + (uint32_t)((b.pos + 7) >> 3);
    if (over || total >= 128) return 0;
    out[0] = (uint8_t)total;
    memcpy(out + 1, buf, hdr);
    memcpy(out + 1 + hdr, bits, total - hdr);
    return 1 + total;
}

/* ------------------------------------------------------------------ one block */
static void put_le(uint8_t* p, uint64_t v, int n) { for (int i = 0; i < n; i++) p[i] = (uint8_t)(v >> (8 * i)); }

long orc_zstd_block_b200(const uint32_t* rows, size_t nseq, const uint8_t* lits, size_t nlit, const uint8_t* raw, size_t regen,
                         int last, uint8_t* dst, size_t cap, orc_zenc_trace_t* tr)
{
    tables();
    if (nseq > T_MAXSEQ || nlit > T_MAXLIT || regen >= (1u << 21)) return ORC_ERR_UNSUPPORTED;
    if (cap < 3 + regen) return ORC_ERR_DST_SMALL;
    orc_zenc_trace_t dummy;
    if (!tr) { memset(&dummy, 0, sizeof dummy); tr = &dummy; }
    tr->nseq = (uint32_t)nseq; tr->nlit = (uint32_t)nlit; tr->regen = (uint32_t)regen;
    tr->lit_reason = tr->raw_reason = 0; tr->est = tr->tot_bits = 0;
    tr->huf_bits[0] = tr->huf_bits[1] = tr->huf_bits[2] = tr->huf_bits[3] = 0;
    tr->tree_bytes = tr->wdesc_len = tr->maxbits = 0;
    memset(tr->hlen, 0, sizeof tr->hlen); memset(tr->hcode, 0, sizeof tr->hcode);

    uint8_t* const sec = dst + 3;                                  /* the literals section, then the sequences section */
    /* -------------------- literals */
    uint32_t hist[256] = {0}, nused = 0, maxsym = 0, maxcnt = 0;
    for (size_t i = 0; i < nlit; i++) hist[lits[i]]++;
    for (uint32_t s = 0; s < 256; s++) if (hist[s]) { nused++; maxsym = s; if (hist[s] > maxcnt) maxcnt = hist[s]; }
    int lmode = 0;                                                 /* 0 raw, 1 RLE, 2 Huffman */
    if (nlit && maxcnt == nlit) lmode = 1;
    else if (nlit >= 64 && nused >= 2) lmode = 2;
    else tr->lit_reason = nlit ? ORC_ZENC_LIT_FEW : 0;
    uint8_t* len = tr->hlen; uint16_t* code = tr->hcode;
    uint8_t wdesc[136]; uint32_t wlen = 0, maxbits = 0, tree_bytes = 0;
    if (lmode == 2) {
        maxbits = huf_lengths(hist, len);
        uint32_t wcnt[16] = {0}, wbase[16] = {0}, acc = 0;
        for (uint32_t s = 0; s < 256; s++) if (len[s]) wcnt[maxbits + 1 - len[s]]++;
        for (uint32_t w = 1; w <= maxbits; w++) { wbase[w] = acc; acc += wcnt[w] << (w - 1); }
        for (uint32_t s = 0; s < 256; s++) {                       /* decoder's table order: ascending weight, then symbol */
            if (!len[s]) continue;
            const uint32_t w = maxbits + 1 - len[s];
            code[s] = (uint16_t)(wbase[w] >> (w - 1)); wbase[w] += 1u << (w - 1);
            tr->tot_bits += hist[s] * len[s];
        }
        int noform = 0;
        if (maxsym <= 128) tree_bytes = 1 + (maxsym + 1) / 2;
        else {
            wlen = fse_weights(len, maxsym, maxbits, wdesc);
            if (wlen == T_OVER) return ORC_ERR_CORRUPT;
            tree_bytes = wlen; noform = wlen == 0;
        }
        tr->maxbits = maxbits; tr->tree_bytes = tree_bytes; tr->wdesc_len = wlen;
        tr->est = (tr->tot_bits + 7) / 8 + 4 + tree_bytes + 6;
        if (noform) tr->lit_reason |= ORC_ZENC_LIT_NOFORM;
        if (tr->est >= nlit) tr->lit_reason |= ORC_ZENC_LIT_EST;
        if (tr->est + 64 > T_BITWORDS * 4) tr->lit_reason |= ORC_ZENC_LIT_BITBUF;
        if (tr->lit_reason) lmode = 0;
    }
    uint32_t lit_hdr, lit_body;
    if (lmode == 2) {
        const size_t per = (nlit + 3) / 4;
        uint8_t* streams[4]; uint32_t ssize[4]; size_t payload = 0;
        uint8_t sbuf[4][T_BITWORDS * 4 + 8];
        for (int k = 0; k < 4; k++) {
            const size_t a = k * per < nlit ? k * per : nlit, e = (k + 1) * per < nlit ? (k + 1) * per : nlit;
            memset(sbuf[k], 0, sizeof sbuf[k]);
            bw_t w = {sbuf[k], sizeof sbuf[k], 0, 0};
            for (size_t i = e; i > a; i--) bw_put(&w, code[lits[i - 1]], len[lits[i - 1]]);   /* the last literal first */
            tr->huf_bits[k] = (uint32_t)w.pos;
            bw_put(&w, 1, 1);
            if (w.over) return ORC_ERR_CORRUPT;
            ssize[k] = (uint32_t)((w.pos + 7) >> 3); streams[k] = sbuf[k]; payload += ssize[k];
        }
        lit_body = tree_bytes + 6 + (uint32_t)payload;
        lit_hdr = (nlit < 1024 && lit_body < 1024) ? 3 : (nlit < 16384 && lit_body < 16384) ? 4 : 5;
        if (cap < 3 + lit_hdr + lit_body) return ORC_ERR_DST_SMALL;
        const uint32_t fmt = lit_hdr - 2, nb = lit_hdr == 3 ? 10 : lit_hdr == 4 ? 14 : 18;
        put_le(sec, 2u | (fmt << 2) | ((uint64_t)nlit << 4) | ((uint64_t)lit_body << (4 + nb)), (int)lit_hdr);
        uint8_t* q = sec + lit_hdr;
        if (wlen) { memcpy(q, wdesc, wlen); q += wlen; }
        else {
            *q++ = (uint8_t)(127 + maxsym);
            for (uint32_t s = 0; s < maxsym; s += 2) {
                const uint32_t w0 = len[s] ? maxbits + 1 - len[s] : 0, w1 = s + 1 < maxsym && len[s + 1] ? maxbits + 1 - len[s + 1] : 0;
                *q++ = (uint8_t)(w0 << 4 | w1);
            }
        }
        for (int k = 0; k < 3; k++) put_le(q + 2 * k, ssize[k], 2);
        q += 6;
        for (int k = 0; k < 4; k++) { memcpy(q, streams[k], ssize[k]); q += ssize[k]; }
    } else {
        lit_body = lmode == 1 ? 1 : (uint32_t)nlit;
        lit_hdr = nlit < 32 ? 1 : nlit < 4096 ? 2 : 3;
        if (cap < 3 + lit_hdr + lit_body) return ORC_ERR_DST_SMALL;
        const uint32_t sf = lit_hdr == 1 ? 0 : lit_hdr == 2 ? 1 : 3;
        put_le(sec, (uint32_t)lmode | (sf << 2) | ((uint64_t)nlit << (lit_hdr == 1 ? 3 : 4)), (int)lit_hdr);
        if (lmode == 1) sec[lit_hdr] = lits[0];
        else if (nlit) memcpy(sec + lit_hdr, lits, nlit);
    }
    tr->lit_mode = (uint32_t)lmode; tr->lit_size = lit_hdr + lit_body; tr->maxsym = maxsym; tr->nused = nused;

    /* -------------------- sequences: the three state chains, last sequence first */
    const fse_t* F[3] = {&g_ll, &g_of, &g_ml};
    int st[3] = {0, 0, 0};
    const size_t sqcap = (nseq + 1) * 16;                        /* a sequence takes at most 17 state and 54 extra bits */
    uint8_t* sq = calloc(sqcap, 1);
    if (!sq) return ORC_ERR_DST_SMALL;
    bw_t w = {sq, sqcap, 0, 0};
    for (size_t t = 0; t < nseq; t++) {
        const uint32_t* r = rows + 3 * (nseq - 1 - t);
        const uint32_t ll = r[0], ofv = r[1] + 3, ml = r[2];
        const int c[3] = {code_of(LL_BASE, 36, ll), highbit(ofv), code_of(ML_BASE, 53, ml)};
        uint32_t v[3] = {0, 0, 0}, n[3] = {0, 0, 0};
        for (int k = 0; k < 3; k++) {
            if (c[k] >= F[k]->nsym) { free(sq); return ORC_ERR_UNSUPPORTED; }
            st[k] = t == 0 ? F[k]->first[c[k]] : fse_enc(F[k], st[k], c[k], &v[k], &n[k]);
            if (st[k] < 0) { free(sq); return ORC_ERR_CORRUPT; }
            if (tr->code[k]) tr->code[k][t] = (uint8_t)c[k];
            if (tr->state[k]) tr->state[k][t] = (uint16_t)((1 << F[k]->log) + st[k]);
        }
        bw_put(&w, v[1], n[1]); bw_put(&w, v[2], n[2]); bw_put(&w, v[0], n[0]);
        bw_put(&w, ll - LL_BASE[c[0]], LL_BITS[c[0]]);
        bw_put(&w, ml - ML_BASE[c[2]], ML_BITS[c[2]]);
        bw_put(&w, ofv - (1u << c[1]), (uint32_t)c[1]);
    }
#define FAIL(e) do { free(sq); return e; } while (0)
    if (nseq) {
        bw_put(&w, (uint32_t)st[2], 6); bw_put(&w, (uint32_t)st[1], 5); bw_put(&w, (uint32_t)st[0], 6);
        for (int k = 0; k < 3; k++) tr->fin[k] = (uint32_t)((1 << F[k]->log) + st[k]);
    }
    tr->seq_bits = (uint32_t)w.pos;
    const uint32_t seq_hdr = nseq == 0 ? 1 : nseq < 128 ? 2 : 3;
    const uint32_t seq_body = nseq ? tr->seq_bits / 8 + 1 : 0;
    if (nseq) bw_put(&w, 1, 1);
    if (w.over) FAIL(ORC_ERR_CORRUPT);
    tr->seq_body = seq_body;
    const uint64_t bsize = (uint64_t)tr->lit_size + seq_hdr + seq_body;
    tr->bsize = (uint32_t)bsize;
    if (bsize >= regen) tr->raw_reason |= ORC_ZENC_RAW_SIZE;
    if (seq_body + 8 > T_BITWORDS * 4) tr->raw_reason |= ORC_ZENC_RAW_BITBUF;
    if (nseq >= 0x7F00) tr->raw_reason |= ORC_ZENC_RAW_NSEQ;

    if (tr->raw_reason) {
        put_le(dst, (uint32_t)(regen << 3) | (last ? 1u : 0u), 3);
        memcpy(dst + 3, raw, regen);
        free(sq);
        return (long)(3 + regen);
    }
    put_le(dst, (uint32_t)(bsize << 3) | (2u << 1) | (last ? 1u : 0u), 3);
    uint8_t* s = sec + tr->lit_size;
    if (nseq == 0) s[0] = 0;
    else if (nseq < 128) { s[0] = (uint8_t)nseq; s[1] = 0; }
    else { s[0] = (uint8_t)((nseq >> 8) + 128); s[1] = (uint8_t)nseq; s[2] = 0; }
    if (cap < 3 + bsize) FAIL(ORC_ERR_DST_SMALL);
    memcpy(s + seq_hdr, sq, seq_body);
    free(sq);
    return (long)(3 + bsize);
}
