/* datagen.c — deterministic synthetic inputs for parity tests and bench.py (SURVEY.md §8d).
 *
 * The reference ships no corpus (its only test compresses /dev/urandom,
 * programs/Makefile:252-260) and Silesia is not part of this repository, so
 * the workloads BASELINE.json names are generated:
 *   ZMT_GEN_ZEROS  0x00 bytes                                   (config 1)
 *   ZMT_GEN_TEXT   Zipf(s=1) words from a 4096-word vocabulary  (config 4)
 *   ZMT_GEN_MIX    "Silesia-mix": class = chunk_index mod 8     (configs 2, 3, 5)
 *                  0,1 text | 2 XML/log records | 3 16-bit random walk | 4 32-byte structs |
 *                  5 opcode soup with back-references | 6 uniform random | 7 long runs
 * Every chunk depends only on (kind, chunk_index, chunk_size): seed =
 * 0x5117E51A ^ chunk_index, so CPU and GPU legs, any rank and any thread count
 * produce identical bytes.  Integer arithmetic only (no libm) for bit-stable output.
 */
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ZMT_GEN_ZEROS 0
#define ZMT_GEN_TEXT  1
#define ZMT_GEN_MIX   2
#define ZMT_GEN_RANDOM 3

typedef struct { uint64_t s; } rng_t;
static inline uint64_t rng_next(rng_t* r)
{   /* splitmix64 */
    uint64_t z = (r->s += 0x9E3779B97F4A7C15ULL);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
static inline uint32_t rng_u32(rng_t* r) { return (uint32_t)(rng_next(r) >> 32); }
static inline uint32_t rng_below(rng_t* r, uint32_t n) { return (uint32_t)(((uint64_t)rng_u32(r) * n) >> 32); }

/* ---- vocabulary + Zipf table (built once, deterministic) */
#define VOCAB 4096
static char     g_words[VOCAB][12];
static uint8_t  g_wlen[VOCAB];
static uint32_t g_zipf[VOCAB];            /* cumulative thresholds scaled to 2^32 */
static uint8_t  g_optab[256];             /* weighted opcode table */
static pthread_once_t g_once = PTHREAD_ONCE_INIT;

static void init_tables(void)
{
    rng_t r = { 1234 };
    double h = 0.0, acc = 0.0;
    int i, j;
    for (i = 0; i < VOCAB; i++) {
        int len = 2 + (int)rng_below(&r, 9);
        g_wlen[i] = (uint8_t)len;
        for (j = 0; j < len; j++) g_words[i][j] = (char)('a' + rng_below(&r, 26));
    }
    for (i = 1; i <= VOCAB; i++) h += 1.0 / i;
    for (i = 0; i < VOCAB; i++) {
        acc += 1.0 / (i + 1);
        double t = acc / h * 4294967296.0;
        g_zipf[i] = t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
    }
    g_zipf[VOCAB - 1] = 0xFFFFFFFFu;
    /* opcode soup: a few very common bytes, a long tail */
    for (i = 0; i < 256; i++) {
        uint32_t u = rng_below(&r, 100);
        static const uint8_t common[8] = { 0x48, 0x8B, 0x89, 0x00, 0xE8, 0xFF, 0x0F, 0x24 };
        g_optab[i] = u < 60 ? common[rng_below(&r, 8)] : (uint8_t)rng_below(&r, 256);
    }
}

static size_t gen_text(rng_t* r, uint8_t* p, size_t n)
{
    size_t o = 0; uint32_t nw = 0;
    while (o < n) {
        uint32_t u = rng_u32(r), lo = 0, hi = VOCAB - 1;
        while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (g_zipf[mid] < u) lo = mid + 1; else hi = mid; }
        {
            size_t l = g_wlen[lo], k;
            for (k = 0; k < l && o < n; k++) p[o++] = (uint8_t)g_words[lo][k];
        }
        if (++nw % 2000 == 0) { if (o < n) p[o++] = '.'; if (o < n) p[o++] = '\n'; }
        else if (o < n) p[o++] = ' ';
    }
    return o;
}

static size_t put_dec(uint8_t* p, size_t o, size_t n, uint32_t v)
{
    char tmp[12]; int k = 0;
    do { tmp[k++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (k && o < n) p[o++] = (uint8_t)tmp[--k];
    return o;
}
static size_t put_str(uint8_t* p, size_t o, size_t n, const char* s) { while (*s && o < n) p[o++] = (uint8_t)*s++; return o; }

static void gen_xml(rng_t* r, uint8_t* p, size_t n)
{
    static const char* lvl[4] = { "INFO", "WARN", "DEBUG", "ERROR" };
    static const char* svc[6] = { "auth", "storage", "gateway", "scheduler", "billing", "search" };
    size_t o = 0; uint32_t ts = 1700000000u + rng_below(r, 1000000), id = rng_below(r, 100000);
    while (o < n) {
        ts += rng_below(r, 3); id += 1 + rng_below(r, 4);
        o = put_str(p, o, n, "<record id=\""); o = put_dec(p, o, n, id);
        o = put_str(p, o, n, "\" ts=\""); o = put_dec(p, o, n, ts);
        o = put_str(p, o, n, "\"><level>"); o = put_str(p, o, n, lvl[rng_below(r, 4)]);
        o = put_str(p, o, n, "</level><service>"); o = put_str(p, o, n, svc[rng_below(r, 6)]);
        o = put_str(p, o, n, "</service><latency_us>"); o = put_dec(p, o, n, 100 + rng_below(r, 90000));
        o = put_str(p, o, n, "</latency_us><bytes>"); o = put_dec(p, o, n, rng_below(r, 1u << 20));
        o = put_str(p, o, n, "</bytes></record>\n");
    }
}

static void gen_walk16(rng_t* r, uint8_t* p, size_t n)
{
    size_t o = 0; int32_t v = (int32_t)rng_below(r, 65536);
    while (o + 1 < n) {
        v += (int32_t)rng_below(r, 33) - 16;
        if (v < 0) v = 0; if (v > 65535) v = 65535;
        p[o++] = (uint8_t)v; p[o++] = (uint8_t)(v >> 8);
    }
    if (o < n) p[o] = 0;
}

static void gen_structs(rng_t* r, uint8_t* p, size_t n)
{
    size_t o = 0; uint32_t a = rng_u32(r), b = rng_below(r, 1000), c = 0; uint64_t t = 0x0001000000000000ULL + rng_u32(r);
    while (o < n) {
        uint8_t rec[32]; int k;
        a += rng_below(r, 8) == 0 ? 1 : 0; b += rng_below(r, 3); c++; t += 1000 + rng_below(r, 50);
        memcpy(rec, &a, 4); memcpy(rec + 4, &b, 4); memcpy(rec + 8, &c, 4); memcpy(rec + 12, &t, 8);
        for (k = 20; k < 28; k++) rec[k] = (uint8_t)(k * 7);
        { uint32_t x = rng_u32(r); memcpy(rec + 28, &x, 4); }
        for (k = 0; k < 32 && o < n; k++) p[o++] = rec[k];
    }
}

static void gen_opcodes(rng_t* r, uint8_t* p, size_t n)
{
    size_t o = 0;
    while (o < n) {
        if (o > 64 && rng_below(r, 5) == 0) {          /* 20 %: back-reference of 4..64 bytes within 32 KiB */
            size_t len = 4 + rng_below(r, 61), win = o < 32768 ? o : 32768, dist = 1 + rng_below(r, (uint32_t)win), k;
            for (k = 0; k < len && o < n; k++, o++) p[o] = p[o - dist];
        } else {
            size_t len = 1 + rng_below(r, 12), k;
            for (k = 0; k < len && o < n; k++) p[o++] = g_optab[rng_below(r, 256)];
        }
    }
}

static void gen_random(rng_t* r, uint8_t* p, size_t n)
{
    size_t o = 0;
    while (o + 8 <= n) { uint64_t x = rng_next(r); memcpy(p + o, &x, 8); o += 8; }
    while (o < n) p[o++] = (uint8_t)rng_u32(r);
}

static void gen_runs(rng_t* r, uint8_t* p, size_t n)
{
    size_t o = 0;
    while (o < n) {
        uint8_t v = (uint8_t)rng_u32(r);
        size_t len = 1;
        while (rng_below(r, 512) != 0 && len < 8192) len += 1 + rng_below(r, 3);    /* ~geometric, mean in the hundreds */
        if (len > n - o) len = n - o;
        memset(p + o, v, len); o += len;
    }
}

/* Fill one chunk.  kind: ZMT_GEN_*; chunk_index selects the class (MIX) and the seed. */
void zmt_gen_chunk(int kind, uint64_t chunk_index, uint8_t* buf, size_t n)
{
    rng_t r;
    pthread_once(&g_once, init_tables);
    r.s = 0x5117E51AULL ^ chunk_index;
    rng_next(&r);
    switch (kind) {
    case ZMT_GEN_ZEROS: memset(buf, 0, n); return;
    case ZMT_GEN_TEXT: gen_text(&r, buf, n); return;
    case ZMT_GEN_RANDOM: gen_random(&r, buf, n); return;
    default:
        switch (chunk_index & 7) {
        case 0: case 1: gen_text(&r, buf, n); return;
        case 2: gen_xml(&r, buf, n); return;
        case 3: gen_walk16(&r, buf, n); return;
        case 4: gen_structs(&r, buf, n); return;
        case 5: gen_opcodes(&r, buf, n); return;
        case 6: gen_random(&r, buf, n); return;
        default: gen_runs(&r, buf, n); return;
        }
    }
}

typedef struct { int kind; uint64_t first, count, stride; size_t chunk; uint8_t* buf; size_t total; uint64_t next; pthread_mutex_t mu;
                 uint64_t batch, rank, world; } gen_job;

static void* gen_worker(void* arg)
{
    gen_job* j = (gen_job*)arg;
    for (;;) {
        uint64_t i;
        pthread_mutex_lock(&j->mu); i = j->next++; pthread_mutex_unlock(&j->mu);
        if (i >= j->count) break;
        {
            size_t off = (size_t)i * j->chunk, n = j->total - off < j->chunk ? j->total - off : j->chunk;
            /* batch != 0: chunks dealt to `world` consumers in batches (the product's granularity): local chunk i of
             * consumer `rank` is global chunk (i / batch) * batch * world + rank * batch + i % batch */
            const uint64_t g = j->batch ? (i / j->batch) * j->batch * j->world + j->rank * j->batch + i % j->batch : j->first + i * j->stride;
            zmt_gen_chunk(j->kind, g, j->buf + off, n);
        }
    }
    return NULL;
}

/* Fill `total` bytes = consecutive chunks of `chunk` bytes; local chunk i gets global index
 * first + i*stride (stride = world size for the round-robin multi-GPU split). */
static void gen_run(int kind, uint64_t first, uint64_t stride, uint64_t batch, uint64_t rank, uint64_t world, size_t chunk, uint8_t* buf, size_t total, int nthreads);

void zmt_gen_stream(int kind, uint64_t first, uint64_t stride, size_t chunk, uint8_t* buf, size_t total, int nthreads)
{
    gen_run(kind, first, stride, 0, 0, 1, chunk, buf, total, nthreads);
}

/* the share of consumer `rank` of `world` when the global stream is dealt round-robin in batches of `batch` chunks */
void zmt_gen_stream_dealt(int kind, uint64_t rank, uint64_t world, uint64_t batch, size_t chunk, uint8_t* buf, size_t total, int nthreads)
{
    gen_run(kind, 0, 1, batch ? batch : 1, rank, world ? world : 1, chunk, buf, total, nthreads);
}

static void gen_run(int kind, uint64_t first, uint64_t stride, uint64_t batch, uint64_t rank, uint64_t world, size_t chunk, uint8_t* buf, size_t total, int nthreads)
{
    gen_job j; pthread_t th[64]; int t;
    if (!total || !chunk) return;
    j.batch = batch; j.rank = rank; j.world = world;
    j.kind = kind; j.first = first; j.stride = stride ? stride : 1; j.chunk = chunk; j.buf = buf; j.total = total; j.next = 0;
    j.count = (total + chunk - 1) / chunk;
    pthread_mutex_init(&j.mu, NULL);
    if (nthreads < 1) nthreads = 1; if (nthreads > 64) nthreads = 64;
    if ((uint64_t)nthreads > j.count) nthreads = (int)j.count;
    for (t = 1; t < nthreads; t++) pthread_create(&th[t], NULL, gen_worker, &j);
    gen_worker(&j);
    for (t = 1; t < nthreads; t++) pthread_join(th[t], NULL);
    pthread_mutex_destroy(&j.mu);
}
