/* memio_glue.c — memory-to-memory driver for the reference-shaped callback API.
 *
 * Drives {LZ4MT,ZSTDCB}_{compressCCtx,decompressDCtx} with fn_read/fn_write
 * callbacks that memcpy from / to caller-provided RAM (the in-process harness
 * SURVEY.md §8d / BASELINE.md §3 prescribe: no files, no pipes).  The SAME
 * source is compiled twice:
 *   - into libzstdmt_b200.so with -DGLUE_PREFIX=zmt_   (drives OUR library)
 *   - into oracle/_ref/libzstdmt_ref.so with -DGLUE_PREFIX=ref_ (drives the
 *     unmodified reference wrapper + liblz4/libzstd)
 * so the e2e and cpu_baseline numbers go through byte-identical callbacks.
 * The callback contract mirrored here: lib/lz4-mt.h:67-89,
 * lib/zstd-mt.h:67-93, CLI callbacks programs/main.c:172-200.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#ifndef GLUE_PREFIX
#define GLUE_PREFIX zmt_
#endif
#define GLUE_CAT2(a, b) a##b
#define GLUE_CAT(a, b) GLUE_CAT2(a, b)
#define GLUE(name) GLUE_CAT(GLUE_PREFIX, name)

/* structurally identical for both codecs (lz4-mt.h:67-71, zstd-mt.h:67-71) */
typedef struct { void* buf; size_t size; size_t allocated; } mt_buffer;
typedef int (mt_rw_fn)(void* arg, mt_buffer* b);
typedef struct { mt_rw_fn* fn_read; void* arg_read; mt_rw_fn* fn_write; void* arg_write; } mt_rdwr;

extern void*  LZ4MT_createCCtx(int threads, int level, int inputsize);
extern size_t LZ4MT_compressCCtx(void* ctx, mt_rdwr* rdwr);
extern size_t LZ4MT_GetFramesCCtx(void* ctx);
extern size_t LZ4MT_GetInsizeCCtx(void* ctx);
extern size_t LZ4MT_GetOutsizeCCtx(void* ctx);
extern void   LZ4MT_freeCCtx(void* ctx);
extern void*  LZ4MT_createDCtx(int threads, int inputsize);
extern size_t LZ4MT_decompressDCtx(void* ctx, mt_rdwr* rdwr);
extern size_t LZ4MT_GetFramesDCtx(void* ctx);
extern size_t LZ4MT_GetInsizeDCtx(void* ctx);
extern size_t LZ4MT_GetOutsizeDCtx(void* ctx);
extern void   LZ4MT_freeDCtx(void* ctx);
extern void*  ZSTDCB_createCCtx(int threads, int level, int inputsize);
extern size_t ZSTDCB_compressCCtx(void* ctx, mt_rdwr* rdwr);
extern size_t ZSTDCB_GetFramesCCtx(void* ctx);
extern size_t ZSTDCB_GetInsizeCCtx(void* ctx);
extern size_t ZSTDCB_GetOutsizeCCtx(void* ctx);
extern void   ZSTDCB_freeCCtx(void* ctx);
extern void*  ZSTDCB_createDCtx(int threads, int inputsize);
extern size_t ZSTDCB_decompressDCtx(void* ctx, mt_rdwr* rdwr);
extern size_t ZSTDCB_GetFramesDCtx(void* ctx);
extern size_t ZSTDCB_GetInsizeDCtx(void* ctx);
extern size_t ZSTDCB_GetOutsizeDCtx(void* ctx);
extern void   ZSTDCB_freeDCtx(void* ctx);

typedef struct {
    const uint8_t* src; size_t srcSize, srcPos;
    uint8_t* dst; size_t dstCap, dstPos;
    size_t nreads, nwrites;
    int overflow;
} memio;

static int mem_read(void* arg, mt_buffer* b)
{
    memio* m = (memio*)arg;
    size_t want = b->size, left = m->srcSize - m->srcPos;
    if (want > left) want = left;
    if (want) memcpy(b->buf, m->src + m->srcPos, want);
    m->srcPos += want; b->size = want; m->nreads++;
    return 0;
}
static int mem_write(void* arg, mt_buffer* b)
{
    memio* m = (memio*)arg;
    m->nwrites++;
    if (b->size > m->dstCap - m->dstPos) { m->overflow = 1; return -1; }
    if (m->dst) memcpy(m->dst + m->dstPos, b->buf, b->size);
    m->dstPos += b->size;
    return 0;
}

/* stats[0..4] = outBytes, frames, insize counter, outsize counter, (reads<<32 | writes) */
#define GLUE_BODY(CREATE, RUN, GF, GI, GO, FREE)                                   \
    memio m; mt_rdwr rw; size_t rc; void* ctx = CREATE;                              \
    if (!ctx) return (size_t)-1000;                                                  \
    memset(&m, 0, sizeof(m)); m.src = (const uint8_t*)src; m.srcSize = n;            \
    m.dst = (uint8_t*)dst; m.dstCap = cap;                                           \
    rw.fn_read = mem_read; rw.arg_read = &m; rw.fn_write = mem_write; rw.arg_write = &m; \
    rc = RUN(ctx, &rw);                                                              \
    if (stats) { stats[0] = m.dstPos; stats[1] = GF(ctx); stats[2] = GI(ctx); stats[3] = GO(ctx); \
                 stats[4] = (m.nreads << 32) | (m.nwrites & 0xFFFFFFFFu); }          \
    FREE(ctx);                                                                       \
    return rc;

size_t GLUE(lz4_compress_mem)(int threads, int level, int chunk, const void* src, size_t n, void* dst, size_t cap, size_t* stats)
{ GLUE_BODY(LZ4MT_createCCtx(threads, level, chunk), LZ4MT_compressCCtx, LZ4MT_GetFramesCCtx, LZ4MT_GetInsizeCCtx, LZ4MT_GetOutsizeCCtx, LZ4MT_freeCCtx) }

size_t GLUE(lz4_decompress_mem)(int threads, int inputsize, const void* src, size_t n, void* dst, size_t cap, size_t* stats)
{ GLUE_BODY(LZ4MT_createDCtx(threads, inputsize), LZ4MT_decompressDCtx, LZ4MT_GetFramesDCtx, LZ4MT_GetInsizeDCtx, LZ4MT_GetOutsizeDCtx, LZ4MT_freeDCtx) }

size_t GLUE(zstd_compress_mem)(int threads, int level, int chunk, const void* src, size_t n, void* dst, size_t cap, size_t* stats)
{ GLUE_BODY(ZSTDCB_createCCtx(threads, level, chunk), ZSTDCB_compressCCtx, ZSTDCB_GetFramesCCtx, ZSTDCB_GetInsizeCCtx, ZSTDCB_GetOutsizeCCtx, ZSTDCB_freeCCtx) }

size_t GLUE(zstd_decompress_mem)(int threads, int inputsize, const void* src, size_t n, void* dst, size_t cap, size_t* stats)
{ GLUE_BODY(ZSTDCB_createDCtx(threads, inputsize), ZSTDCB_decompressDCtx, ZSTDCB_GetFramesDCtx, ZSTDCB_GetInsizeDCtx, ZSTDCB_GetOutsizeDCtx, ZSTDCB_freeDCtx) }
