/* oracle/shim/zstd.h — TEST INFRASTRUCTURE ONLY.
 *
 * Hand-declared subset of the libzstd stable API (ABI of the image's
 * /usr/lib/x86_64-linux-gnu/libzstd.so.1.5.5; no dev headers installed).
 * Lets the UNMODIFIED reference wrapper (lib/zstd-mt_*.c)
 * compile into oracle/_ref/ (oracle/Makefile).  The reference pins v1.5.6
 * (programs/Makefile:11); 1.5.5 is format-identical.  Not used by the product.
 */
#ifndef ORACLE_SHIM_ZSTD_H
#define ORACLE_SHIM_ZSTD_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

unsigned    ZSTD_isError(size_t code);
const char* ZSTD_getErrorName(size_t code);
size_t ZSTD_compress(void* dst, size_t dstCapacity, const void* src, size_t srcSize, int level);
size_t ZSTD_decompress(void* dst, size_t dstCapacity, const void* src, size_t compressedSize);
size_t ZSTD_compressBound(size_t srcSize);
unsigned long long ZSTD_getFrameContentSize(const void* src, size_t srcSize);

typedef struct ZSTD_DCtx_s ZSTD_DCtx;
typedef ZSTD_DCtx ZSTD_DStream;
typedef struct { const void* src; size_t size; size_t pos; } ZSTD_inBuffer;
typedef struct { void* dst; size_t size; size_t pos; } ZSTD_outBuffer;

ZSTD_DStream* ZSTD_createDStream(void);
size_t ZSTD_freeDStream(ZSTD_DStream* zds);
size_t ZSTD_initDStream(ZSTD_DStream* zds);
size_t ZSTD_resetDStream(ZSTD_DStream* zds);
size_t ZSTD_decompressStream(ZSTD_DStream* zds, ZSTD_outBuffer* output, ZSTD_inBuffer* input);
size_t ZSTD_DStreamInSize(void);
size_t ZSTD_DStreamOutSize(void);

#ifdef __cplusplus
}
#endif
#endif
