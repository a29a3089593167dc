/* zstdmt_b200_lz4.h — drop-in C boundary for the LZ4 half of zstdmt's hot path.
 *
 * libzstdmt_b200.so exports every symbol that lib/lz4-mt.h
 * declares (lz4-mt.h:39-61 error handling, :67-89 buffer + callbacks, :106-159
 * contexts), with the same argument meaning and error convention, so a program
 * written against the reference (programs/lz4-mt.c:24-43 -> programs/main.c)
 * links against this library unchanged.  Behind the boundary the pthread pool +
 * liblz4 of lib/lz4-mt_compress.c / lib/lz4-mt_decompress.c is replaced by a
 * host pipeline feeding sm_90a CUDA kernels (DESIGN.md).
 *
 * Each entry point cites the reference definition it replaces.
 */
#ifndef ZSTDMT_B200_LZ4_H
#define ZSTDMT_B200_LZ4_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

/* limits — lib/lz4-mt.h:27-33 */
#define LZ4MT_THREAD_MAX        128
#define LZ4MT_LEVEL_MIN         1
#define LZ4MT_LEVEL_MAX         12
#define LZ4FMT_MAGICNUMBER      0x184D2204U
#define LZ4FMT_MAGIC_SKIPPABLE  0x184D2A50U

/* error codes: functions returning size_t return 0 on success or (size_t)-code
 * (lib/lz4-mt.h:41-53, lz4-mt_common.c:25-28) */
typedef enum {
    LZ4MT_error_no_error,
    LZ4MT_error_memory_allocation,
    LZ4MT_error_read_fail,
    LZ4MT_error_write_fail,
    LZ4MT_error_data_error,
    LZ4MT_error_frame_compress,
    LZ4MT_error_frame_decompress,
    LZ4MT_error_compressionParameter_unsupported,
    LZ4MT_error_compression_library,
    LZ4MT_error_canceled,
    LZ4MT_error_maxCode
} LZ4MT_ErrorCode;

/* lib/lz4-mt.h:39 — holds the device-side status of the last failed frame
 * (ZMT_ST_* of include/zstdmt_b200_dev.h) instead of a liblz4 error code */
extern size_t lz4mt_errcode;

#ifdef ERROR
#  undef ERROR
#endif
#define PREFIX(name) LZ4MT_error_##name
#define ERROR(name)  ((size_t)-PREFIX(name))
unsigned    LZ4MT_isError(size_t code);          /* lib/lz4-mt_common.c:25 */
const char* LZ4MT_getErrorString(size_t code);   /* lib/lz4-mt_common.c:33 */

/* I/O contract — lib/lz4-mt.h:67-89.  The library owns `buf`.
 *   fn_read : on entry size = bytes wanted; callee fills buf and sets size to the
 *             bytes delivered (0 = end of input).
 *   fn_write: buf/size = bytes to emit; the value of size after the call is what
 *             the Outsize counter accumulates (lz4-mt_compress.c:194-197).
 *   return 0 ok, -1 I/O error, -2 user abort, -3 out of memory.
 * Reads are never concurrent with reads, writes never with writes; a read and a
 * write may overlap (as in the reference's worker pool). */
typedef struct {
    void*  buf;
    size_t size;
    size_t allocated;
} LZ4MT_Buffer;

typedef int (fn_read)(void* args, LZ4MT_Buffer* in);
typedef int (fn_write)(void* args, LZ4MT_Buffer* out);

typedef struct {
    fn_read*  fn_read;
    void*     arg_read;
    fn_write* fn_write;
    void*     arg_write;
} LZ4MT_RdWr_t;

/* compression — lib/lz4-mt_compress.c:92 (create), :312 (compress), :356-380 (stats), :382 (free).
 * `threads` (1..128) bounds the batches kept in flight per GPU; `level` 1..12 is
 * accepted, the device encoder implements the level-1 class; `inputsize` is the
 * chunk size (0 -> 4 MiB). */
typedef struct LZ4MT_CCtx_s LZ4MT_CCtx;
LZ4MT_CCtx* LZ4MT_createCCtx(int threads, int level, int inputsize);
size_t LZ4MT_compressCCtx(LZ4MT_CCtx* ctx, LZ4MT_RdWr_t* rdwr);
size_t LZ4MT_GetFramesCCtx(LZ4MT_CCtx* ctx);
size_t LZ4MT_GetInsizeCCtx(LZ4MT_CCtx* ctx);
size_t LZ4MT_GetOutsizeCCtx(LZ4MT_CCtx* ctx);
void   LZ4MT_freeCCtx(LZ4MT_CCtx* ctx);

/* decompression — lib/lz4-mt_decompress.c:90 (create), :485 (decompress), :569-593 (stats), :595 (free) */
typedef struct LZ4MT_DCtx_s LZ4MT_DCtx;
LZ4MT_DCtx* LZ4MT_createDCtx(int threads, int inputsize);
size_t LZ4MT_decompressDCtx(LZ4MT_DCtx* ctx, LZ4MT_RdWr_t* rdwr);
size_t LZ4MT_GetFramesDCtx(LZ4MT_DCtx* ctx);
size_t LZ4MT_GetInsizeDCtx(LZ4MT_DCtx* ctx);
size_t LZ4MT_GetOutsizeDCtx(LZ4MT_DCtx* ctx);
void   LZ4MT_freeDCtx(LZ4MT_DCtx* ctx);

#ifdef __cplusplus
}
#endif
#endif
