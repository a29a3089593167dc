/* zstdmt_b200_zstd.h — drop-in C boundary for the Zstandard half of zstdmt's hot path.
 *
 * Same contract as lib/zstd-mt.h (:41-60 errors, :67-93 buffer +
 * callbacks, :115-205 contexts).  The symbols the reference really exports carry
 * the ZSTDCB_ prefix (programs/zstd-mt.c:24-43 binds them); the ZSTDMT_ names of
 * lib/README.md:43-76 / BASELINE.json are exported as aliases of the same code.
 */
#ifndef ZSTDMT_B200_ZSTD_H
#define ZSTDMT_B200_ZSTD_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

/* limits and magics — lib/zstd-mt.h:26-35 */
#define ZSTDCB_THREAD_MAX       128
#define ZSTDCB_LEVEL_MIN        1
#define ZSTDCB_LEVEL_MAX        22
#define ZSTDCB_MAGICNUMBER_V01  0x1EB52FFDU
#define ZSTDCB_MAGICNUMBER_MIN  0xFD2FB522U
#define ZSTDCB_MAGICNUMBER_MAX  0xFD2FB528U
#define ZSTDCB_MAGIC_SKIPPABLE  0x184D2A50U

/* error codes (numbering differs from the LZ4 twin: init_missing) — lib/zstd-mt.h:41-54 */
typedef enum {
    ZSTDCB_error_no_error,
    ZSTDCB_error_memory_allocation,
    ZSTDCB_error_init_missing,
    ZSTDCB_error_read_fail,
    ZSTDCB_error_write_fail,
    ZSTDCB_error_data_error,
    ZSTDCB_error_frame_compress,
    ZSTDCB_error_frame_decompress,
    ZSTDCB_error_compressionParameter_unsupported,
    ZSTDCB_error_compression_library,
    ZSTDCB_error_canceled,
    ZSTDCB_error_maxCode
} ZSTDCB_ErrorCode;

extern size_t zstdmt_errcode;                     /* lib/zstd-mt.h:56 */

#define ZSTDCB_PREFIX(name) ZSTDCB_error_##name
#define ZSTDCB_ERROR(name)  ((size_t)-ZSTDCB_PREFIX(name))
unsigned    ZSTDCB_isError(size_t code);          /* lib/zstd-mt_common.c:26 */
const char* ZSTDCB_getErrorString(size_t code);   /* lib/zstd-mt_common.c:34 */

/* I/O contract — lib/zstd-mt.h:67-93; identical to the LZ4 twin */
typedef struct {
    void*  buf;
    size_t size;
    size_t allocated;
} ZSTDCB_Buffer;

typedef int (fn_read)(void* args, ZSTDCB_Buffer* in);
typedef int (fn_write)(void* args, ZSTDCB_Buffer* out);

typedef struct {
    fn_read*  fn_read;
    void*     arg_read;
    fn_write* fn_write;
    void*     arg_write;
} ZSTDCB_RdWr_t;

/* compression — lib/zstd-mt_compress.c:94, :322, :395-420, :423.
 * inputsize 0 selects 1 << (windowLog(level)+1) with the reference's table
 * (zstd-mt_compress.c:118-127). */
typedef struct ZSTDCB_CCtx_s ZSTDCB_CCtx;
ZSTDCB_CCtx* ZSTDCB_createCCtx(int threads, int level, int inputsize);
size_t ZSTDCB_compressCCtx(ZSTDCB_CCtx* ctx, ZSTDCB_RdWr_t* rdwr);
size_t ZSTDCB_GetFramesCCtx(ZSTDCB_CCtx* ctx);
size_t ZSTDCB_GetInsizeCCtx(ZSTDCB_CCtx* ctx);
size_t ZSTDCB_GetOutsizeCCtx(ZSTDCB_CCtx* ctx);
void   ZSTDCB_freeCCtx(ZSTDCB_CCtx* ctx);

/* decompression — lib/zstd-mt_decompress.c:105, :693, :845-869, :871 */
typedef struct ZSTDCB_DCtx_s ZSTDCB_DCtx;
ZSTDCB_DCtx* ZSTDCB_createDCtx(int threads, int inputsize);
size_t ZSTDCB_decompressDCtx(ZSTDCB_DCtx* ctx, ZSTDCB_RdWr_t* rdwr);
size_t ZSTDCB_GetFramesDCtx(ZSTDCB_DCtx* ctx);
size_t ZSTDCB_GetInsizeDCtx(ZSTDCB_DCtx* ctx);
size_t ZSTDCB_GetOutsizeDCtx(ZSTDCB_DCtx* ctx);
void   ZSTDCB_freeDCtx(ZSTDCB_DCtx* ctx);

/* ZSTDMT_* spellings (lib/README.md:43-76): same entry points, same types */
typedef ZSTDCB_CCtx   ZSTDMT_CCtx;
typedef ZSTDCB_DCtx   ZSTDMT_DCtx;
typedef ZSTDCB_Buffer ZSTDMT_Buffer;
typedef ZSTDCB_RdWr_t ZSTDMT_RdWr_t;
ZSTDMT_CCtx* ZSTDMT_createCCtx(int threads, int level, int inputsize);
size_t ZSTDMT_compressCCtx(ZSTDMT_CCtx* ctx, ZSTDMT_RdWr_t* rdwr);
size_t ZSTDMT_GetFramesCCtx(ZSTDMT_CCtx* ctx);
size_t ZSTDMT_GetInsizeCCtx(ZSTDMT_CCtx* ctx);
size_t ZSTDMT_GetOutsizeCCtx(ZSTDMT_CCtx* ctx);
void   ZSTDMT_freeCCtx(ZSTDMT_CCtx* ctx);
ZSTDMT_DCtx* ZSTDMT_createDCtx(int threads, int inputsize);
size_t ZSTDMT_decompressDCtx(ZSTDMT_DCtx* ctx, ZSTDMT_RdWr_t* rdwr);
size_t ZSTDMT_GetFramesDCtx(ZSTDMT_DCtx* ctx);
size_t ZSTDMT_GetInsizeDCtx(ZSTDMT_DCtx* ctx);
size_t ZSTDMT_GetOutsizeDCtx(ZSTDMT_DCtx* ctx);
void   ZSTDMT_freeDCtx(ZSTDMT_DCtx* ctx);
unsigned    ZSTDMT_isError(size_t code);
const char* ZSTDMT_getErrorString(size_t code);

#ifdef __cplusplus
}
#endif
#endif
