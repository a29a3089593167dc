/* oracle/shim/lz4frame.h — TEST INFRASTRUCTURE ONLY.
 *
 * Hand-declared subset of the liblz4 v1.9.4 frame API (public ABI of
 * /usr/lib/x86_64-linux-gnu/liblz4.so.1.9.4; the image ships the .so but no
 * dev headers).  Exists only so that the UNMODIFIED reference wrapper
 * (lib/lz4-mt_*.c) can be compiled into oracle/_ref/ — see
 * oracle/Makefile.  Struct layouts follow the documented v1.9.4 ABI
 * (sizeof(LZ4F_frameInfo_t)==32, sizeof(LZ4F_preferences_t)==56; checked by
 * tests/test_oracle_ref.py).  Nothing in the product links against this.
 */
#ifndef ORACLE_SHIM_LZ4FRAME_H
#define ORACLE_SHIM_LZ4FRAME_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define LZ4F_VERSION 100
typedef size_t LZ4F_errorCode_t;

typedef enum { LZ4F_default = 0, LZ4F_max64KB = 4, LZ4F_max256KB = 5,
               LZ4F_max1MB = 6, LZ4F_max4MB = 7 } LZ4F_blockSizeID_t;
typedef enum { LZ4F_blockLinked = 0, LZ4F_blockIndependent } LZ4F_blockMode_t;
typedef enum { LZ4F_noContentChecksum = 0, LZ4F_contentChecksumEnabled } LZ4F_contentChecksum_t;
typedef enum { LZ4F_noBlockChecksum = 0, LZ4F_blockChecksumEnabled } LZ4F_blockChecksum_t;
typedef enum { LZ4F_frame = 0, LZ4F_skippableFrame } LZ4F_frameType_t;

typedef struct {
    LZ4F_blockSizeID_t     blockSizeID;
    LZ4F_blockMode_t       blockMode;
    LZ4F_contentChecksum_t contentChecksumFlag;
    LZ4F_frameType_t       frameType;
    unsigned long long     contentSize;
    unsigned               dictID;
    LZ4F_blockChecksum_t   blockChecksumFlag;
} LZ4F_frameInfo_t;

typedef struct {
    LZ4F_frameInfo_t frameInfo;
    int      compressionLevel;
    unsigned autoFlush;
    unsigned favorDecSpeed;
    unsigned reserved[3];
} LZ4F_preferences_t;

typedef struct LZ4F_dctx_s LZ4F_dctx;
typedef LZ4F_dctx* LZ4F_decompressionContext_t;

typedef struct {
    unsigned stableDst;
    unsigned skipChecksums;
    unsigned reserved1;
    unsigned reserved0;
} LZ4F_decompressOptions_t;

unsigned    LZ4F_isError(LZ4F_errorCode_t code);
const char* LZ4F_getErrorName(LZ4F_errorCode_t code);
size_t LZ4F_compressFrameBound(size_t srcSize, const LZ4F_preferences_t* prefs);
size_t LZ4F_compressFrame(void* dst, size_t dstCapacity, const void* src, size_t srcSize,
                          const LZ4F_preferences_t* prefs);
LZ4F_errorCode_t LZ4F_createDecompressionContext(LZ4F_dctx** dctxPtr, unsigned version);
LZ4F_errorCode_t LZ4F_freeDecompressionContext(LZ4F_dctx* dctx);
size_t LZ4F_decompress(LZ4F_dctx* dctx, void* dst, size_t* dstSizePtr,
                       const void* src, size_t* srcSizePtr,
                       const LZ4F_decompressOptions_t* opts);

#ifdef __cplusplus
}
#endif
#endif
