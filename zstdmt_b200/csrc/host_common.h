// host_common.h — host-side pieces shared by the launcher files (lz4_kernels.cu, zstd_decode.cu) and host_api.cpp.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <mutex>

// SM count of the current device, cached per device (contexts may run on several host threads)
static inline int zmt_sm_count()
{
    static std::mutex mu; static int n[64];
    int dev = 0; cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return 132;
    std::lock_guard<std::mutex> g(mu);
    if (!n[dev]) { cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev); if (n[dev] <= 0) n[dev] = 132; }
    return n[dev];
}

// zstd's predefined distributions (RFC 8878 §3.1.1.3.2.2): literal lengths, match lengths, offsets; and the baselines
// and extra-bit counts of the literal-length and match-length codes (§3.1.1.3.2.1.1).  The encoder builds its FSE
// encoding tables from them, the decoder its decoding tables.
static const int16_t  ZSTD_LL_NORM[36] = { 4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1 };
static const int16_t  ZSTD_ML_NORM[53] = { 1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1 };
static const int16_t  ZSTD_OF_NORM[29] = { 1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1 };
static const uint32_t ZSTD_LL_BASE[36] = { 0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,18,20,22,24,28,32,40,48,64,128,256,512,1024,2048,4096,8192,16384,32768,65536 };
static const uint8_t  ZSTD_LL_BITS[36] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16 };
static const uint32_t ZSTD_ML_BASE[53] = { 3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,35,37,39,41,43,47,51,59,67,83,99,131,259,515,1027,2051,4099,8195,16387,32771,65539 };
static const uint8_t  ZSTD_ML_BITS[53] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16 };
