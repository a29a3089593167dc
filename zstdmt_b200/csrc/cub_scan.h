// cub_scan.h — cub's exclusive sums for frame_index.cu and range_read.cu (not in launch.h: cub adds a kernel to every module).
#pragma once
#include <cub/device/device_scan.cuh>

// bytes of cub's temporary storage for an exclusive sum over nitems entries of either width (0: cub failed)
inline size_t scan_tmp_bytes(uint32_t nitems)
{
    size_t a = 0, b = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, a, (uint64_t*)nullptr, (int)nitems) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, b, (uint32_t*)nullptr, (int)nitems) != cudaSuccess) { cudaGetLastError(); return 0; }
    return a > b ? a : b;
}
// in-place exclusive sum of a[0..n) in the scan storage of workspace k (k.tmp, k.tmp_bytes >= scan_tmp_bytes(n))
template <typename Work, typename T>
bool exclusive_sum(const Work& k, T* a, uint64_t n, cudaStream_t st) { size_t t = k.tmp_bytes; return cub::DeviceScan::ExclusiveSum(k.tmp, t, a, (int)n, st) == cudaSuccess; }
