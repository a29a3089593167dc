// launch.h — host-side launch pieces shared by lz4_kernels.cu, zstd_decode.cu, frame_index.cu and range_read.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

__host__ __device__ inline uint64_t a256(uint64_t x) { return (x + 255) & ~255ull; }

// A workspace layout: one function per entry point places the regions from `base`; with base == nullptr it only adds up
// their sizes.  The *_workspace_bytes function and the launcher both call it, so the size a caller allocates is the
// size the launcher carves.
struct ZmtCarve {
    uint8_t* base; uint64_t off;
    template <class T> T* take(uint64_t bytes) { T* p = base ? (T*)(base + off) : nullptr; off += bytes; return p; }
};

// Per-kernel timing (zmt_prof_begin / zmt_prof_end, lz4_kernels.cu): while profiling is on, the scope records an event on
// its stream where it opens and one where it closes, reported under its ZMT_K_* id.  zmt_prof_open returns nullptr when off.
cudaEvent_t zmt_prof_open(cudaStream_t st);
void zmt_prof_close(int id, cudaEvent_t a, cudaStream_t st);
struct ZmtProfScope {
    int id; cudaStream_t st; cudaEvent_t a;
    ZmtProfScope(int id_, cudaStream_t s) : id(id_), st(s), a(zmt_prof_open(s)) {}
    ~ZmtProfScope() { if (a) zmt_prof_close(id, a, st); }
};
