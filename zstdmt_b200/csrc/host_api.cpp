// host_api.cpp — the drop-in boundary: LZ4MT_* / ZSTDCB_* (+ ZSTDMT_* aliases) on top of the CUDA kernels.
//
// Replaces the pthread worker pools of
//   lib/lz4-mt_compress.c:207-353   (pt_compress, pt_write, LZ4MT_compressCCtx)
//   lib/lz4-mt_decompress.c:165-567 (pt_read, pt_decompress, pt_write, LZ4MT_decompressDCtx)
//   lib/zstd-mt_compress.c:177-392  and  lib/zstd-mt_decompress.c:209-843
// with one software pipeline per call:
//
//   reader thread  : fn_read -> pinned staging slot (B chunks / frames per slot)
//   submit (caller): H2D -> kernels -> D2H of the size table, one CUDA stream per slot,
//                    slots dealt round-robin over the GPUs named by ZSTDMT_GPUS
//   writer thread  : waits for the slot's event, D2H of the used bytes, fn_write strictly in
//                    frame order (the pt_write rule, lz4-mt_compress.c:186-202)
//
// Callback contract kept: reads never overlap reads, writes never overlap writes, a read and a
// write may overlap (as with the reference's read_mutex / write_mutex).  No CPU codec fallback:
// if the CUDA runtime or a kernel fails the call returns *_error_compression_library.
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <cuda_runtime.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>
#include "zmt_dev.h"

extern "C" {
size_t   zmt_zstdc_workspace_bytes(uint32_t nchunks, uint32_t chunk_size);
uint64_t zmt_zstdc_out_bound(uint32_t nchunks, uint32_t chunk_size);
int      zmt_zstd_compress_device(const void*, uint64_t, uint32_t, const uint32_t*, uint32_t, void*, void*, uint64_t*, void*);
size_t   zmt_zstd_blk_desc_bytes(void);
int      zmt_zstd_scan_frame_host(const uint8_t* frame, size_t n, uint64_t base_off, uint32_t frame_idx, void* blocks_out, uint32_t* nblocks_io,
                                  uint32_t max_blocks, uint64_t* scratch_used, uint64_t* content_size, uint32_t* needs_seq);
int      zmt_zstd_scan_frame_host2(const uint8_t* frame, size_t n, uint64_t base_off, uint32_t frame_idx, void* blocks_out, uint32_t* nblocks_io,
                                   uint32_t max_blocks, uint64_t* scratch_used, uint64_t* content_size, uint32_t* needs_seq, size_t* consumed);
size_t   zmt_zstdd_workspace_bytes(uint32_t nframes, uint32_t nblocks, uint64_t scratch_bytes);
int      zmt_zstd_decompress_device(const void* d_in, const void* d_blocks, uint32_t nblocks, const uint32_t* d_frame_first_blk, const uint64_t* d_expect,
                                    const uint32_t* d_frame_seq, uint32_t nframes, void* d_out, const uint64_t* d_out_off, uint64_t* d_out_size, uint32_t* d_status,
                                    void* d_work, void* stream);
}

namespace {

// ------------------------------------------------------------------ generic boundary types
struct GenBuffer { void* buf; size_t size; size_t allocated; };     // == LZ4MT_Buffer == ZSTDCB_Buffer
typedef int (gen_rw_fn)(void* arg, GenBuffer* b);
struct GenRdWr { gen_rw_fn* fn_read; void* arg_read; gen_rw_fn* fn_write; void* arg_write; };

enum { CODEC_LZ4 = 1, CODEC_ZSTD = 2 };
#define MT_MAGIC_SKIPPABLE 0x184D2A50u
#define LZ4F_MAGIC         0x184D2204u
#define ZSTD_MAGIC         0xFD2FB528u

// error numbering differs between the codecs (lz4-mt.h:41-53 vs zstd-mt.h:41-54)
struct ErrCodes { size_t mem, read_fail, write_fail, data_error, frame_compress, frame_decompress, param, library, canceled, init_missing; };
const ErrCodes kErrLz4  = { (size_t)-1, (size_t)-2, (size_t)-3, (size_t)-4, (size_t)-5, (size_t)-6, (size_t)-7, (size_t)-8, (size_t)-9, (size_t)-7 };
const ErrCodes kErrZstd = { (size_t)-1, (size_t)-3, (size_t)-4, (size_t)-5, (size_t)-6, (size_t)-7, (size_t)-8, (size_t)-9, (size_t)-10, (size_t)-2 };

inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline uint64_t rd64(const uint8_t* p) { return (uint64_t)rd32(p) | ((uint64_t)rd32(p + 4) << 32); }

// callback return -> library error (mt_error, lz4-mt_compress.c:161-173: write failures also map to read_fail)
inline size_t mt_error(const ErrCodes& E, int rv)
{
    switch (rv) { case -1: return E.read_fail; case -2: return E.canceled; case -3: return E.mem; }
    return E.read_fail;
}

size_t env_size(const char* name, size_t dflt)
{
    const char* v = getenv(name);
    if (!v || !*v) return dflt;
    char* end = nullptr; unsigned long long x = strtoull(v, &end, 10);
    return (end && end != v) ? (size_t)x : dflt;
}

std::vector<int> env_devices()
{
    std::vector<int> devs;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return devs;
    const char* v = getenv("ZSTDMT_GPUS");
    if (v && *v) {
        if (!strcmp(v, "all")) { for (int i = 0; i < ndev; i++) devs.push_back(i); return devs; }
        const char* p = v;
        while (*p) {
            char* end = nullptr; long d = strtol(p, &end, 10);
            if (end == p) break;
            if (d >= 0 && d < ndev) devs.push_back((int)d);
            p = (*end == ',') ? end + 1 : end;
            if (*end != ',' && *end != 0) break;
        }
        if (!devs.empty()) return devs;
    }
    int cur = 0;
    if (cudaGetDevice(&cur) != cudaSuccess) cur = 0;
    devs.push_back(cur);
    return devs;
}

// batches submitted per device since the library was loaded (zmt_device_batches: lets a caller / test see the round-robin deal)
std::atomic<uint64_t> g_dev_batches[64];

// ------------------------------------------------------------------ NUMA placement
// The staging rings are the memcpy targets / sources of the (serialised) fn_read / fn_write callbacks and the DMA
// sources / targets of the GPU: both want them on the GPU's own NUMA node.  Linux places pages on the node of the
// thread that first touches them, so the pinned buffers are allocated with the calling thread temporarily bound to
// the CPUs of the GPU's PCIe root (/sys/bus/pci/devices/<id>/local_cpulist), and the reader / writer threads of a
// call run there too.  ZSTDMT_B200_NUMA=0 turns both off.
struct CpuSet { cpu_set_t set; bool ok = false; };

bool numa_enabled() { static int on = -1; if (on < 0) { const char* v = getenv("ZSTDMT_B200_NUMA"); on = (v && *v == '0') ? 0 : 1; } return on == 1; }

CpuSet device_local_cpus(int dev)
{
    CpuSet r; CPU_ZERO(&r.set);
    if (!numa_enabled()) return r;
    char id[32] = {0};
    if (cudaDeviceGetPCIBusId(id, (int)sizeof(id), dev) != cudaSuccess) { cudaGetLastError(); return r; }
    for (char* q = id; *q; q++) if (*q >= 'A' && *q <= 'Z') *q = (char)(*q - 'A' + 'a');
    char path[128]; snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/local_cpulist", id);
    FILE* f = fopen(path, "r");
    if (!f) return r;
    char buf[1024] = {0};
    const bool got = fgets(buf, sizeof(buf), f) != nullptr;
    fclose(f);
    if (!got) return r;
    int n = 0;
    for (const char* q = buf; *q && *q != '\n';) {          // "0-31,64-95"
        char* end = nullptr; long a = strtol(q, &end, 10); if (end == q) break;
        long b = a; q = end;
        if (*q == '-') { b = strtol(q + 1, &end, 10); if (end == q + 1) break; q = end; }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) { if (c >= 0) { CPU_SET((int)c, &r.set); n++; } }
        if (*q == ',') q++;
    }
    // stay inside the affinity the process was given (containers, numactl)
    cpu_set_t cur; CPU_ZERO(&cur);
    if (sched_getaffinity(0, sizeof(cur), &cur) == 0) {
        cpu_set_t both; CPU_AND(&both, &cur, &r.set);
        if (CPU_COUNT(&both) == 0) return r;
        r.set = both;
    }
    r.ok = n > 0;
    return r;
}

// binds the calling thread for the lifetime of the object (or for good with keep())
struct ScopedAffinity {
    cpu_set_t old; bool active = false;
    explicit ScopedAffinity(const CpuSet& c) {
        if (!c.ok) return;
        CPU_ZERO(&old);
        if (sched_getaffinity(0, sizeof(old), &old) != 0) return;
        active = sched_setaffinity(0, sizeof(c.set), &c.set) == 0;
    }
    ~ScopedAffinity() { if (active) sched_setaffinity(0, sizeof(old), &old); }
};

// all devices of a call on one node -> that node's CPUs, else nothing (the staging rings then live on several nodes)
CpuSet common_local_cpus(const std::vector<int>& devs)
{
    CpuSet r; CPU_ZERO(&r.set);
    for (size_t i = 0; i < devs.size(); i++) {
        const CpuSet c = device_local_cpus(devs[i]);
        if (!c.ok) return CpuSet();
        if (i == 0) r = c; else if (!CPU_EQUAL(&r.set, &c.set)) return CpuSet();
    }
    return r;
}

// The pipeline switches the calling thread's current CUDA device while it deals batches over ZSTDMT_GPUS; a drop-in
// library must hand the thread back as it found it (a torch / CUDA caller keeps its own notion of the current device).
struct DeviceRestore {
    int prev = -1;
    DeviceRestore() { if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; } }
    ~DeviceRestore() { if (prev >= 0) cudaSetDevice(prev); }
};

// ------------------------------------------------------------------ optional stage timing (ZSTDMT_B200_TRACE=1)
struct StageClock {
    double cb = 0, wait = 0, gpu = 0;       // seconds: inside callbacks / waiting for a slot or queue / CUDA sync + copies
    static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
};
inline bool trace_on() { static int on = -1; if (on < 0) on = getenv("ZSTDMT_B200_TRACE") ? 1 : 0; return on == 1; }

// ------------------------------------------------------------------ device codec table
struct CodecOps {
    size_t   (*c_work)(uint32_t nchunks, uint32_t chunk);
    uint64_t (*c_bound)(uint32_t nchunks, uint32_t chunk);
    int      (*compress)(const void*, uint64_t, uint32_t, const uint32_t*, uint32_t, void*, void*, uint64_t*, void*);
};


const CodecOps* codec_ops(int codec)
{
    static const CodecOps lz4 = { zmt_lz4c_workspace_bytes, zmt_lz4c_out_bound, zmt_lz4_compress_device };
    static const CodecOps zstd = { zmt_zstdc_workspace_bytes, zmt_zstdc_out_bound, zmt_zstd_compress_device };
    return codec == CODEC_LZ4 ? &lz4 : &zstd;
}

// ------------------------------------------------------------------ staging slots
struct Slot {
    int dev = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev = nullptr, evp[2] = { nullptr, nullptr };       // evp: decompress writer, output pieces in flight
    uint8_t *h_in = nullptr, *h_out = nullptr, *d_in = nullptr, *d_out = nullptr, *d_work = nullptr;
    size_t in_cap = 0, out_cap = 0, work_cap = 0, tab_cap = 0;   // tab_cap: entries in the tables below
    // tables: pinned host mirror + device copy, one allocation each
    uint8_t *h_tab = nullptr, *d_tab = nullptr; size_t tab_bytes = 0;
    // batch contents
    uint32_t n = 0;              // chunks / frames in this batch
    uint32_t nslots = 1;         // lz4 decompress: block-table slots of this batch (sum over frames of max(1, ceil(out / 64 KiB)))
    uint64_t scr_cap = 0;        // zstd decompress: entropy scratch bytes the workspace was sized for
    // zstd decompress: block descriptors built by the reader (pinned) + device copy, scratch demand of the batch
    uint8_t *h_blk = nullptr, *d_blk = nullptr; uint32_t blk_cap = 0, nblk = 0; uint64_t scratch_used = 0;
    size_t in_used = 0, out_used = 0;
    int state = 0;               // 0 free, 1 filled, 2 submitted
    bool ok = false;
    bool host_alias = false;     // h_in / h_out are borrowed from another slot of the same context (never pooled, never freed here)
};

// table layout (entries = tab_cap):  u64 a[cap+1] | u64 b[cap+1] | u64 c[cap+1] | u64 f[cap+1] | u32 d[cap] | u32 e[cap] | u32 g[cap+1]
struct Tables { uint64_t *a, *b, *c, *f; uint32_t *d, *e, *g; };
inline size_t tables_bytes(size_t cap) { return 4 * (cap + 1) * 8 + 2 * cap * 4 + (cap + 1) * 4 + 64; }
inline Tables tables_at(uint8_t* base, size_t cap)
{
    Tables t; t.a = (uint64_t*)base; t.b = t.a + cap + 1; t.c = t.b + cap + 1; t.f = t.c + cap + 1;
    t.d = (uint32_t*)(t.f + cap + 1); t.e = t.d + cap; t.g = t.e + cap; return t;
}

// lz4 decode block table capacity of a slot: every frame owns max(1, ceil(out / 64 KiB)) slots
inline uint32_t lz4_slot_cap(size_t out_cap, size_t tab_cap) { return (uint32_t)(out_cap / 65536 + tab_cap + 1); }

void slot_free_raw(Slot& s)
{
    cudaSetDevice(s.dev);
    if (s.stream) cudaStreamSynchronize(s.stream);
    if (s.h_in) cudaFreeHost(s.h_in);
    if (s.h_out) cudaFreeHost(s.h_out);
    if (s.h_tab) cudaFreeHost(s.h_tab);
    if (s.d_in) cudaFree(s.d_in);
    if (s.d_out) cudaFree(s.d_out);
    if (s.d_work) cudaFree(s.d_work);
    if (s.d_tab) cudaFree(s.d_tab);
    if (s.h_blk) cudaFreeHost(s.h_blk);
    if (s.d_blk) cudaFree(s.d_blk);
    if (s.ev) cudaEventDestroy(s.ev);
    for (int k = 0; k < 2; k++) if (s.evp[k]) cudaEventDestroy(s.evp[k]);
    if (s.stream) cudaStreamDestroy(s.stream);
    s = Slot();
}

bool slot_alloc_raw(Slot& s, int dev, size_t in_cap, size_t out_cap, size_t work_cap, size_t tab_cap)
{
    s.dev = dev;
    if (cudaSetDevice(dev) != cudaSuccess) return false;
    const ScopedAffinity bind(device_local_cpus(dev));     // first touch of the pinned rings happens on the GPU's node
    bool ok = true;
    ok = ok && cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming) == cudaSuccess;
    for (int k = 0; k < 2; k++) ok = ok && cudaEventCreateWithFlags(&s.evp[k], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaHostAlloc((void**)&s.h_in, in_cap + 64, cudaHostAllocPortable) == cudaSuccess;
    ok = ok && cudaHostAlloc((void**)&s.h_out, out_cap + 64, cudaHostAllocPortable) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_in, in_cap + 256) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_out, out_cap + 256) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_work, work_cap + 256) == cudaSuccess;
    s.tab_bytes = tables_bytes(tab_cap);
    ok = ok && cudaHostAlloc((void**)&s.h_tab, s.tab_bytes, cudaHostAllocPortable) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_tab, s.tab_bytes) == cudaSuccess;
    s.in_cap = in_cap; s.out_cap = out_cap; s.work_cap = work_cap; s.tab_cap = tab_cap; s.ok = ok;
    if (!ok) { cudaGetLastError(); slot_free_raw(s); }
    return ok;
}

// Process-wide pool of staging slots: pinned allocations cost ~0.1 s per context otherwise (the reference's
// malloc'd buffers are free by comparison).  Slots go back to the pool when a context is freed and are
// reused by the next context that needs the same device and no larger capacities.
std::mutex g_pool_mu;
std::vector<Slot> g_pool;
const size_t kPoolMax = 16;

bool slot_alloc(Slot& s, int dev, size_t in_cap, size_t out_cap, size_t work_cap, size_t tab_cap)
{
    {
        std::lock_guard<std::mutex> g(g_pool_mu);
        for (size_t i = 0; i < g_pool.size(); i++) {
            Slot& c = g_pool[i];
            if (c.h_in && c.dev == dev && c.in_cap >= in_cap && c.out_cap >= out_cap && c.work_cap >= work_cap && c.tab_cap == tab_cap) {
                s = c; g_pool.erase(g_pool.begin() + (long)i);
                s.state = 0; s.n = 0; s.in_used = s.out_used = 0;
                return true;
            }
        }
    }
    return slot_alloc_raw(s, dev, in_cap, out_cap, work_cap, tab_cap);
}

// A slot whose pinned staging buffers are those of `owner` (a call over more devices than it keeps batches in flight: the
// host ring stays 4 x 8 MiB — cache-resident for the callbacks' memcpy — while every device has its own device-side buffers).
bool slot_alloc_alias(Slot& s, const Slot& owner, int dev, size_t in_cap, size_t out_cap, size_t work_cap, size_t tab_cap)
{
    {
        std::lock_guard<std::mutex> g(g_pool_mu);                       // a pooled device-only slot of a previous call
        for (size_t i = 0; i < g_pool.size(); i++) {
            Slot& c = g_pool[i];
            if (!c.h_in && c.dev == dev && c.in_cap >= in_cap && c.out_cap >= out_cap && c.work_cap >= work_cap && c.tab_cap == tab_cap) {
                s = c; g_pool.erase(g_pool.begin() + (long)i);
                s.state = 0; s.n = 0; s.in_used = s.out_used = 0;
                s.h_in = owner.h_in; s.h_out = owner.h_out; s.host_alias = true;
                return true;
            }
        }
    }
    s.dev = dev;
    if (cudaSetDevice(dev) != cudaSuccess) return false;
    bool ok = true;
    ok = ok && cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming) == cudaSuccess;
    for (int k = 0; k < 2; k++) ok = ok && cudaEventCreateWithFlags(&s.evp[k], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_in, in_cap + 256) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_out, out_cap + 256) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_work, work_cap + 256) == cudaSuccess;
    s.tab_bytes = tables_bytes(tab_cap);
    ok = ok && cudaHostAlloc((void**)&s.h_tab, s.tab_bytes, cudaHostAllocPortable) == cudaSuccess;
    ok = ok && cudaMalloc((void**)&s.d_tab, s.tab_bytes) == cudaSuccess;
    s.in_cap = in_cap; s.out_cap = out_cap; s.work_cap = work_cap; s.tab_cap = tab_cap; s.ok = ok;
    if (!ok) { cudaGetLastError(); slot_free_raw(s); return false; }
    s.h_in = owner.h_in; s.h_out = owner.h_out; s.host_alias = true;
    return true;
}

void slot_free(Slot& s)
{
    if (s.host_alias) {
        // hand the borrowed buffers back (they belong to the owner slot); the device side goes to the pool as a device-only slot
        s.h_in = nullptr; s.h_out = nullptr; s.host_alias = false;
        if (s.ok) {
            cudaSetDevice(s.dev);
            if (s.stream) cudaStreamSynchronize(s.stream);
            std::lock_guard<std::mutex> g(g_pool_mu);
            if (g_pool.size() < kPoolMax && !getenv("ZSTDMT_B200_NO_POOL")) { g_pool.push_back(s); s = Slot(); return; }
        }
        slot_free_raw(s); return;
    }
    if (s.ok) {
        cudaSetDevice(s.dev);
        if (s.stream) cudaStreamSynchronize(s.stream);
        std::lock_guard<std::mutex> g(g_pool_mu);
        if (g_pool.size() < kPoolMax && !getenv("ZSTDMT_B200_NO_POOL")) { g_pool.push_back(s); s = Slot(); return; }
    }
    slot_free_raw(s);
}

bool slot_ensure_blocks(Slot& s, uint32_t cap)
{
    if (s.blk_cap >= cap) return true;
    cudaSetDevice(s.dev);
    if (s.h_blk) cudaFreeHost(s.h_blk);
    if (s.d_blk) cudaFree(s.d_blk);
    s.h_blk = s.d_blk = nullptr; s.blk_cap = 0;
    const size_t bytes = (size_t)cap * zmt_zstd_blk_desc_bytes();
    if (cudaHostAlloc((void**)&s.h_blk, bytes, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return false; }
    if (cudaMalloc((void**)&s.d_blk, bytes) != cudaSuccess) { cudaGetLastError(); return false; }
    s.blk_cap = cap;
    return true;
}

// ------------------------------------------------------------------ pipeline state shared by the 3 threads
struct Pipe {
    std::mutex mu;
    std::condition_variable cv;
    std::vector<Slot> slots;
    size_t fill_seq = 0, submit_seq = 0, write_seq = 0;
    bool reader_done = false;
    size_t error = 0;                 // first error wins
    void fail(size_t e) { std::lock_guard<std::mutex> g(mu); if (!error) error = e; cv.notify_all(); }
};

struct Ctx {
    int codec = 0, level = 0, threads = 0;
    size_t inputsize = 0;
    size_t insize = 0, outsize = 0, frames = 0, curframe = 0;
    bool is_comp = false;
    std::vector<int> devs;
    Pipe pipe;
    size_t lib_errcode = 0;
    const ErrCodes* E = nullptr;
};

void ctx_release_slots(Ctx* c)
{
    for (auto& s : c->pipe.slots) if (s.ok && s.host_alias) slot_free(s);         // borrowers before the owners of the host buffers
    for (auto& s : c->pipe.slots) if (s.ok) slot_free(s);
    c->pipe.slots.clear();
}

// ------------------------------------------------------------------ compression
size_t compress_run(Ctx* c, GenRdWr* rw)
{
    const DeviceRestore restore_device;
    const ErrCodes& E = *c->E;
    const CodecOps* ops = codec_ops(c->codec);
    if (!ops->compress || !ops->c_work || !ops->c_bound) { c->lib_errcode = ZMT_ST_UNSUPPORTED; return E.library; }
    Pipe& P = c->pipe;
    const size_t chunk = c->inputsize;
    // Slots in flight: the call is bound by the serialised callbacks (one memcpy stream); a GPU turns a batch around in a
    // fraction of the time the reader needs to fill the next one, so more devices do not need more slots per device — one each
    // is enough.  4 slots x 8 MiB measured best end to end on 2-socket Xeon hosts (not re-measured with an H100): a ring that
    // outgrows the last-level cache slows the callbacks' memcpy, and small batches pay the per-batch launch + copy latency.
    if (P.slots.empty()) {
        c->devs = env_devices();
        if (c->devs.empty()) { c->lib_errcode = ZMT_ST_CUDA; return E.library; }
    }
    const size_t base_slots = c->threads >= 4 ? 4 : c->threads >= 3 ? 3 : 2;
    size_t nsl = env_size("ZSTDMT_B200_SLOTS", base_slots > c->devs.size() ? base_slots : c->devs.size());
    if (nsl < 2) nsl = 2; if (nsl < c->devs.size()) nsl = c->devs.size(); if (nsl > 64) nsl = 64;
    size_t batch_bytes = env_size("ZSTDMT_B200_BATCH_MB", 8) << 20;
    const bool no_alias = getenv("ZSTDMT_B200_NO_RING_SHARE") != nullptr;          // A/B knob: every slot its own pinned buffers
    if (!no_alias && nsl > base_slots) nsl = (nsl + base_slots - 1) / base_slots * base_slots;   // batch q uses host buffer q % base_slots: needs base_slots | slots
    size_t B = batch_bytes / chunk; if (B < 1) B = 1; if (B > 65536) B = 65536;

    if (P.slots.empty()) {
        P.slots.resize(nsl);
        for (size_t i = 0; i < P.slots.size(); i++) {
            const size_t ic = B * chunk, oc = (size_t)ops->c_bound((uint32_t)B, (uint32_t)chunk), wc = ops->c_work((uint32_t)B, (uint32_t)chunk);
            const bool okk = (i < base_slots || no_alias) ? slot_alloc(P.slots[i], c->devs[i % c->devs.size()], ic, oc, wc, B)
                                                          : slot_alloc_alias(P.slots[i], P.slots[i % base_slots], c->devs[i % c->devs.size()], ic, oc, wc, B);
            if (!okk) { ctx_release_slots(c); return E.mem; }
        }
    }
    const size_t N = P.slots.size();
    // batches in flight: slots beyond the first `base_slots` borrow their pinned buffers from slot i % base_slots, so batch q + H
    // may only be filled once batch q has been written
    const size_t H = (N > base_slots && !no_alias) ? base_slots : N;
    P.fill_seq = P.submit_seq = P.write_seq = 0; P.reader_done = false; P.error = 0;
    for (auto& s : P.slots) s.state = 0;

    // ---- reader: fills slots in sequence order (pt_compress read section, lz4-mt_compress.c:255-277)
    StageClock ck_r, ck_w, ck_s;
    const CpuSet host_cpus = common_local_cpus(c->devs);
    std::thread reader([&]() {
        const ScopedAffinity bind(host_cpus);
        size_t frames_read = 0; bool eof = false;
        while (!eof) {
            Slot* s;
            {
                const double t0 = StageClock::now();
                std::unique_lock<std::mutex> lk(P.mu);
                s = &P.slots[P.fill_seq % N];
                P.cv.wait(lk, [&] { return (s->state == 0 && P.fill_seq - P.write_seq < H) || P.error; });
                ck_r.wait += StageClock::now() - t0;
                if (P.error) break;
            }
            Tables T = tables_at(s->h_tab, s->tab_cap);
            uint32_t n = 0; size_t got_bytes = 0;
            while (n < B) {
                GenBuffer b; b.buf = s->h_in + (size_t)n * chunk; b.size = chunk; b.allocated = chunk;
                const double t0 = StageClock::now();
                int rv = rw->fn_read(rw->arg_read, &b);
                ck_r.cb += StageClock::now() - t0;
                if (rv != 0) { P.fail(mt_error(E, rv)); eof = true; n = 0; break; }
                if (b.size > chunk) { P.fail(E.read_fail); eof = true; n = 0; break; }
                if (b.size == 0 && frames_read > 0) { eof = true; break; }
                T.d[n] = (uint32_t)b.size; got_bytes += b.size; frames_read++; n++;
            }
            if (n == 0) break;
            s->n = n; s->in_used = got_bytes;
            {
                std::lock_guard<std::mutex> g(P.mu);
                c->insize += got_bytes; c->frames += n;
                s->state = 1; P.fill_seq++;
            }
            P.cv.notify_all();
        }
        { std::lock_guard<std::mutex> g(P.mu); P.reader_done = true; }
        P.cv.notify_all();
    });

    // ---- writer: in-order emission (pt_write, lz4-mt_compress.c:178-205)
    std::thread writer([&]() {
        const ScopedAffinity bind(host_cpus);
        for (;;) {
            Slot* s;
            {
                const double t0 = StageClock::now();
                std::unique_lock<std::mutex> lk(P.mu);
                s = &P.slots[P.write_seq % N];
                P.cv.wait(lk, [&] { return s->state == 2 || P.error || (P.reader_done && P.write_seq == P.fill_seq); });
                ck_w.wait += StageClock::now() - t0;
                if (P.error || s->state != 2) break;
            }
            cudaSetDevice(s->dev);
            const double tg = StageClock::now();
            if (cudaEventSynchronize(s->ev) != cudaSuccess) { c->lib_errcode = ZMT_ST_CUDA; P.fail(E.library); break; }
            Tables T = tables_at(s->h_tab, s->tab_cap);
            const uint64_t total = T.a[s->n];
            if (total > s->out_cap) { c->lib_errcode = ZMT_ST_DST_SMALL; P.fail(E.library); break; }
            if (cudaMemcpyAsync(s->h_out, s->d_out, total, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess ||
                cudaStreamSynchronize(s->stream) != cudaSuccess) { c->lib_errcode = ZMT_ST_CUDA; P.fail(E.library); break; }
            ck_w.gpu += StageClock::now() - tg;
            bool bad = false;
            const double tc = StageClock::now();
            for (uint32_t i = 0; i < s->n; i++) {
                GenBuffer b; b.buf = s->h_out + T.a[i]; b.size = (size_t)(T.a[i + 1] - T.a[i]); b.allocated = b.size;
                int rv = rw->fn_write(rw->arg_write, &b);
                if (rv != 0) { P.fail(mt_error(E, rv)); bad = true; break; }
                c->outsize += b.size; c->curframe++;
            }
            ck_w.cb += StageClock::now() - tc;
            if (bad) break;
            { std::lock_guard<std::mutex> g(P.mu); s->state = 0; P.write_seq++; }
            P.cv.notify_all();
        }
    });

    // ---- submit (calling thread)
    for (;;) {
        Slot* s;
        {
            const double t0 = StageClock::now();
            std::unique_lock<std::mutex> lk(P.mu);
            s = &P.slots[P.submit_seq % N];
            P.cv.wait(lk, [&] { return s->state == 1 || P.error || (P.reader_done && P.submit_seq == P.fill_seq); });
            ck_s.wait += StageClock::now() - t0;
            if (P.error || s->state != 1) break;
        }
        const double ts = StageClock::now();
        cudaSetDevice(s->dev);
        Tables Th = tables_at(s->h_tab, s->tab_cap), Td = tables_at(s->d_tab, s->tab_cap);
        bool full = true;
        for (uint32_t i = 0; i < s->n; i++) if (Th.d[i] != chunk) { full = false; break; }
        cudaError_t ce = cudaSuccess;
        if (full) ce = cudaMemcpyAsync(s->d_in, s->h_in, (size_t)s->n * chunk, cudaMemcpyHostToDevice, s->stream);
        else for (uint32_t i = 0; i < s->n && ce == cudaSuccess; i++)
            if (Th.d[i]) ce = cudaMemcpyAsync(s->d_in + (size_t)i * chunk, s->h_in + (size_t)i * chunk, Th.d[i], cudaMemcpyHostToDevice, s->stream);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(Td.d, Th.d, (size_t)s->n * 4, cudaMemcpyHostToDevice, s->stream);
        int st = ZMT_ST_CUDA;
        if (ce == cudaSuccess) st = ops->compress(s->d_in, 0, (uint32_t)chunk, Td.d, s->n, s->d_work, s->d_out, Td.a, s->stream);
        if (s->dev >= 0 && s->dev < 64) g_dev_batches[s->dev]++;
        if (st == ZMT_ST_OK) {
            ce = cudaMemcpyAsync(Th.a, Td.a, ((size_t)s->n + 1) * 8, cudaMemcpyDeviceToHost, s->stream);
            if (ce == cudaSuccess) ce = cudaEventRecord(s->ev, s->stream);
            if (ce != cudaSuccess) st = ZMT_ST_CUDA;
        }
        if (st != ZMT_ST_OK) { c->lib_errcode = (size_t)st; P.fail(E.library); break; }
        ck_s.gpu += StageClock::now() - ts;
        { std::lock_guard<std::mutex> g(P.mu); s->state = 2; P.submit_seq++; }
        P.cv.notify_all();
    }
    reader.join(); writer.join();
    for (auto& s : P.slots) { cudaSetDevice(s.dev); cudaStreamSynchronize(s.stream); }
    if (trace_on())
        fprintf(stderr, "[zstdmt_b200] compress: reader cb %.3fs wait %.3fs | submit enqueue %.3fs wait %.3fs | writer gpu-wait %.3fs cb %.3fs wait %.3fs | slots %zu x %zu chunks\n",
                ck_r.cb, ck_r.wait, ck_s.gpu, ck_s.wait, ck_w.gpu, ck_w.cb, ck_w.wait, N, B);
    return P.error;
}

// ------------------------------------------------------------------ decompression
// Output size of one payload, from its own header (pt_decompress sizes the buffer from
// LE64 @ payload+6, lz4-mt_decompress.c:329-335; zstd: frame content size).
// Returns false if the header is unusable.
bool lz4f_out_size(const uint8_t* p, size_t n, uint64_t* out)
{
    if (n < 7 || rd32(p) != LZ4F_MAGIC) { *out = 0; return true; }     // the device decoder reports the precise status
    const uint32_t flg = p[4], bd = p[5];
    if (flg & 0x08) {
        if (n < 15) return false;
        // untrusted field: LZ4 cannot expand by more than 255x, anything larger is a corrupt header (the reference
        // fails its malloc there); without this bound a huge value would wrap the running output offsets
        const uint64_t v = rd64(p + 6);
        if (v > (uint64_t)n * 255 + 65536) return false;
        *out = v; return true;
    }
    // no content-size field: bound it by walking the block headers (each block <= blockMaxSize)
    const uint32_t id = (bd >> 4) & 7; if (id < 4) return false;
    const uint64_t blkmax = 1ull << (8 + 2 * id);
    size_t pos = 4 + 2 + ((flg & 1) ? 4 : 0) + 1; uint64_t total = 0;
    while (pos + 4 <= n) {
        const uint32_t bh = rd32(p + pos); pos += 4;
        if (bh == 0) break;
        const uint32_t bs = bh & 0x7FFFFFFFu;
        total += (bh & 0x80000000u) ? bs : blkmax;
        pos += (size_t)bs + ((flg & 0x10) ? 4 : 0);
    }
    *out = total; return true;
}

// reads exactly `want` bytes unless EOF; returns 0 ok / error; *got = delivered
size_t read_some(const ErrCodes& E, GenRdWr* rw, void* dst, size_t want, size_t* got)
{
    GenBuffer b; b.buf = dst; b.size = want; b.allocated = want;
    int rv = rw->fn_read(rw->arg_read, &b);
    if (rv != 0) return mt_error(E, rv);
    if (b.size > want) return E.read_fail;
    *got = b.size; return 0;
}

// ------------------------------------------------------------------ plain (unframed) single streams
// What the reference routes to st_decompress (lz4-mt_decompress.c:391-483, zstd-mt_decompress.c:552-687): an ordinary
// .lz4 / .zst file, i.e. codec frames back to back without the 12-byte size headers.  Frame lengths are only known after
// walking the block headers, so the host reads ahead, cuts the bytes it holds into complete frames, and decodes them in
// batches of at most ~kPlainBatch input bytes with the same GPU kernels; the consumed bytes are dropped before the next
// read, so memory is bounded by the batch size or by the largest single frame, whichever is larger (the reference streams
// through two fixed buffers; a frame here must fit in host and device memory as a whole).  `first`/`have` = the bytes
// already consumed by the stream-type sniffing.
struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    ~DevBuf() { if (p) cudaFree(p); }
    bool need(size_t n) {                                   // grow-only
        if (n <= cap && p) return true;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        const size_t want = n + n / 4 + 4096;
        if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); if (cudaMalloc(&p, n ? n : 1) != cudaSuccess) { cudaGetLastError(); p = nullptr; return false; } cap = n; return true; }
        cap = want; return true;
    }
};

size_t decompress_single_stream(Ctx* c, GenRdWr* rw, const uint8_t* first, size_t have)
{
    const ErrCodes& E = *c->E;
    const bool is_zstd = c->codec == CODEC_ZSTD;
    const size_t kPlainBatch = env_size("ZSTDMT_B200_PLAIN_MB", 64) << 20;
    const size_t piece = c->inputsize < (64u << 10) ? (size_t)1 << 20 : c->inputsize;
    const size_t dsz = zmt_zstd_blk_desc_bytes();
    std::vector<uint8_t> in(12, 0);                         // 12 pad bytes: the LZ4 kernel addresses a frame as base + off + 12
    in.insert(in.end(), first, first + have);
    bool eof = false;
    size_t pos = 0;                                         // parse position inside in[12..]
    const std::vector<int> devs = env_devices();
    if (devs.empty() || cudaSetDevice(devs[0]) != cudaSuccess) { c->lib_errcode = ZMT_ST_CUDA; return E.library; }
    DevBuf d_in, d_out, d_tab, d_blk, d_work;
    cudaStream_t st = nullptr;
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { c->lib_errcode = ZMT_ST_CUDA; return E.library; }
    struct StreamGuard { cudaStream_t s; ~StreamGuard() { cudaStreamDestroy(s); } } guard{st};
    std::vector<uint8_t> out, blocks, h_tab;
    std::vector<uint64_t> foff, ooff, expect; std::vector<uint32_t> fcs, first_blk, fflags;
    c->insize = have;

    for (;;) {
        // ---- cut complete frames out of what we hold, up to one batch
        foff.clear(); ooff.assign(1, 0); expect.clear(); fcs.clear(); first_blk.assign(1, 0); fflags.clear();
        uint32_t nblk = 0; uint64_t scratch = 0, nslots = 0;
        const size_t batch_start = pos;
        bool need_more = false;
        while (!need_more) {
            const uint8_t* s = in.data() + 12; const size_t n = in.size() - 12;
            if (pos >= n) { need_more = !eof; break; }
            if (!foff.empty() && pos - batch_start >= kPlainBatch) break;
            if (n - pos < 4) { if (eof) return E.data_error; need_more = true; break; }
            const uint32_t magic = rd32(s + pos);
            if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {          // skippable frame: magic, LE32 size, payload
                if (n - pos < 8 || n - pos - 8 < rd32(s + pos + 4)) { if (eof) return E.data_error; need_more = true; break; }
                pos += 8 + (size_t)rd32(s + pos + 4); continue;
            }
            if (!is_zstd) {
                if (magic != LZ4F_MAGIC) return E.data_error;
                if (n - pos < 7) { if (eof) return E.data_error; need_more = true; break; }
                const uint32_t flg = s[pos + 4], bd = s[pos + 5], id = (bd >> 4) & 7;
                if ((flg >> 6) != 1 || id < 4) { c->lib_errcode = ZMT_ST_BAD_HEADER; return E.library; }
                const uint64_t blkmax = 1ull << (8 + 2 * id);
                size_t q = pos + 4 + 2 + ((flg & 8) ? 8 : 0) + ((flg & 1) ? 4 : 0) + 1;
                uint64_t bound = 0; bool cut = false;
                for (;;) {
                    if (q + 4 > n) { cut = true; break; }
                    const uint32_t bh = rd32(s + q); q += 4;
                    if (bh == 0) break;
                    const uint32_t bs = bh & 0x7FFFFFFFu;
                    bound += (bh & 0x80000000u) ? bs : blkmax;
                    q += (size_t)bs + ((flg & 0x10) ? 4 : 0);
                }
                if (!cut && (flg & 4)) q += 4;
                if (cut || q > n) { if (eof) { c->lib_errcode = ZMT_ST_TRUNCATED; return E.frame_decompress; } need_more = true; break; }
                uint64_t osz = bound;
                if (flg & 8) { osz = rd64(s + pos + 6); if (osz > bound) { c->lib_errcode = ZMT_ST_CONTENT_SIZE; return E.library; } }    // untrusted field, bounded by the block walk
                foff.push_back(pos); fcs.push_back((uint32_t)(q - pos)); ooff.push_back(ooff.back() + osz);
                { const uint64_t nb = (osz + 65535) / 65536; nslots += nb ? nb : 1; }
                pos = q;
            } else {
                if (magic < 0xFD2FB522u || magic > 0xFD2FB528u) return E.data_error;
                uint64_t cs = 0; uint32_t fl = 0; size_t used = 0;
                const uint32_t nblk0 = nblk; const uint64_t scr0 = scratch;
                int zr;
                for (;;) {
                    nblk = nblk0; scratch = scr0;
                    zr = zmt_zstd_scan_frame_host2(s + pos, n - pos, 12 + pos, (uint32_t)foff.size(), blocks.data(), &nblk, (uint32_t)(blocks.size() / dsz), &scratch, &cs, &fl, &used);
                    if (zr != ZMT_ST_DST_SMALL) break;
                    blocks.resize(blocks.size() * 2 + 4096 * dsz);            // block table full: grow and rescan this frame
                }
                if (zr == ZMT_ST_TRUNCATED && !eof) { nblk = nblk0; scratch = scr0; need_more = true; break; }
                if (zr != ZMT_ST_OK) { c->lib_errcode = (size_t)zr; return zr == ZMT_ST_TRUNCATED ? E.frame_decompress : E.library; }
                foff.push_back(pos); expect.push_back((fl & 4u) ? ~0ull : cs); fflags.push_back(fl); first_blk.push_back(nblk); ooff.push_back(ooff.back() + cs);
                pos += used;
            }
        }
        const uint32_t nf = (uint32_t)foff.size();
        if (nf == 0) {
            if (!need_more) break;                                            // EOF, everything consumed
        } else {
            // ---- decode this batch
            const uint64_t total = ooff.back();
            const size_t in_bytes = pos + 12;                                   // frames address the buffer from its 12-byte pad
            const size_t tab_bytes = tables_bytes(nf);
            h_tab.resize(tab_bytes);
            Tables T = tables_at(h_tab.data(), nf);
            for (uint32_t i = 0; i < nf; i++) { T.a[i] = foff[i]; T.b[i] = ooff[i]; if (is_zstd) { T.f[i] = expect[i]; T.d[i] = fflags[i]; T.g[i] = first_blk[i]; } else T.d[i] = fcs[i]; }
            T.b[nf] = total; if (is_zstd) T.g[nf] = nblk;
            const size_t wk = is_zstd ? zmt_zstdd_workspace_bytes(nf, nblk, scratch) : zmt_lz4d_workspace_bytes(nf, (uint32_t)nslots, in_bytes);
            if (!d_in.need(in_bytes + 256) || !d_out.need(total + 256) || !d_tab.need(tab_bytes) || !d_work.need(wk) || (is_zstd && !d_blk.need((size_t)nblk * dsz + 16))) return E.mem;
            Tables Td = tables_at((uint8_t*)d_tab.p, nf);
            // only the bytes of this batch travel (the device addresses them at their buffer offsets)
            const size_t lo = 12 + batch_start, hi = in_bytes;
            cudaMemcpyAsync((uint8_t*)d_in.p + lo, in.data() + lo, hi - lo, cudaMemcpyHostToDevice, st);
            cudaMemcpyAsync(d_tab.p, h_tab.data(), tab_bytes, cudaMemcpyHostToDevice, st);
            if (is_zstd && nblk) cudaMemcpyAsync(d_blk.p, blocks.data(), (size_t)nblk * dsz, cudaMemcpyHostToDevice, st);
            const int rc = is_zstd ? zmt_zstd_decompress_device(d_in.p, d_blk.p, nblk, Td.g, Td.f, Td.d, nf, d_out.p, Td.b, Td.c, Td.e, d_work.p, st)
                                   : zmt_lz4_decompress_device(d_in.p, in_bytes, Td.a, Td.d, nf, (uint32_t)nslots, d_out.p, Td.b, Td.c, Td.e, d_work.p, st);
            out.resize(total ? total : 1);
            std::vector<uint32_t> status(nf); std::vector<uint64_t> osz(nf);
            cudaError_t ce = cudaSuccess;
            if (rc == ZMT_ST_OK) {
                if (total) ce = cudaMemcpyAsync(out.data(), d_out.p, total, cudaMemcpyDeviceToHost, st);
                if (ce == cudaSuccess) ce = cudaMemcpyAsync(status.data(), Td.e, (size_t)nf * 4, cudaMemcpyDeviceToHost, st);
                if (ce == cudaSuccess) ce = cudaMemcpyAsync(osz.data(), Td.c, (size_t)nf * 8, cudaMemcpyDeviceToHost, st);
                if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
            }
            if (rc != ZMT_ST_OK || ce != cudaSuccess) { cudaGetLastError(); c->lib_errcode = ZMT_ST_CUDA; return E.library; }
            for (uint32_t i = 0; i < nf; i++) {
                if (status[i] != ZMT_ST_OK) { c->lib_errcode = status[i]; return (status[i] == ZMT_ST_TRUNCATED || status[i] == ZMT_ST_TRAILING) ? E.frame_decompress : E.library; }
                // frame by frame, in pieces of at most `piece` bytes (st_decompress writes as it goes)
                uint64_t o = 0;
                while (o < osz[i]) {
                    GenBuffer b; b.buf = out.data() + ooff[i] + o; b.size = (size_t)((osz[i] - o) < piece ? (osz[i] - o) : piece); b.allocated = b.size;
                    const size_t want = b.size;
                    const int rv = rw->fn_write(rw->arg_write, &b);
                    if (rv != 0) return mt_error(E, rv);
                    c->outsize += b.size; o += want;
                }
            }
            // drop what has been decoded
            in.erase(in.begin() + 12, in.begin() + 12 + (long)pos);
            pos = 0;
        }
        if (need_more) {
            // ---- read ahead: at least one more piece, up to a batch beyond the parse position
            size_t goal = in.size() + piece;
            if (goal < 12 + pos + kPlainBatch) goal = 12 + pos + kPlainBatch;
            if (in.size() - 12 - pos >= kPlainBatch) goal = in.size() + (in.size() - 12 - pos) / 2;     // one frame larger than a batch: read ahead geometrically
            while (!eof && in.size() < goal) {
                const size_t old = in.size();
                in.resize(old + piece);
                size_t got = 0;
                const size_t e = read_some(E, rw, in.data() + old, piece, &got);
                in.resize(old + got);
                if (e) return e;
                c->insize += got;
                if (got == 0) eof = true;
            }
        } else if (eof && pos >= in.size() - 12) break;
    }
    return 0;
}

size_t decompress_run(Ctx* c, GenRdWr* rw)
{
    const DeviceRestore restore_device;
    const ErrCodes& E = *c->E;
    Pipe& P = c->pipe;
    const bool is_zstd = c->codec == CODEC_ZSTD;
    const uint32_t kBlkCap = 32768;
    // decode batches must hold enough frames to fill the GPU (one warp per 64 KiB block; a linked-block frame is a chain)
    const size_t in_cap0 = (env_size("ZSTDMT_B200_DBATCH_MB", 32) << 20), out_cap0 = in_cap0 * 2, tab_cap = 8192;
    const uint64_t piece_bytes = (uint64_t)env_size("ZSTDMT_B200_D2H_PIECE_MB", 2) << 20;      // 0: whole slot right after the kernels

    // ---- stream-type sniffing on the calling thread (LZ4MT_decompressDCtx, lz4-mt_decompress.c:503-520;
    //      ZSTDCB_decompressDCtx, zstd-mt_decompress.c:721-759)
    uint8_t first[16]; size_t have = 0, got = 0;
    bool hdr_pending = false;                 // first 12-byte header already (partly) read into `first`
    size_t first_payload_have = 0;            // zstd pzstd-style: 4 payload bytes already read
    if (c->codec == CODEC_LZ4) {
        size_t e = read_some(E, rw, first, 4, &got); if (e) return e;
        if (got != 4) return E.data_error;
        if (rd32(first) != MT_MAGIC_SKIPPABLE) {
            if (rd32(first) != LZ4F_MAGIC) return E.data_error;
            return decompress_single_stream(c, rw, first, 4);          // plain .lz4 stream (st_decompress, lz4-mt_decompress.c:512-520)
        }
        e = read_some(E, rw, first + 4, 8, &got); if (e) return e;
        if (got != 8) return E.read_fail;
        have = 12; hdr_pending = true;
    } else {
        size_t e = read_some(E, rw, first, 16, &got); if (e) return e;
        have = got;
        auto is_zstd = [](const uint8_t* p) { uint32_t m = rd32(p); return m >= 0xFD2FB522u && m <= 0xFD2FB528u; };
        auto is_skip = [](const uint8_t* p) { return rd32(p) == MT_MAGIC_SKIPPABLE && rd32(p + 4) == 4; };
        if (have < 16) {
            if (have < 4 || !is_zstd(first)) return E.data_error;
            if (have == 9) return 0;                                   // empty file (zstd-mt_decompress.c:735-740)
            return decompress_single_stream(c, rw, first, have);       // short plain zstd stream
        }
        c->insize += 16;
        if (is_skip(first) && is_zstd(first + 12)) { hdr_pending = true; first_payload_have = 4; }          // pzstd style
        else if (is_zstd(first) && rd32(first + 9) == MT_MAGIC_SKIPPABLE) {                                    // zstdmt style: 9-byte empty frame + 12-byte header
            // (only the magic can be tested here, as IsZstd_Skippable does, zstd-mt_decompress.c:156-159: 7 of the header's 12
            //  bytes are in hand; the size field is checked with the assembled header.  Round 1 read its 4 bytes past the buffer.)
            uint8_t tmp[12]; memcpy(tmp, first + 9, 7);
            size_t e2 = read_some(E, rw, tmp + 7, 5, &got); if (e2) return e2;
            if (got != 5) return E.data_error;
            c->insize += 5; memcpy(first, tmp, 12); hdr_pending = true; first_payload_have = 0;
        } else if (is_zstd(first)) return decompress_single_stream(c, rw, first, have);    // plain .zst (zstd-mt_decompress.c:747-752)
        else return E.data_error;
    }

    if (P.slots.empty()) {
        c->devs = env_devices();
        if (c->devs.empty()) { c->lib_errcode = ZMT_ST_CUDA; return E.library; }
        const size_t base_slots = c->threads >= 4 ? 4 : c->threads >= 3 ? 3 : 2;       // see compress_run
        P.slots.resize(base_slots > c->devs.size() ? base_slots : c->devs.size());
        for (size_t i = 0; i < P.slots.size(); i++)
        {
            // zstd scratch: 16 B per sequence + the literals: ~2x the output on text, bounded at 3x + tables (the reader closes a batch early otherwise)
            const size_t wk = is_zstd ? zmt_zstdd_workspace_bytes((uint32_t)tab_cap, kBlkCap, 3 * (uint64_t)out_cap0) : zmt_lz4d_workspace_bytes((uint32_t)tab_cap, lz4_slot_cap(out_cap0, tab_cap), in_cap0);
            if (!slot_alloc(P.slots[i], c->devs[i % c->devs.size()], in_cap0, out_cap0, wk, tab_cap) || (is_zstd && !slot_ensure_blocks(P.slots[i], kBlkCap))) { ctx_release_slots(c); return E.mem; }
            P.slots[i].scr_cap = is_zstd ? 3 * (uint64_t)P.slots[i].out_cap : 0;
        }
    }
    const size_t N = P.slots.size();
    P.fill_seq = P.submit_seq = P.write_seq = 0; P.reader_done = false; P.error = 0;
    for (auto& s : P.slots) s.state = 0;

    StageClock rd_clk, wr_clk; double rd_scan = 0, rd_total = 0, wr_total = 0;     // ZSTDMT_B200_TRACE=1
    const bool tr = trace_on();
    // ---- reader (pt_read, lz4-mt_decompress.c:192-281 / zstd-mt_decompress.c:209-369)
    const CpuSet host_cpus = common_local_cpus(c->devs);
    std::thread reader([&]() {
        const ScopedAffinity bind(host_cpus);
        const double t_start = tr ? StageClock::now() : 0;
        bool eof = false;
        std::vector<uint8_t> carry;              // a frame that did not fit the previous slot
        uint64_t carry_out = 0;
        while (!eof) {
            Slot* s;
            {
                std::unique_lock<std::mutex> lk(P.mu);
                s = &P.slots[P.fill_seq % N];
                const double t0 = tr ? StageClock::now() : 0;
                P.cv.wait(lk, [&] { return s->state == 0 || P.error; });
                if (tr) rd_clk.wait += StageClock::now() - t0;
                if (P.error) break;
            }
            Tables T = tables_at(s->h_tab, s->tab_cap);
            uint32_t n = 0; size_t in_used = 0; uint64_t out_used = 0; size_t stat_in = 0;
            bool failed = false;
            uint32_t nblk = 0; uint64_t scr = 0;                 // zstd: block descriptors + scratch demand of this batch
            // (re)allocate the still empty slot so that one frame of these dimensions fits; takes P.mu for the swap because the
            // writer's wait predicate reads s->state
            auto grow = [&](size_t need_in, uint64_t need_out, uint64_t need_scr, uint32_t need_blk) -> bool {
                if (need_in <= s->in_cap && need_out <= s->out_cap && need_scr <= s->scr_cap && need_blk <= s->blk_cap) return true;
                const int dev = s->dev;
                const size_t nin = need_in > s->in_cap ? need_in : s->in_cap, nout = need_out > s->out_cap ? (size_t)need_out : s->out_cap;
                const uint64_t nscr = is_zstd ? (need_scr > 3 * (uint64_t)nout ? need_scr : 3 * (uint64_t)nout) : 0;
                const uint32_t nb = need_blk > s->blk_cap ? need_blk : s->blk_cap;
                const size_t tc = s->tab_cap;
                const size_t wk = is_zstd ? zmt_zstdd_workspace_bytes((uint32_t)tc, nb, nscr) : zmt_lz4d_workspace_bytes((uint32_t)tc, lz4_slot_cap(nout, tc), nin);
                std::lock_guard<std::mutex> g(P.mu);
                slot_free(*s);
                if (!slot_alloc(*s, dev, nin, nout, wk, tc) || (is_zstd && !slot_ensure_blocks(*s, nb))) return false;
                s->scr_cap = nscr;
                return true;
            };
            // Put one whole frame (12-byte header + payload, held in `fr`) at the start of the empty slot, growing the slot
            // (input, output, zstd block table and entropy scratch) until it fits.  Returns false after P.fail().
            auto place_first = [&](const std::vector<uint8_t>& fr) -> bool {
                const size_t toRead = fr.size() - 12;
                if (!grow(fr.size(), 0, 0, 0)) { P.fail(E.mem); return false; }
                uint64_t osz = 0; uint32_t nsq = 0;
                if (!is_zstd) {
                    if (!lz4f_out_size(fr.data() + 12, toRead, &osz)) { c->lib_errcode = ZMT_ST_BAD_HEADER; P.fail(E.library); return false; }
                    if (!grow(fr.size(), osz, 0, 0)) { P.fail(E.mem); return false; }
                    memcpy(s->h_in, fr.data(), fr.size());
                } else {
                    for (int tries = 0;; tries++) {
                        memcpy(s->h_in, fr.data(), fr.size());
                        uint64_t cs = 0; nblk = 0; scr = 0;
                        const int zr = zmt_zstd_scan_frame_host(s->h_in + 12, toRead, 12, 0, s->h_blk, &nblk, s->blk_cap, &scr, &cs, &nsq);
                        if (zr == ZMT_ST_DST_SMALL && tries < 2) {          // more blocks than descriptors: every block costs >= 3 bytes
                            if (!grow(fr.size(), 0, 0, (uint32_t)(toRead / 3 + 16))) { P.fail(E.mem); return false; }
                            continue;
                        }
                        if (zr != ZMT_ST_OK) { c->lib_errcode = (size_t)zr; P.fail(zr == ZMT_ST_TRUNCATED || zr == ZMT_ST_TRAILING ? E.frame_decompress : E.library); return false; }
                        osz = cs;
                        if (osz <= s->out_cap && scr <= s->scr_cap) break;
                        if (tries >= 2 || !grow(fr.size(), osz, scr, 0)) { P.fail(E.mem); return false; }
                    }
                }
                T = tables_at(s->h_tab, s->tab_cap);
                T.a[0] = 0; T.d[0] = (uint32_t)toRead; T.b[0] = 0;
                if (is_zstd) { T.g[0] = 0; T.f[0] = (nsq & 4u) ? ~0ull : osz; T.d[0] = nsq; }      // flag 4: no content size in the header, osz is a bound
                in_used = fr.size(); out_used = osz; n = 1;
                return true;
            };
            if (!carry.empty()) {
                if (!place_first(carry)) break;
                carry.clear();
            }
            while (n < s->tab_cap) {
                uint8_t hdr[12]; size_t pre = 0;
                if (hdr_pending) { memcpy(hdr, first, 12); hdr_pending = false; pre = first_payload_have; }
                else {
                    size_t g = 0; size_t e = read_some(E, rw, hdr, 12, &g);
                    if (e) { P.fail(e); failed = true; break; }
                    if (g == 0) { eof = true; break; }
                    if (g != 12) { P.fail(E.read_fail); failed = true; break; }
                    if (rd32(hdr) != MT_MAGIC_SKIPPABLE) { P.fail(E.data_error); failed = true; break; }
                    if (c->codec == CODEC_ZSTD) stat_in += 12;
                }
                if (rd32(hdr + 4) != 4) { P.fail(E.data_error); failed = true; break; }
                if (c->codec == CODEC_LZ4) stat_in += 12;
                const size_t toRead = rd32(hdr + 8);
                if (toRead < pre) { P.fail(E.data_error); failed = true; break; }
                // where to put it: the current slot if it fits behind the frames already there, else a temporary buffer
                // (first frame of a batch that needs a bigger slot, or a frame that moves to the next batch)
                uint8_t* dstp; bool to_tmp = false;
                if (in_used + 12 + toRead <= s->in_cap) dstp = s->h_in + in_used;
                else { carry.resize(12 + toRead); dstp = carry.data(); to_tmp = true; }
                memcpy(dstp, hdr, 12);
                if (pre) memcpy(dstp + 12, first + 12, pre);
                const double tc0 = tr ? StageClock::now() : 0;
                size_t g = 0; size_t e = read_some(E, rw, dstp + 12 + pre, toRead - pre, &g);
                if (tr) rd_clk.cb += StageClock::now() - tc0;
                if (e) { P.fail(e); failed = true; break; }
                if (g != toRead - pre) { P.fail(E.data_error); failed = true; break; }
                stat_in += g;
                if (to_tmp) {
                    if (n > 0) break;                                   // next batch starts with it
                    if (!place_first(carry)) { failed = true; break; }
                    carry.clear();
                    continue;
                }
                uint64_t osz = 0; uint32_t nsq = 0;
                uint32_t nblk_new = nblk; uint64_t scr_new = scr;
                bool moves = false;                                     // does not fit behind the others: first frame of the next batch
                if (!is_zstd) {
                    if (!lz4f_out_size(dstp + 12, toRead, &osz)) { c->lib_errcode = ZMT_ST_BAD_HEADER; P.fail(E.library); failed = true; break; }
                } else {
                    // block table of this frame (descriptors are appended; dropped again if the frame moves to the next batch)
                    uint64_t cs = 0;
                    const double ts0 = tr ? StageClock::now() : 0;
                    const int zr = zmt_zstd_scan_frame_host(dstp + 12, toRead, in_used + 12, n, s->h_blk, &nblk_new, s->blk_cap, &scr_new, &cs, &nsq);
                    if (tr) rd_scan += StageClock::now() - ts0;
                    if (zr == ZMT_ST_DST_SMALL) moves = true;
                    else if (zr != ZMT_ST_OK) { c->lib_errcode = (size_t)zr; P.fail(zr == ZMT_ST_TRUNCATED || zr == ZMT_ST_TRAILING ? E.frame_decompress : E.library); failed = true; break; }
                    else if (scr_new > s->scr_cap) moves = true;
                    osz = cs;
                }
                if (!moves && osz > s->out_cap - out_used) moves = true;
                if (moves) {
                    carry.assign(dstp, dstp + 12 + toRead);
                    if (n > 0) break;
                    if (!place_first(carry)) { failed = true; break; }  // a single frame larger than the slot: grow the slot
                    carry.clear();
                    continue;
                }
                T.a[n] = in_used; T.d[n] = (uint32_t)toRead; T.b[n] = out_used;
                if (is_zstd) { T.g[n] = nblk; T.f[n] = (nsq & 4u) ? ~0ull : osz; T.d[n] = nsq; nblk = nblk_new; scr = scr_new; }     // T.d = frame flags (sequential pass, checksum, no size)
                in_used += 12 + toRead; out_used += osz; n++;
            }
            if (failed) break;
            if (n == 0) break;
            T.b[n] = out_used;
            if (is_zstd) { T.g[n] = nblk; s->nblk = nblk; s->scratch_used = scr; }
            s->n = n; s->in_used = in_used; s->out_used = (size_t)out_used;
            { uint64_t ns = 0; for (uint32_t i = 0; i < n; i++) { const uint64_t nb = (T.b[i + 1] - T.b[i] + 65535) / 65536; ns += nb ? nb : 1; } s->nslots = (uint32_t)ns; }
            {
                std::lock_guard<std::mutex> g(P.mu);
                c->insize += stat_in; c->frames += n;
                s->state = 1; P.fill_seq++;
            }
            P.cv.notify_all();
        }
        if (tr) rd_total = StageClock::now() - t_start;
        { std::lock_guard<std::mutex> g(P.mu); P.reader_done = true; }
        P.cv.notify_all();
    });

    // ---- writer (pt_write, lz4-mt_decompress.c:165-187)
    std::thread writer([&]() {
        const ScopedAffinity bind(host_cpus);
        const double t_start = tr ? StageClock::now() : 0;
        for (;;) {
            Slot* s;
            {
                std::unique_lock<std::mutex> lk(P.mu);
                s = &P.slots[P.write_seq % N];
                const double t0 = tr ? StageClock::now() : 0;
                P.cv.wait(lk, [&] { return s->state == 2 || P.error || (P.reader_done && P.write_seq == P.fill_seq); });
                if (tr) wr_clk.wait += StageClock::now() - t0;
                if (P.error || s->state != 2) break;
            }
            cudaSetDevice(s->dev);
            const double tg0 = tr ? StageClock::now() : 0;
            if (cudaEventSynchronize(s->ev) != cudaSuccess) { c->lib_errcode = ZMT_ST_CUDA; P.fail(E.library); break; }
            if (tr) wr_clk.gpu += StageClock::now() - tg0;
            Tables T = tables_at(s->h_tab, s->tab_cap);
            bool bad = false;
            // The decoded bytes come over in pieces of a few MiB, one piece ahead of the one being written: what fn_write's
            // memcpy reads was DMA-written moments ago and is still in the last-level cache, instead of a whole 64 MiB slot that
            // was copied long before its first byte is used.
            uint32_t issued = 0, ready = 0; int np_issued = 0, np_ready = 0;       // frames [0, issued) requested, [0, ready) landed
            auto issue_piece = [&]() -> bool {
                if (issued >= s->n) return true;
                uint32_t j = issued; uint64_t lo = T.b[j], hi = lo;
                while (j < s->n && hi - lo < piece_bytes) { hi = T.b[j] + T.c[j]; j++; }
                if (hi > s->out_cap) hi = s->out_cap;
                if (hi > lo && cudaMemcpyAsync(s->h_out + lo, s->d_out + lo, (size_t)(hi - lo), cudaMemcpyDeviceToHost, s->stream) != cudaSuccess) return false;
                if (cudaEventRecord(s->evp[np_issued & 1], s->stream) != cudaSuccess) return false;
                np_issued++; issued = j;
                return true;
            };
            uint32_t piece_end[2] = { 0, 0 };
            for (uint32_t i = 0; i < s->n; i++) {
                const uint32_t st = T.e[i];
                if (st != ZMT_ST_OK) {
                    c->lib_errcode = st;
                    P.fail((st == ZMT_ST_TRUNCATED || st == ZMT_ST_TRAILING) ? E.frame_decompress : E.library);
                    bad = true; break;
                }
                if (piece_bytes && i >= ready) {
                    bool okp = true;
                    if (np_issued == np_ready) { okp = issue_piece(); piece_end[(np_issued - 1) & 1] = issued; }
                    if (okp && issued < s->n && np_issued == np_ready + 1) { okp = issue_piece(); piece_end[(np_issued - 1) & 1] = issued; }   // one ahead
                    if (okp) okp = cudaEventSynchronize(s->evp[np_ready & 1]) == cudaSuccess;
                    if (!okp) { c->lib_errcode = ZMT_ST_CUDA; P.fail(E.library); bad = true; break; }
                    ready = piece_end[np_ready & 1]; np_ready++;
                }
                GenBuffer b; b.buf = s->h_out + T.b[i]; b.size = (size_t)T.c[i]; b.allocated = b.size;
                const double tc0 = tr ? StageClock::now() : 0;
                int rv = rw->fn_write(rw->arg_write, &b);
                if (tr) wr_clk.cb += StageClock::now() - tc0;
                if (rv != 0) { P.fail(mt_error(E, rv)); bad = true; break; }
                c->outsize += b.size; c->curframe++;
            }
            if (bad) break;
            { std::lock_guard<std::mutex> g(P.mu); s->state = 0; P.write_seq++; }
            P.cv.notify_all();
        }
    });

    // ---- submit
    for (;;) {
        Slot* s;
        {
            std::unique_lock<std::mutex> lk(P.mu);
            s = &P.slots[P.submit_seq % N];
            P.cv.wait(lk, [&] { return s->state == 1 || P.error || (P.reader_done && P.submit_seq == P.fill_seq); });
            if (P.error || s->state != 1) break;
        }
        cudaSetDevice(s->dev);
        Tables Th = tables_at(s->h_tab, s->tab_cap), Td = tables_at(s->d_tab, s->tab_cap);
        cudaError_t ce = cudaMemcpyAsync(s->d_in, s->h_in, s->in_used, cudaMemcpyHostToDevice, s->stream);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(s->d_tab, s->h_tab, s->tab_bytes, cudaMemcpyHostToDevice, s->stream);
        int st = ZMT_ST_CUDA;
        if (ce == cudaSuccess && is_zstd && s->nblk) ce = cudaMemcpyAsync(s->d_blk, s->h_blk, (size_t)s->nblk * zmt_zstd_blk_desc_bytes(), cudaMemcpyHostToDevice, s->stream);
        if (ce == cudaSuccess) st = is_zstd ? zmt_zstd_decompress_device(s->d_in, s->d_blk, s->nblk, Td.g, Td.f, Td.d, s->n, s->d_out, Td.b, Td.c, Td.e, s->d_work, s->stream)
                                            : zmt_lz4_decompress_device(s->d_in, s->in_used, Td.a, Td.d, s->n, s->nslots, s->d_out, Td.b, Td.c, Td.e, s->d_work, s->stream);
        if (s->dev >= 0 && s->dev < 64) g_dev_batches[s->dev]++;
        if (st == ZMT_ST_OK) {
            if (s->out_used && piece_bytes == 0) ce = cudaMemcpyAsync(s->h_out, s->d_out, s->out_used, cudaMemcpyDeviceToHost, s->stream);
            if (ce == cudaSuccess) ce = cudaMemcpyAsync(Th.c, Td.c, (size_t)s->n * 8, cudaMemcpyDeviceToHost, s->stream);
            if (ce == cudaSuccess) ce = cudaMemcpyAsync(Th.e, Td.e, (size_t)s->n * 4, cudaMemcpyDeviceToHost, s->stream);
            if (ce == cudaSuccess) ce = cudaEventRecord(s->ev, s->stream);
            if (ce != cudaSuccess) st = ZMT_ST_CUDA;
        }
        if (st != ZMT_ST_OK) { c->lib_errcode = (size_t)st; P.fail(E.library); break; }
        { std::lock_guard<std::mutex> g(P.mu); s->state = 2; P.submit_seq++; }
        P.cv.notify_all();
    }
    reader.join(); writer.join();
    for (auto& s : P.slots) { if (s.ok) { cudaSetDevice(s.dev); cudaStreamSynchronize(s.stream); } }
    if (tr)
        fprintf(stderr, "[zstdmt_b200] decompress: reader total %.3fs cb %.3fs scan %.3fs wait %.3fs | writer gpu-wait %.3fs cb %.3fs wait %.3fs | slots %zu, batch %zu MiB\n",
                rd_total, rd_clk.cb, rd_scan, rd_clk.wait, wr_clk.gpu, wr_clk.cb, wr_clk.wait, N, in_cap0 >> 20);
    (void)wr_total;
    return P.error;
}

// ------------------------------------------------------------------ context helpers
Ctx* ctx_new(int codec, bool comp, int threads, int level, size_t inputsize)
{
    Ctx* c = new (std::nothrow) Ctx();
    if (!c) return nullptr;
    c->codec = codec; c->is_comp = comp; c->threads = threads; c->level = level; c->inputsize = inputsize;
    c->E = codec == CODEC_LZ4 ? &kErrLz4 : &kErrZstd;
    return c;
}
void ctx_delete(Ctx* c) { if (!c) return; const DeviceRestore restore_device; ctx_release_slots(c); delete c; }

// Levels.  The device encoders implement one search class per codec (LZ4: the greedy single-probe parse of level 1-2;
// zstd: the same parse + Huffman / predefined-FSE entropy stage, "level 3 (predefined FSE tables)" in BASELINE terms).
// Higher levels are accepted — the CLI default for lz4 is 3 (programs/lz4-mt.c:19) and must keep working — and produce
// the same stream; that is said once on stderr (ZSTDMT_B200_QUIET=1 silences it) instead of silently, and
// ZSTDMT_B200_STRICT_LEVEL=1 turns it into the reference's own answer for a bad parameter (create returns NULL,
// lib/lz4-mt_compress.c:103-108).
bool level_ok(int codec, int level)
{
    const int implemented = codec == CODEC_LZ4 ? 2 : 3;
    if (level <= implemented) return true;
    if (getenv("ZSTDMT_B200_STRICT_LEVEL")) return false;
    static std::atomic<int> told[3];
    if (!getenv("ZSTDMT_B200_QUIET") && told[codec].exchange(1) == 0)
        fprintf(stderr, "[zstdmt_b200] %s level %d requested: the device encoder implements the level-%d search class, the stream is valid but its ratio is that class's\n",
                codec == CODEC_LZ4 ? "lz4" : "zstd", level, implemented);
    return true;
}

const char* status_string(size_t st)
{
    switch (st) {
    case ZMT_ST_TRUNCATED: return "frame truncated";
    case ZMT_ST_BAD_MAGIC: return "ERROR_frameType_unknown";
    case ZMT_ST_BAD_HEADER: return "ERROR_frameHeader_incomplete";
    case ZMT_ST_HDR_CHECKSUM: return "ERROR_headerChecksum_invalid";
    case ZMT_ST_BLOCK: return "ERROR_decompressionFailed";
    case ZMT_ST_DST_SMALL: return "ERROR_dstMaxSize_tooSmall";
    case ZMT_ST_CONTENT_CHECKSUM: return "ERROR_contentChecksum_invalid";
    case ZMT_ST_CONTENT_SIZE: return "ERROR_frameSize_wrong";
    case ZMT_ST_TRAILING: return "trailing bytes after frame";
    case ZMT_ST_UNSUPPORTED: return "stream type not supported by the GPU path";
    case ZMT_ST_CUDA: return "CUDA runtime / kernel failure";
    case ZMT_ST_BAD_ARG: return "bad argument";
    }
    return nullptr;
}

const char* error_string(bool lz4, size_t code, size_t lib_errcode)
{
    static const char* none = nullptr;
    (void)none;
    const size_t neg = 0 - code;
    // the reference returns the codec library's own message whenever its global errcode is set
    // (lz4-mt_common.c:37-38); we own the status table instead of liblz4 / libzstd
    if (lib_errcode && status_string(lib_errcode) && neg == (lz4 ? 8u : 9u)) return status_string(lib_errcode);
    static const char* lz4s[] = { "No error detected", "Allocation error : not enough memory", "Read failure", "Write failure", "Malformed input",
                                  "Could not compress frame at once", "Could not decompress frame at once", "Compression parameter is out of bound",
                                  "Compression library reports failure" };
    static const char* zs[] = { "No error detected", "Allocation error : not enough memory", nullptr, "Read failure", "Write failure", "Malformed input",
                                "Could not compress frame at once", "Could not decompress frame at once", "Compression parameter is out of bound",
                                "Compression library reports failure" };
    if (lz4) { if (neg < 9) return lz4s[neg]; return "Unspecified lz4mt error code"; }
    if (neg < 10 && zs[neg]) return zs[neg];
    return "Unspecified zstmt error code";
}

}  // namespace

// =================================================================== exported C ABI
extern "C" {

uint64_t zmt_device_batches(int dev) { return (dev >= 0 && dev < 64) ? g_dev_batches[dev].load() : 0; }

size_t lz4mt_errcode = 0;      // lib/lz4-mt_common.c:16
size_t zstdmt_errcode = 0;     // lib/zstd-mt_common.c:19

// ---------------- LZ4MT_*
unsigned LZ4MT_isError(size_t code) { return code > (size_t)-10; }                     // lz4-mt_common.c:25-28 (maxCode = 10)
const char* LZ4MT_getErrorString(size_t code) { return error_string(true, code, lz4mt_errcode); }

void* LZ4MT_createCCtx(int threads, int level, int inputsize)                          // lz4-mt_compress.c:92-156
{
    if (threads < 1 || threads > 128) return nullptr;
    if (level < 1 || level > 12) return nullptr;
    if (inputsize < 0) return nullptr;
    if (!level_ok(CODEC_LZ4, level)) return nullptr;
    return ctx_new(CODEC_LZ4, true, threads, level, inputsize ? (size_t)inputsize : (size_t)4 << 20);
}
size_t LZ4MT_compressCCtx(void* ctx, void* rdwr)                                       // lz4-mt_compress.c:312-353
{
    Ctx* c = (Ctx*)ctx;
    if (!c) return kErrLz4.param;
    if (!rdwr) return kErrLz4.param;
    size_t r = compress_run(c, (GenRdWr*)rdwr);
    if (c->lib_errcode) lz4mt_errcode = c->lib_errcode;
    return r;
}
size_t LZ4MT_GetFramesCCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->curframe : 0; }     // lz4-mt_compress.c:374-380
size_t LZ4MT_GetInsizeCCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->insize : 0; }
size_t LZ4MT_GetOutsizeCCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->outsize : 0; }
void LZ4MT_freeCCtx(void* ctx) { ctx_delete((Ctx*)ctx); }

void* LZ4MT_createDCtx(int threads, int inputsize)                                     // lz4-mt_decompress.c:90-142
{
    if (threads < 1 || threads > 128) return nullptr;
    if (inputsize < 0) return nullptr;
    return ctx_new(CODEC_LZ4, false, threads, 0, inputsize ? (size_t)inputsize : (size_t)64 << 10);
}
size_t LZ4MT_decompressDCtx(void* ctx, void* rdwr)                                     // lz4-mt_decompress.c:485-567
{
    Ctx* c = (Ctx*)ctx;
    if (!c || !rdwr) return kErrLz4.param;
    size_t r = decompress_run(c, (GenRdWr*)rdwr);
    if (c->lib_errcode) lz4mt_errcode = c->lib_errcode;
    return r;
}
size_t LZ4MT_GetFramesDCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->curframe : 0; }
size_t LZ4MT_GetInsizeDCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->insize : 0; }
size_t LZ4MT_GetOutsizeDCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->outsize : 0; }
void LZ4MT_freeDCtx(void* ctx) { ctx_delete((Ctx*)ctx); }

// ---------------- ZSTDCB_*
unsigned ZSTDCB_isError(size_t code) { return code > (size_t)-11; }                    // zstd-mt_common.c:26-29 (maxCode = 11)
const char* ZSTDCB_getErrorString(size_t code) { return error_string(false, code, zstdmt_errcode); }

void* ZSTDCB_createCCtx(int threads, int level, int inputsize)                         // zstd-mt_compress.c:94-155
{
    if (threads < 1 || threads > 128) return nullptr;
    if (level < 1 || level > 22) return nullptr;
    if (inputsize < 0) return nullptr;
    if (!level_ok(CODEC_ZSTD, level)) return nullptr;
    size_t chunk = (size_t)inputsize;
    if (!chunk) {
        // the reference indexes its table by `level`, not level-1 (zstd-mt_compress.c:119-127); level 22 reads past
        // the end there — we clamp to the last entry instead of replicating the overrun
        static const int windowLog[] = { 19, 19, 20, 20, 20, 21, 21, 21, 21, 21, 22, 22, 22, 22, 22, 23, 23, 23, 23, 25, 26, 27 };
        int idx = level > 21 ? 21 : level;
        chunk = (size_t)1 << (windowLog[idx] + 1);
        if (chunk > ((size_t)1 << 30)) chunk = (size_t)1 << 30;     // keep int-sized like the reference's int inputsize
    }
    return ctx_new(CODEC_ZSTD, true, threads, level, chunk);
}
size_t ZSTDCB_compressCCtx(void* ctx, void* rdwr)                                      // zstd-mt_compress.c:322-392
{
    Ctx* c = (Ctx*)ctx;
    if (!c) return kErrZstd.init_missing;
    if (!rdwr) return kErrZstd.param;
    c->insize = c->outsize = c->frames = c->curframe = 0;                               // counters reset per call (:337-341)
    c->lib_errcode = 0;
    size_t r = compress_run(c, (GenRdWr*)rdwr);
    if (c->lib_errcode) zstdmt_errcode = c->lib_errcode;
    return r;
}
size_t ZSTDCB_GetFramesCCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->curframe : kErrZstd.init_missing; }  // :395-420
size_t ZSTDCB_GetInsizeCCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->insize : kErrZstd.init_missing; }
size_t ZSTDCB_GetOutsizeCCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->outsize : kErrZstd.init_missing; }
void ZSTDCB_freeCCtx(void* ctx) { ctx_delete((Ctx*)ctx); }

void* ZSTDCB_createDCtx(int threads, int inputsize)                                    // zstd-mt_decompress.c:105-139
{
    if (threads < 1 || threads > 128) return nullptr;
    if (inputsize < 0) return nullptr;
    return ctx_new(CODEC_ZSTD, false, threads, 0, inputsize ? (size_t)inputsize : (size_t)512 << 10);
}
size_t ZSTDCB_decompressDCtx(void* ctx, void* rdwr)                                    // zstd-mt_decompress.c:693-843
{
    Ctx* c = (Ctx*)ctx;
    if (!c || !rdwr) return kErrZstd.param;
    size_t r = decompress_run(c, (GenRdWr*)rdwr);
    if (c->lib_errcode) zstdmt_errcode = c->lib_errcode;
    return r;
}
size_t ZSTDCB_GetFramesDCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->curframe : 0; }    // :845-869
size_t ZSTDCB_GetInsizeDCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->insize : 0; }
size_t ZSTDCB_GetOutsizeDCtx(void* ctx) { return ctx ? ((Ctx*)ctx)->outsize : 0; }
void ZSTDCB_freeDCtx(void* ctx) { ctx_delete((Ctx*)ctx); }

// ---------------- ZSTDMT_* spellings (lib/README.md:43-76)
unsigned ZSTDMT_isError(size_t code) { return ZSTDCB_isError(code); }
const char* ZSTDMT_getErrorString(size_t code) { return ZSTDCB_getErrorString(code); }
void* ZSTDMT_createCCtx(int t, int l, int i) { return ZSTDCB_createCCtx(t, l, i); }
size_t ZSTDMT_compressCCtx(void* c, void* r) { return ZSTDCB_compressCCtx(c, r); }
size_t ZSTDMT_GetFramesCCtx(void* c) { return ZSTDCB_GetFramesCCtx(c); }
size_t ZSTDMT_GetInsizeCCtx(void* c) { return ZSTDCB_GetInsizeCCtx(c); }
size_t ZSTDMT_GetOutsizeCCtx(void* c) { return ZSTDCB_GetOutsizeCCtx(c); }
void ZSTDMT_freeCCtx(void* c) { ZSTDCB_freeCCtx(c); }
void* ZSTDMT_createDCtx(int t, int i) { return ZSTDCB_createDCtx(t, i); }
size_t ZSTDMT_decompressDCtx(void* c, void* r) { return ZSTDCB_decompressDCtx(c, r); }
size_t ZSTDMT_GetFramesDCtx(void* c) { return ZSTDCB_GetFramesDCtx(c); }
size_t ZSTDMT_GetInsizeDCtx(void* c) { return ZSTDCB_GetInsizeDCtx(c); }
size_t ZSTDMT_GetOutsizeDCtx(void* c) { return ZSTDCB_GetOutsizeDCtx(c); }
void ZSTDMT_freeDCtx(void* c) { ZSTDCB_freeDCtx(c); }

}  // extern "C"
