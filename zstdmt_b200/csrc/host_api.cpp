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
#include <functional>
#include <mutex>
#include <thread>
#include <vector>
#include "frame_format.h"
#include "host_common.h"
#include "zmt_dev.h"

namespace {

// ------------------------------------------------------------------ generic boundary types
struct GenBuffer { void* buf; size_t size; size_t allocated; };     // == LZ4MT_Buffer == ZSTDCB_Buffer
typedef int (gen_rw_fn)(void* arg, GenBuffer* b);
struct GenRdWr { gen_rw_fn* fn_read; void* arg_read; gen_rw_fn* fn_write; void* arg_write; };

enum { CODEC_LZ4 = 1, CODEC_ZSTD = 2 };

// error numbering differs between the codecs (lz4-mt.h:41-53 vs zstd-mt.h:41-54)
struct ErrCodes { size_t mem, read_fail, write_fail, data_error, frame_compress, frame_decompress, param, library, canceled, init_missing; };
const ErrCodes kErrLz4  = { (size_t)-1, (size_t)-2, (size_t)-3, (size_t)-4, (size_t)-5, (size_t)-6, (size_t)-7, (size_t)-8, (size_t)-9, (size_t)-7 };
const ErrCodes kErrZstd = { (size_t)-1, (size_t)-3, (size_t)-4, (size_t)-5, (size_t)-6, (size_t)-7, (size_t)-8, (size_t)-9, (size_t)-10, (size_t)-2 };

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
inline bool trace_on() { static const bool on = getenv("ZSTDMT_B200_TRACE") != nullptr; return on; }
// seconds on a steady clock when tracing, else 0 (the clock is not read)
inline double trace_now() { return trace_on() ? std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count() : 0; }

// ------------------------------------------------------------------ device codec table
// the workspace and the compress call follow the context's level (both codecs have more than one encoder)
struct CodecOps {
    size_t   (*c_work)(uint32_t nchunks, uint32_t chunk, int level);
    uint64_t (*c_bound)(uint32_t nchunks, uint32_t chunk);
    int      (*compress)(const void*, uint64_t, uint32_t, const uint32_t*, uint32_t, int level, void*, void*, uint64_t*, void*);
};

const CodecOps& codec_ops(int codec)
{
    static const CodecOps lz4 = { zmt_lz4c_level_workspace_bytes, zmt_lz4c_out_bound, zmt_lz4_compress_level_device };
    static const CodecOps zstd = { zmt_zstdc_level_workspace_bytes, zmt_zstdc_out_bound, zmt_zstd_compress_level_device };
    return codec == CODEC_LZ4 ? lz4 : zstd;
}

// ------------------------------------------------------------------ batch tables
// Per-chunk / per-frame tables of a batch (entries = tab_cap).  Layout:
//   u64 frame_off[cap+1] | u64 out_off[cap+1] | u64 out_size[cap+1] | u64 expect[cap+1] | u32 per_frame[cap] | u32 status[cap] | u32 first_blk[cap+1]
struct Tables {
    uint64_t* frame_off;         // compress: where each frame starts in the output (+ total); decompress: where its 12-byte header starts in the input
    uint64_t* out_off;           // decompress: where each frame's content goes (+ total)
    uint64_t* out_size;          // decompress: bytes each frame decoded to
    uint64_t* expect;            // zstd decompress: content size from the frame header, ~0 when the header has none
    uint32_t* per_frame;         // compress: bytes in the chunk; lz4 decompress: payload bytes of the frame;
                                 // zstd decompress: frame flags of the host scan (sequential pass, checksum, no size)
    uint32_t* status;            // decompress: ZMT_ST_* per frame
    uint32_t* first_blk;         // zstd decompress: the frame's first block descriptor (+ total)
};
inline size_t tables_bytes(size_t cap) { return 4 * (cap + 1) * 8 + 2 * cap * 4 + (cap + 1) * 4 + 64; }
inline Tables tables_at(uint8_t* base, size_t cap)
{
    Tables t; t.frame_off = (uint64_t*)base; t.out_off = t.frame_off + cap + 1; t.out_size = t.out_off + cap + 1; t.expect = t.out_size + cap + 1;
    t.per_frame = (uint32_t*)(t.expect + cap + 1); t.status = t.per_frame + cap; t.first_blk = t.status + cap; return t;
}

// lz4 decode block table capacity of a slot: every frame owns max(1, ceil(out / 64 KiB)) slots
inline uint32_t lz4_slot_cap(size_t out_cap, size_t tab_cap) { return (uint32_t)(out_cap / 65536 + tab_cap + 1); }

// The frames of one decode batch, in the order the decoder takes them, with the totals its workspace is sized from.
// Every host decode batch is built here (a container slot, a batch of plain frames, one segment of an LZ4F frame) and
// packed into a Tables view just before it is copied to the device.
struct FrameList {
    std::vector<uint64_t> in_off;     // where each frame starts in the batch input (LZ4: its 12-byte header)
    std::vector<uint64_t> out_off;    // where each frame's content goes, + the end of the last one
    std::vector<uint64_t> expect;     // zstd: the content size from the header, ~0 without one
    std::vector<uint32_t> per_frame;  // LZ4: payload bytes; zstd: ZF_* flags of the frame walk
    std::vector<uint32_t> first_blk;  // zstd: each frame's first block descriptor, + the total
    uint32_t nblk = 0;                // zstd: block descriptors of the batch
    uint64_t scratch = 0;             // zstd: entropy scratch bytes of the batch
    uint64_t nslots = 0;              // LZ4: block-table slots of the batch (lz4_frame_slots per frame)

    FrameList() { clear(); }
    uint32_t n() const { return (uint32_t)in_off.size(); }
    uint64_t out_end() const { return out_off.back(); }
    // an empty batch whose output starts at out_at
    void clear(uint64_t out_at = 0)
    {
        in_off.clear(); expect.clear(); per_frame.clear();
        out_off.assign(1, out_at); first_blk.assign(1, 0);
        nblk = 0; scratch = 0; nslots = 0;
    }
    // one frame at `at` with `room` bytes of output; zstd: its descriptors end at blk_to and the batch's scratch at scr_to
    void push(uint64_t at, uint32_t pf, uint64_t room, uint64_t exp = 0, uint32_t blk_to = 0, uint64_t scr_to = 0)
    {
        in_off.push_back(at); per_frame.push_back(pf); expect.push_back(exp);
        out_off.push_back(out_end() + room); first_blk.push_back(blk_to);
        nblk = blk_to; scratch = scr_to; nslots += lz4_frame_slots(room);
    }
    void pack(const Tables& T) const
    {
        const size_t k = n();
        memcpy(T.frame_off, in_off.data(), k * 8); memcpy(T.out_off, out_off.data(), (k + 1) * 8); memcpy(T.expect, expect.data(), k * 8);
        memcpy(T.per_frame, per_frame.data(), k * 4); memcpy(T.first_blk, first_blk.data(), (k + 1) * 4);
    }
};

// The zstd block-table rule of a decode batch.  Walks the zstd frame f[0..n), at base_off in the batch input, as the
// next frame of `fl`: its descriptors go to blk[fl.nblk, cap), and *w gets the batch's block and scratch totals with it,
// the frame's room (its content size, or the block bound with ZF_NO_SIZE), its flags and its length.  When the table is
// full (ZMT_ST_DST_SMALL) and `count` is set, a counting walk fills *w instead and returns the frame's own status if that
// is not OK: the caller grows the table, or carries the frame to the next batch, and walks once more.  A frame that fits
// is walked once.
struct ZWalk { uint32_t nblk = 0, flags = 0; uint64_t scratch = 0, room = 0; size_t end = 0; };
int zstd_blocks(const FrameList& fl, const uint8_t* f, size_t n, uint64_t base_off, void* blk, uint32_t cap, bool count, ZWalk& w)
{
    w.nblk = fl.nblk; w.scratch = fl.scratch;
    int r = zstd_frame_walk<true>(f, n, base_off, fl.n(), (ZBlk*)blk, &w.nblk, cap, &w.scratch, &w.room, &w.flags, &w.end);
    if (r != ZMT_ST_DST_SMALL || !count) return r;
    w.nblk = fl.nblk; w.scratch = fl.scratch;
    r = zstd_frame_walk<false>(f, n, base_off, fl.n(), nullptr, &w.nblk, 0xFFFFFFFFu, &w.scratch, &w.room, &w.flags, &w.end);
    return r == ZMT_ST_OK ? ZMT_ST_DST_SMALL : r;
}
inline uint64_t zstd_expect(const ZWalk& w) { return (w.flags & ZF_NO_SIZE) ? ~0ull : w.room; }

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
    uint32_t n = 0;              // compress: chunks in this batch
    FrameList frames;            // decompress: frames in this batch
    uint64_t scr_cap = 0;        // zstd decompress: entropy scratch bytes the workspace was sized for
    // zstd decompress: block descriptors built by the reader (pinned) + device copy
    uint8_t *h_blk = nullptr, *d_blk = nullptr; uint32_t blk_cap = 0;
    size_t in_used = 0;
    int state = 0;               // 0 free, 1 filled, 2 submitted
    bool ok = false;
    bool host_alias = false;     // h_in / h_out are borrowed from another slot of the same context (never freed here)
};

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

// Process-wide pool of staging slots: pinned allocations cost ~0.1 s per context otherwise (the reference's
// malloc'd buffers are free by comparison).  Slots go back to the pool when a context is freed and are
// reused by the next context that needs the same device and no larger capacities.
std::mutex g_pool_mu;
std::vector<Slot> g_pool;
const size_t kPoolMax = 16;

// host_owner: the slot whose pinned staging buffers this one borrows (a call over more devices than it keeps batches in
// flight: the host ring stays 4 x 8 MiB — cache-resident for the callbacks' memcpy — while every device has its own
// device-side buffers); nullptr: the slot gets pinned buffers of its own.
bool slot_alloc(Slot& s, int dev, size_t in_cap, size_t out_cap, size_t work_cap, size_t tab_cap, const Slot* host_owner)
{
    bool ok = false;
    {
        std::lock_guard<std::mutex> g(g_pool_mu);                       // a pooled slot of a previous call (device-only for a borrower)
        for (size_t i = 0; i < g_pool.size() && !ok; i++) {
            Slot& c = g_pool[i];
            if ((c.h_in == nullptr) == (host_owner != nullptr) && c.dev == dev && c.in_cap >= in_cap && c.out_cap >= out_cap &&
                c.work_cap >= work_cap && c.tab_cap == tab_cap) {
                s = c; g_pool.erase(g_pool.begin() + (long)i);
                s.state = 0; s.n = 0; s.in_used = 0; s.frames.clear();
                ok = true;
            }
        }
    }
    if (!ok) {
        s.dev = dev;
        if (cudaSetDevice(dev) != cudaSuccess) return false;
        const ScopedAffinity bind(device_local_cpus(dev));     // first touch of the pinned buffers happens on the GPU's node
        ok = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) == cudaSuccess;
        ok = ok && cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming) == cudaSuccess;
        for (int k = 0; k < 2; k++) ok = ok && cudaEventCreateWithFlags(&s.evp[k], cudaEventDisableTiming) == cudaSuccess;
        if (!host_owner) {
            ok = ok && cudaHostAlloc((void**)&s.h_in, in_cap + 64, cudaHostAllocPortable) == cudaSuccess;
            ok = ok && cudaHostAlloc((void**)&s.h_out, out_cap + 64, cudaHostAllocPortable) == cudaSuccess;
        }
        ok = ok && cudaMalloc((void**)&s.d_in, in_cap + 256) == cudaSuccess;
        ok = ok && cudaMalloc((void**)&s.d_out, out_cap + 256) == cudaSuccess;
        ok = ok && cudaMalloc((void**)&s.d_work, work_cap + 256) == cudaSuccess;
        s.tab_bytes = tables_bytes(tab_cap);
        ok = ok && cudaHostAlloc((void**)&s.h_tab, s.tab_bytes, cudaHostAllocPortable) == cudaSuccess;
        ok = ok && cudaMalloc((void**)&s.d_tab, s.tab_bytes) == cudaSuccess;
        s.in_cap = in_cap; s.out_cap = out_cap; s.work_cap = work_cap; s.tab_cap = tab_cap; s.ok = ok;
        if (!ok) { cudaGetLastError(); slot_free_raw(s); return false; }
    }
    if (host_owner) { s.h_in = host_owner->h_in; s.h_out = host_owner->h_out; s.host_alias = true; }
    return true;
}

void slot_free(Slot& s)
{
    // borrowed buffers belong to the owner slot: the device side goes to the pool as a device-only slot
    if (s.host_alias) { s.h_in = nullptr; s.h_out = nullptr; s.host_alias = false; }
    if (s.ok) {
        cudaSetDevice(s.dev);
        if (s.stream) cudaStreamSynchronize(s.stream);
        std::lock_guard<std::mutex> g(g_pool_mu);
        if (g_pool.size() < kPoolMax) { g_pool.push_back(s); s = Slot(); return; }
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

// a frame's ZMT_ST_* -> the library error of the call, the status kept for *_getErrorString: a cut or overlong frame is the
// frame's fault, the rest the codec's
inline size_t frame_error(Ctx* c, uint32_t st)
{
    c->lib_errcode = st;
    return st == ZMT_ST_TRUNCATED || st == ZMT_ST_TRAILING ? c->E->frame_decompress : c->E->library;
}

// ------------------------------------------------------------------ the pipeline of one call
// reader thread  : fill    — fn_read into the free slot, in sequence order (pt_read / the read section of pt_compress)
// calling thread : submit  — H2D, the device entry point, D2H of the tables, s.ev recorded
// writer thread  : drain   — after s.ev: fn_write the slot's frames in order (pt_write)
// A slot goes 0 free -> 1 filled -> 2 submitted -> 0.  Batch q + in_flight is filled only once batch q has been written
// (slots beyond the first in_flight share their pinned buffers).  The first error any stage raises with P.fail() stops all
// three; the call returns it.
struct PipeOps {
    std::function<bool(Slot&)> fill;     // false: no batch (end of input, or after P.fail)
    std::function<int(Slot&)>  submit;   // ZMT_ST_*
    std::function<bool(Slot&)> drain;    // false after P.fail
    const char* name = "";               // ZSTDMT_B200_TRACE line
    size_t batch_bytes = 0;
    const double* scan = nullptr;        // decompress: the reader's time in the frame scan (traced only)
};

size_t run_pipeline(Ctx* c, size_t in_flight, const PipeOps& ops)
{
    const ErrCodes& E = *c->E;
    Pipe& P = c->pipe;
    const size_t N = P.slots.size();
    P.fill_seq = P.submit_seq = P.write_seq = 0; P.reader_done = false; P.error = 0;
    for (auto& s : P.slots) s.state = 0;
    struct { double wait = 0, work = 0, gpu = 0; } rd, sb, wr;             // seconds, ZSTDMT_B200_TRACE only
    const CpuSet host_cpus = common_local_cpus(c->devs);

    std::thread reader([&]() {
        const ScopedAffinity bind(host_cpus);
        for (;;) {
            Slot* s;
            {
                const double t0 = trace_now();
                std::unique_lock<std::mutex> lk(P.mu);
                s = &P.slots[P.fill_seq % N];
                P.cv.wait(lk, [&] { return (s->state == 0 && P.fill_seq - P.write_seq < in_flight) || P.error; });
                rd.wait += trace_now() - t0;
                if (P.error) break;
            }
            const double t0 = trace_now();
            const bool filled = ops.fill(*s);
            rd.work += trace_now() - t0;
            if (!filled) break;
            { std::lock_guard<std::mutex> g(P.mu); s->state = 1; P.fill_seq++; }
            P.cv.notify_all();
        }
        { std::lock_guard<std::mutex> g(P.mu); P.reader_done = true; }
        P.cv.notify_all();
    });

    std::thread writer([&]() {
        const ScopedAffinity bind(host_cpus);
        for (;;) {
            Slot* s;
            {
                const double t0 = trace_now();
                std::unique_lock<std::mutex> lk(P.mu);
                s = &P.slots[P.write_seq % N];
                P.cv.wait(lk, [&] { return s->state == 2 || P.error || (P.reader_done && P.write_seq == P.fill_seq); });
                wr.wait += trace_now() - t0;
                if (P.error || s->state != 2) break;
            }
            cudaSetDevice(s->dev);
            const double t0 = trace_now();
            if (cudaEventSynchronize(s->ev) != cudaSuccess) { c->lib_errcode = ZMT_ST_CUDA; P.fail(E.library); break; }
            const double t1 = trace_now();
            const bool drained = ops.drain(*s);
            wr.gpu += t1 - t0; wr.work += trace_now() - t1;
            if (!drained) break;
            { std::lock_guard<std::mutex> g(P.mu); s->state = 0; P.write_seq++; }
            P.cv.notify_all();
        }
    });

    for (;;) {
        Slot* s;
        {
            const double t0 = trace_now();
            std::unique_lock<std::mutex> lk(P.mu);
            s = &P.slots[P.submit_seq % N];
            P.cv.wait(lk, [&] { return s->state == 1 || P.error || (P.reader_done && P.submit_seq == P.fill_seq); });
            sb.wait += trace_now() - t0;
            if (P.error || s->state != 1) break;
        }
        cudaSetDevice(s->dev);
        const double t0 = trace_now();
        const int st = ops.submit(*s);
        sb.work += trace_now() - t0;
        if (s->dev >= 0 && s->dev < 64) g_dev_batches[s->dev]++;
        if (st != ZMT_ST_OK) { c->lib_errcode = (size_t)st; P.fail(E.library); break; }
        { std::lock_guard<std::mutex> g(P.mu); s->state = 2; P.submit_seq++; }
        P.cv.notify_all();
    }
    reader.join(); writer.join();
    for (auto& s : P.slots) if (s.ok) { cudaSetDevice(s.dev); cudaStreamSynchronize(s.stream); }
    if (trace_on()) {
        char scan[48] = "";
        if (ops.scan) snprintf(scan, sizeof(scan), " | reader scan %.3fs", *ops.scan);
        fprintf(stderr, "[zstdmt_b200] %s: reader fill %.3fs wait %.3fs | submit enqueue %.3fs wait %.3fs | writer gpu-wait %.3fs drain %.3fs wait %.3fs"
                " | slots %zu, batch %zu KiB%s\n", ops.name, rd.work, rd.wait, sb.work, sb.wait, wr.gpu, wr.work, wr.wait, N, ops.batch_bytes >> 10, scan);
    }
    return P.error;
}

// ------------------------------------------------------------------ compression
size_t compress_run(Ctx* c, GenRdWr* rw)
{
    const DeviceRestore restore_device;
    const ErrCodes& E = *c->E;
    const CodecOps& ops = codec_ops(c->codec);
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
    if (nsl > base_slots) nsl = (nsl + base_slots - 1) / base_slots * base_slots;   // batch q uses host buffer q % base_slots: needs base_slots | slots
    size_t B = batch_bytes / chunk; if (B < 1) B = 1; if (B > 65536) B = 65536;

    if (P.slots.empty()) {
        P.slots.resize(nsl);
        for (size_t i = 0; i < P.slots.size(); i++) {
            const size_t ic = B * chunk, oc = (size_t)ops.c_bound((uint32_t)B, (uint32_t)chunk), wc = ops.c_work((uint32_t)B, (uint32_t)chunk, c->level);
            if (!slot_alloc(P.slots[i], c->devs[i % c->devs.size()], ic, oc, wc, B, i < base_slots ? nullptr : &P.slots[i % base_slots])) {
                ctx_release_slots(c); return E.mem;
            }
        }
    }

    size_t frames_read = 0; bool eof = false;
    PipeOps po;
    // pt_compress read section, lz4-mt_compress.c:255-277
    po.fill = [&](Slot& s) -> bool {
        if (eof) return false;
        Tables T = tables_at(s.h_tab, s.tab_cap);
        uint32_t n = 0; size_t got_bytes = 0;
        while (n < B) {
            GenBuffer b; b.buf = s.h_in + (size_t)n * chunk; b.size = chunk; b.allocated = chunk;
            int rv = rw->fn_read(rw->arg_read, &b);
            if (rv != 0) { P.fail(mt_error(E, rv)); return false; }
            if (b.size > chunk) { P.fail(E.read_fail); return false; }
            if (b.size == 0 && frames_read > 0) { eof = true; break; }
            T.per_frame[n] = (uint32_t)b.size; got_bytes += b.size; frames_read++; n++;
        }
        if (n == 0) return false;
        s.n = n; s.in_used = got_bytes;
        c->insize += got_bytes; c->frames += n;
        return true;
    };
    po.submit = [&](Slot& s) -> int {
        Tables Th = tables_at(s.h_tab, s.tab_cap), Td = tables_at(s.d_tab, s.tab_cap);
        bool full = true;
        for (uint32_t i = 0; i < s.n; i++) if (Th.per_frame[i] != chunk) { full = false; break; }
        cudaError_t ce = cudaSuccess;
        if (full) ce = cudaMemcpyAsync(s.d_in, s.h_in, (size_t)s.n * chunk, cudaMemcpyHostToDevice, s.stream);
        else for (uint32_t i = 0; i < s.n && ce == cudaSuccess; i++)
            if (Th.per_frame[i]) ce = cudaMemcpyAsync(s.d_in + (size_t)i * chunk, s.h_in + (size_t)i * chunk, Th.per_frame[i], cudaMemcpyHostToDevice, s.stream);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(Td.per_frame, Th.per_frame, (size_t)s.n * 4, cudaMemcpyHostToDevice, s.stream);
        if (ce != cudaSuccess) return ZMT_ST_CUDA;
        const int st = ops.compress(s.d_in, 0, (uint32_t)chunk, Td.per_frame, s.n, c->level, s.d_work, s.d_out, Td.frame_off, s.stream);
        if (st != ZMT_ST_OK) return st;
        if (cudaMemcpyAsync(Th.frame_off, Td.frame_off, ((size_t)s.n + 1) * 8, cudaMemcpyDeviceToHost, s.stream) != cudaSuccess ||
            cudaEventRecord(s.ev, s.stream) != cudaSuccess) return ZMT_ST_CUDA;
        return ZMT_ST_OK;
    };
    // pt_write, lz4-mt_compress.c:178-205
    po.drain = [&](Slot& s) -> bool {
        Tables T = tables_at(s.h_tab, s.tab_cap);
        const uint64_t total = T.frame_off[s.n];
        if (total > s.out_cap) { c->lib_errcode = ZMT_ST_DST_SMALL; P.fail(E.library); return false; }
        if (cudaMemcpyAsync(s.h_out, s.d_out, total, cudaMemcpyDeviceToHost, s.stream) != cudaSuccess ||
            cudaStreamSynchronize(s.stream) != cudaSuccess) { c->lib_errcode = ZMT_ST_CUDA; P.fail(E.library); return false; }
        for (uint32_t i = 0; i < s.n; i++) {
            GenBuffer b; b.buf = s.h_out + T.frame_off[i]; b.size = (size_t)(T.frame_off[i + 1] - T.frame_off[i]); b.allocated = b.size;
            int rv = rw->fn_write(rw->arg_write, &b);
            if (rv != 0) { P.fail(mt_error(E, rv)); return false; }
            c->outsize += b.size; c->curframe++;
        }
        return true;
    };
    po.name = "compress"; po.batch_bytes = B * chunk;
    return run_pipeline(c, P.slots.size() > base_slots ? base_slots : P.slots.size(), po);
}

// ------------------------------------------------------------------ decompression
// reads exactly `want` bytes unless EOF; returns 0 ok / error; *got = delivered
size_t read_some(const ErrCodes& E, GenRdWr* rw, void* dst, size_t want, size_t* got)
{
    GenBuffer b; b.buf = dst; b.size = want; b.allocated = want;
    int rv = rw->fn_read(rw->arg_read, &b);
    if (rv != 0) return mt_error(E, rv);
    if (b.size > want) return E.read_fail;
    *got = b.size; return 0;
}

// One decode step on `st`: the batch's tables (packed into h_tab, `cap` entries; the device copy at d_tab) and, for zstd,
// its block descriptors go to the device, the batch is decoded (with `seg` / `zseg`: as one segment of an LZ4F / a zstd
// frame), and its status and sizes come back into h_tab.  The batch's input must be in place on the stream before.
// Returns ZMT_ST_*.
int decode_step(bool is_zstd, const FrameList& fl, uint8_t* h_tab, uint8_t* d_tab, size_t cap, const void* h_blk, void* d_blk,
                const void* d_in, size_t in_bytes, void* d_out, void* d_work, zmt_lz4_segment* seg, zmt_zstd_segment* zseg, cudaStream_t st)
{
    const Tables Th = tables_at(h_tab, cap), Td = tables_at(d_tab, cap);
    const uint32_t n = fl.n(), nslots = (uint32_t)fl.nslots;
    fl.pack(Th);
    if (cudaMemcpyAsync(d_tab, h_tab, tables_bytes(cap), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (is_zstd && fl.nblk && cudaMemcpyAsync(d_blk, h_blk, (size_t)fl.nblk * sizeof(ZBlk), cudaMemcpyHostToDevice, st) != cudaSuccess))
        return ZMT_ST_CUDA;
    const int r = is_zstd ? (zseg ? zmt_zstd_decompress_segments_device(d_in, d_blk, fl.nblk, Td.first_blk, Td.expect, Td.per_frame, n, d_out, Td.out_off, Td.out_size,
                                                                        Td.status, zseg, d_work, st)
                                  : zmt_zstd_decompress_device(d_in, d_blk, fl.nblk, Td.first_blk, Td.expect, Td.per_frame, n, d_out, Td.out_off, Td.out_size, Td.status, d_work, st))
                : seg ? zmt_lz4_decompress_segments_device(d_in, in_bytes, Td.frame_off, Td.per_frame, n, nslots, d_out, Td.out_off, Td.out_size, Td.status, seg, d_work, st)
                      : zmt_lz4_decompress_device(d_in, in_bytes, Td.frame_off, Td.per_frame, n, nslots, d_out, Td.out_off, Td.out_size, Td.status, d_work, st);
    if (r != ZMT_ST_OK) return r;
    if (cudaMemcpyAsync(Th.out_size, Td.out_size, (size_t)n * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(Th.status, Td.status, (size_t)n * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) return ZMT_ST_CUDA;
    return ZMT_ST_OK;
}

// ------------------------------------------------------------------ plain (unframed) single streams
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

// What the reference routes to st_decompress (lz4-mt_decompress.c:391-483, zstd-mt_decompress.c:552-687): an ordinary
// .lz4 / .zst file, i.e. codec frames back to back without the 12-byte size headers.  Frame lengths are only known after
// walking the block headers, so the host reads ahead, cuts the bytes it holds into complete frames, and decodes them in
// batches of at most ~`batch` input bytes with the same GPU kernels; the consumed bytes are dropped before the next read.
// A frame larger than a batch is decoded in segments (lz4_segments, zstd_segments), so memory is O(batch + 64 KiB) for
// LZ4 and O(batch + window) for zstd.  Single-threaded: a batch's frames are written before the next read.
struct PlainStream {
    Ctx* c; GenRdWr* rw;
    const bool is_zstd;
    const size_t batch, piece;              // input bytes per batch (ZSTDMT_B200_PLAIN_MB); bytes per fn_read and per fn_write
    std::vector<uint8_t> in;                // 12 pad bytes (the LZ4 kernel addresses a frame as base + off + 12), then the bytes held
    size_t pos = 0;                         // parse position inside in[12..]
    bool eof = false;
    cudaStream_t st = nullptr;
    DevBuf d_in, d_out, d_tab, d_blk, d_work, d_seg, d_hist;         // d_seg, d_hist: frames decoded in segments
    std::vector<uint8_t> h_tab, out;        // the batch's tables (status and sizes come back here) and decoded bytes
    std::vector<ZBlk> blocks;               // zstd: the batch's block table
    FrameList fl;

    // `first`/`have` = the bytes already consumed by the stream-type sniffing
    PlainStream(Ctx* c_, GenRdWr* rw_, const uint8_t* first, size_t have)
        : c(c_), rw(rw_), is_zstd(c_->codec == CODEC_ZSTD), batch(env_size("ZSTDMT_B200_PLAIN_MB", 64) << 20),
          piece(c_->inputsize < (64u << 10) ? (size_t)1 << 20 : c_->inputsize), in(12, 0)
    {
        in.insert(in.end(), first, first + have);
    }
    ~PlainStream() { if (st) cudaStreamDestroy(st); }

    // Appends reads of up to `piece` bytes to `in`, at least one, until it holds `goal` bytes or the input ends.
    size_t read_to(size_t goal)
    {
        do {
            const size_t old = in.size();
            in.resize(old + piece);
            size_t got = 0;
            const size_t e = read_some(*c->E, rw, in.data() + old, piece, &got);
            in.resize(old + got);
            if (e) return e;
            c->insize += got;
            if (got == 0) eof = true;
        } while (!eof && in.size() < goal);
        return 0;
    }

    // Writes p[0..size) to fn_write in pieces of at most `piece` bytes (st_decompress writes as it goes).
    size_t write(const uint8_t* p, uint64_t size)
    {
        for (uint64_t o = 0; o < size;) {
            GenBuffer b; b.buf = (void*)(p + o); b.size = (size_t)(size - o < piece ? size - o : piece); b.allocated = b.size;
            const size_t want = b.size;
            const int rv = rw->fn_write(rw->arg_write, &b);
            if (rv != 0) return mt_error(*c->E, rv);
            c->outsize += b.size; o += want;
        }
        return 0;
    }

    // Decodes the batch `fl`: src[0 .. in_bytes - lo) goes to d_in + lo (the device addresses the frames at their offsets in
    // the batch input), the decode step runs, and the output room [out_off[0], out_end) comes back into `out` with the
    // status and sizes (in h_tab), in one stream synchronisation.
    size_t decode(const uint8_t* src, size_t lo, size_t in_bytes, zmt_lz4_segment* seg, zmt_zstd_segment* zseg = nullptr)
    {
        const uint32_t nf = fl.n();
        const uint64_t out_at = fl.out_off[0], room = fl.out_end() - out_at;
        const size_t tab_bytes = tables_bytes(nf);
        const size_t wk = is_zstd ? zmt_zstdd_workspace_bytes(nf, fl.nblk, fl.scratch) : zmt_lz4d_workspace_bytes(nf, (uint32_t)fl.nslots, in_bytes);
        if (!d_in.need(in_bytes + 256) || !d_out.need(fl.out_end() + 256) || !d_tab.need(tab_bytes) || !d_work.need(wk) ||
            (is_zstd && !d_blk.need((size_t)fl.nblk * sizeof(ZBlk) + 16))) return c->E->mem;
        h_tab.resize(tab_bytes);
        out.resize(room ? room : 1);
        cudaError_t ce = cudaMemcpyAsync((uint8_t*)d_in.p + lo, src, in_bytes - lo, cudaMemcpyHostToDevice, st);
        const int rc = ce == cudaSuccess ? decode_step(is_zstd, fl, h_tab.data(), (uint8_t*)d_tab.p, nf, blocks.data(), d_blk.p, d_in.p, in_bytes,
                                                       d_out.p, d_work.p, seg, zseg, st) : ZMT_ST_CUDA;
        if (rc == ZMT_ST_OK && room) ce = cudaMemcpyAsync(out.data(), (uint8_t*)d_out.p + out_at, room, cudaMemcpyDeviceToHost, st);
        if (rc == ZMT_ST_OK && ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        if (rc != ZMT_ST_OK || ce != cudaSuccess) { cudaGetLastError(); return frame_error(c, ZMT_ST_CUDA); }
        return 0;
    }

    // One LZ4F frame that reaches a batch of input (or four of output) before its end, at in[12 + pos], decoded as a chain
    // of segments of whole blocks (zmt_lz4_decompress_segments_device): each segment is read, decoded and written before
    // the next one is read, and its input dropped.  The device keeps the frame's state between segments (zmt_lz4_segment:
    // XXH32, content size) in d_seg and, for linked blocks, the last 64 KiB of content in d_hist; the segment's output goes
    // to d_out + 64 KiB with the history copied directly below.  Memory stays O(batch) whatever the frame's size.  One
    // stream synchronisation per segment: status, size and the output room come back together, and the history of the
    // next segment is saved behind them.  On return the frame has been consumed (pos = 0, in holds what follows it).
    size_t lz4_segments()
    {
        const uint32_t flg = in[12 + pos + 4], bd = in[12 + pos + 5];
        const bool linked = !(flg & 0x20);
        const uint64_t H = 65536;                               // the history's room below each segment's output
        if (!d_seg.need(sizeof(zmt_lz4_segment)) || !d_hist.need(H)) return c->E->mem;
        if (cudaMemsetAsync(d_seg.p, 0, sizeof(zmt_lz4_segment), st) != cudaSuccess) { cudaGetLastError(); return frame_error(c, ZMT_ST_CUDA); }
        zmt_lz4_segment* ds = (zmt_lz4_segment*)d_seg.p;
        uint64_t produced = 0;
        for (bool first = true;; first = false) {
            // ---- the next segment: whole blocks up to a batch of input / four of output room
            size_t end = 0; uint64_t room = 0; uint32_t last = 0;
            while (zmt_lz4f_segment_host(in.data() + 12 + pos, in.size() - 12 - pos, first ? lz4f_header_len(flg) : 0, flg, bd,
                                         batch, 4 * (uint64_t)batch, &end, &room, &last) != ZMT_ST_OK) {
                if (eof) return frame_error(c, ZMT_ST_TRUNCATED);
                const size_t e = read_to(12 + pos + batch + piece);
                if (e) return e;
            }
            // ---- decode it: a batch of one frame, its bytes at d_in + 12, its output at d_out + H above `hlen` bytes of history
            const uint64_t hlen = linked ? (produced < H ? produced : H) : 0;
            const uint32_t flags = (first ? ZMT_SEG_FIRST : 0u) | (last ? ZMT_SEG_LAST : 0u);
            if (!d_out.need(H + room + 256)) return c->E->mem;
            cudaError_t ce = cudaMemcpyAsync(&ds->history, &hlen, sizeof(hlen), cudaMemcpyHostToDevice, st);
            if (ce == cudaSuccess) ce = cudaMemcpyAsync(&ds->flags, &flags, sizeof(flags), cudaMemcpyHostToDevice, st);
            if (ce == cudaSuccess && hlen) ce = cudaMemcpyAsync((uint8_t*)d_out.p + H - hlen, d_hist.p, hlen, cudaMemcpyDeviceToDevice, st);
            if (ce != cudaSuccess) { cudaGetLastError(); return frame_error(c, ZMT_ST_CUDA); }
            fl.clear(H); fl.push(0, (uint32_t)end, room);
            const size_t e = decode(in.data() + 12 + pos, 12, 12 + end, ds);
            if (e) return e;
            const Tables T = tables_at(h_tab.data(), 1);
            if (T.status[0] != ZMT_ST_OK) return frame_error(c, T.status[0]);
            const uint64_t osz = T.out_size[0];
            if (osz > room) return frame_error(c, ZMT_ST_DST_SMALL);
            // ---- the history of the next segment: the last 64 KiB of [history | this segment], contiguous below H + osz; queued
            //      behind this segment, ahead of the next one (a reallocation of d_out in between synchronises in cudaFree)
            const uint64_t hnext = linked ? (hlen + osz < H ? hlen + osz : H) : 0;
            if (hnext && !last && cudaMemcpyAsync(d_hist.p, (uint8_t*)d_out.p + H + osz - hnext, hnext, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
                cudaGetLastError(); return frame_error(c, ZMT_ST_CUDA);
            }
            const size_t we = write(out.data(), osz);
            if (we) return we;
            produced += osz;
            in.erase(in.begin() + 12, in.begin() + 12 + (long)(pos + end));       // drop the decoded segment
            pos = 0;
            if (last) return 0;
        }
    }

    // The same for one zstd frame (zmt_zstd_decompress_segments_device).  What crosses a cut:
    //   - the window: the last min(Window_Size, produced) content bytes, saved to d_hist behind each segment and copied
    //     back directly below the next segment's output (the two ranges overlap when a segment is shorter than the window);
    //   - the table sources: the bytes of the (at most four) blocks that describe the tables the next blocks may inherit,
    //     kept in `carry` and placed in front of the segment's bytes in d_in, where the walk's ZB_SRC descriptors name them;
    //   - repeat offsets, XXH64 state, content size and produced bytes: in the device record d_seg.
    // Memory stays O(batch + window).
    size_t zstd_segments()
    {
        if (!d_seg.need(sizeof(zmt_zstd_segment))) return c->E->mem;
        if (cudaMemsetAsync(d_seg.p, 0, sizeof(zmt_zstd_segment), st) != cudaSuccess) { cudaGetLastError(); return frame_error(c, ZMT_ST_CUDA); }
        zmt_zstd_segment* ds = (zmt_zstd_segment*)d_seg.p;
        zmt_zstd_walk w = {};
        std::vector<uint8_t> carry, next;
        uint64_t produced = 0;
        if (blocks.size() < 4096) blocks.resize(4096);
        for (bool first = true;; first = false) {
            // ---- the next segment: whole blocks up to a batch of input / four of output room
            const uint64_t seg_at = w.pos;
            uint64_t so[4]; uint32_t sl[4];
            const uint32_t ns = zstd_walk_sources(&w, so, sl);
            zmt_zstd_walk t;
            uint32_t nb; uint64_t scr, room;
            for (;;) {
                t = w; nb = 0; scr = 0;
                const int r = zstd_walk_blocks<true>(in.data() + 12 + pos, in.size() - 12 - pos, 12 + carry.size(), 0, blocks.data(), &nb,
                                                     (uint32_t)blocks.size(), &scr, &t, batch, 4 * (uint64_t)batch, &room);
                if (r == ZMT_ST_OK) break;
                if (r == ZMT_ST_DST_SMALL) { blocks.resize(2 * blocks.size()); continue; }
                if (r != ZMT_ST_TRUNCATED) return frame_error(c, r);
                if (eof) return frame_error(c, ZMT_ST_TRUNCATED);
                const size_t e = read_to(12 + pos + batch + piece);
                if (e) return e;
            }
            const size_t end = (size_t)(t.pos - seg_at);
            const bool last = t.done != 0;
            // ---- decode it: a batch of one frame, [carry | segment bytes] at d_in + 12, its output at d_out + hlen above the history
            const uint64_t hlen = produced < w.window ? produced : w.window;
            const uint32_t flags = (first ? ZMT_SEG_FIRST : 0u) | (last ? ZMT_SEG_LAST : 0u);
            if (!d_out.need(hlen + room + 256) || !d_in.need(12 + carry.size() + end + 256)) return c->E->mem;
            cudaError_t ce = cudaMemcpyAsync(&ds->history, &hlen, sizeof(hlen), cudaMemcpyHostToDevice, st);
            if (ce == cudaSuccess) ce = cudaMemcpyAsync(&ds->flags, &flags, sizeof(flags), cudaMemcpyHostToDevice, st);
            if (ce == cudaSuccess && hlen) ce = cudaMemcpyAsync(d_out.p, d_hist.p, hlen, cudaMemcpyDeviceToDevice, st);
            if (ce == cudaSuccess && !carry.empty()) ce = cudaMemcpyAsync((uint8_t*)d_in.p + 12, carry.data(), carry.size(), cudaMemcpyHostToDevice, st);
            if (ce != cudaSuccess) { cudaGetLastError(); return frame_error(c, ZMT_ST_CUDA); }
            fl.clear(hlen);
            fl.push(0, t.flags | ZF_NEEDS_SEQ, room, (t.flags & ZF_NO_SIZE) ? ~0ull : t.content_size, nb, scr);
            const size_t e = decode(in.data() + 12 + pos, 12 + carry.size(), 12 + carry.size() + end, nullptr, ds);
            if (e) return e;
            const Tables T = tables_at(h_tab.data(), 1);
            if (T.status[0] != ZMT_ST_OK) return frame_error(c, T.status[0]);
            const uint64_t osz = T.out_size[0];
            if (osz > room) return frame_error(c, ZMT_ST_DST_SMALL);
            // ---- the history of the next segment: the last Window_Size bytes of [history | this segment], queued behind
            //      this segment, ahead of the next one (a reallocation of d_out in between synchronises in cudaFree)
            const uint64_t hnext = hlen + osz < t.window ? hlen + osz : t.window;
            if (!last && hnext) {
                if (!d_hist.need(hnext)) return c->E->mem;
                if (cudaMemcpyAsync(d_hist.p, (uint8_t*)d_out.p + hlen + osz - hnext, hnext, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
                    cudaGetLastError(); return frame_error(c, ZMT_ST_CUDA);
                }
            }
            const size_t we = write(out.data(), osz);
            if (we) return we;
            produced += osz;
            // ---- the table sources of the next segment: from this segment's bytes, or carried on from the current ones
            if (!last) {
                uint64_t to[4]; uint32_t tln[4];
                const uint32_t nt = zstd_walk_sources(&t, to, tln);
                next.clear();
                for (uint32_t i = 0; i < nt; i++) {
                    const uint8_t* b = nullptr;
                    if (to[i] >= seg_at) b = in.data() + 12 + pos + (to[i] - seg_at);
                    else for (uint32_t k = 0, at = 0; k < ns; at += sl[k], k++) if (so[k] == to[i]) b = carry.data() + at;
                    if (!b) return frame_error(c, ZMT_ST_BLOCK);
                    next.insert(next.end(), b, b + tln[i]);
                }
                carry.swap(next);
            }
            in.erase(in.begin() + 12, in.begin() + 12 + (long)(pos + end));       // drop the decoded segment
            pos = 0;
            w = t;
            if (last) return 0;
        }
    }
};

size_t decompress_single_stream(Ctx* c, GenRdWr* rw, const uint8_t* first, size_t have)
{
    const ErrCodes& E = *c->E;
    PlainStream S(c, rw, first, have);
    std::vector<uint8_t>& in = S.in;
    size_t& pos = S.pos;
    FrameList& fl = S.fl;
    const std::vector<int> devs = env_devices();
    if (devs.empty() || cudaSetDevice(devs[0]) != cudaSuccess) return frame_error(c, ZMT_ST_CUDA);
    if (cudaStreamCreateWithFlags(&S.st, cudaStreamNonBlocking) != cudaSuccess) return frame_error(c, ZMT_ST_CUDA);
    c->insize = have;

    for (;;) {
        // ---- cut complete frames out of what we hold, up to one batch
        fl.clear();
        const size_t batch_start = pos;
        bool need_more = false, segmented = false;
        while (!need_more) {
            const uint8_t* s = in.data() + 12; const size_t n = in.size() - 12;
            if (pos >= n) { need_more = !S.eof; break; }
            if (fl.n() && pos - batch_start >= S.batch) break;
            // the frame start: a skippable frame, or a codec frame whose head is usable (the rule the device's plain
            // index takes too, frame_format.h); a start cut short or a foreign magic is a data error of the stream
            uint64_t skip = 0;
            const int h = plain_frame_head(s + pos, n - pos, S.is_zstd, &skip);
            if (h == ZMT_ST_TRUNCATED) { if (S.eof) return E.data_error; need_more = true; break; }
            if (h == ZMT_ST_BAD_MAGIC) return E.data_error;
            if (h != ZMT_ST_OK) return frame_error(c, h);
            if (skip) { pos += (size_t)skip; continue; }
            if (!S.is_zstd) {
                const uint32_t flg = s[pos + 4], bd = s[pos + 5];
                {
                    // a frame whose blocks reach a batch of input or four of output before its end: decoded in segments,
                    // after the frames in front of it
                    Lz4fWalk w; w.pos = lz4f_header_len(flg); w.bound = 0; w.nblk = 0; w.done = 0;
                    if (lz4f_walk_blocks(s + pos, n - pos, flg, bd, &w, S.batch, 4 * (uint64_t)S.batch) && !w.done) {
                        if (fl.n()) break;
                        const size_t e = S.lz4_segments();
                        if (e) return e;
                        segmented = true; break;
                    }
                }
                uint64_t len = 0, osz = 0, stop = 0;
                const int r = lz4f_plain_frame(s + pos, n - pos, &len, &osz, &stop);
                if (r == ZMT_ST_TRUNCATED) {
                    if (S.eof) return frame_error(c, ZMT_ST_TRUNCATED);
                    need_more = true; break;
                }
                if (r != ZMT_ST_OK) return frame_error(c, r);
                fl.push(pos, (uint32_t)len, osz);
                pos += (size_t)len;
            } else {
                {
                    // a frame whose blocks reach a batch of input or four of output before its end: decoded in segments,
                    // after the frames in front of it
                    zmt_zstd_walk sw = {}; uint32_t nb = 0; uint64_t scr = 0, room = 0;
                    if (zstd_walk_blocks<false>(s + pos, n - pos, 0, 0, nullptr, &nb, 0xFFFFFFFFu, &scr, &sw, S.batch, 4 * (uint64_t)S.batch, &room) == ZMT_ST_OK &&
                        !sw.done) {
                        if (fl.n()) break;
                        const size_t e = S.zstd_segments();
                        if (e) return e;
                        segmented = true; break;
                    }
                }
                ZWalk w;
                int zr = zstd_blocks(fl, s + pos, n - pos, 12 + pos, S.blocks.data(), (uint32_t)S.blocks.size(), true, w);
                if (zr == ZMT_ST_DST_SMALL) {                     // block table full: grow it and walk once more
                    S.blocks.resize(w.nblk > 2 * S.blocks.size() + 4096 ? w.nblk : 2 * S.blocks.size() + 4096);
                    zr = zstd_blocks(fl, s + pos, n - pos, 12 + pos, S.blocks.data(), (uint32_t)S.blocks.size(), false, w);
                }
                if (zr == ZMT_ST_TRUNCATED && !S.eof) { need_more = true; break; }
                if (zr != ZMT_ST_OK) return frame_error(c, zr);
                fl.push(pos, w.flags, w.room, zstd_expect(w), w.nblk, w.scratch);
                pos += w.end;
            }
        }
        if (segmented) continue;                                              // a segmented frame was decoded and consumed
        if (fl.n() == 0) {
            if (!need_more) break;                                            // EOF, everything consumed
        } else {
            // ---- decode this batch (only its bytes travel) and write it frame by frame
            const size_t e = S.decode(in.data() + 12 + batch_start, 12 + batch_start, 12 + pos, nullptr);
            if (e) return e;
            const Tables T = tables_at(S.h_tab.data(), fl.n());
            for (uint32_t i = 0; i < fl.n(); i++) {
                if (T.status[i] != ZMT_ST_OK) return frame_error(c, T.status[i]);
                const size_t we = S.write(S.out.data() + T.out_off[i], T.out_size[i]);
                if (we) return we;
            }
            in.erase(in.begin() + 12, in.begin() + 12 + (long)pos);         // drop what has been decoded
            pos = 0;
        }
        if (need_more) {
            // ---- read ahead: at least one more piece, up to a batch beyond the parse position
            size_t goal = in.size() + S.piece;
            if (goal < 12 + pos + S.batch) goal = 12 + pos + S.batch;
            const size_t e = S.read_to(goal);
            if (e) return e;
        } else if (S.eof && pos >= in.size() - 12) break;
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
    // The decoded bytes come over in pieces of a few MiB, one piece ahead of the one being written: what fn_write's memcpy
    // reads was DMA-written moments ago and is still in the last-level cache, instead of a whole 64 MiB slot that was
    // copied long before its first byte is used.
    const uint64_t kPieceBytes = 2 << 20;

    // ---- stream-type sniffing on the calling thread (LZ4MT_decompressDCtx, lz4-mt_decompress.c:503-520;
    //      ZSTDCB_decompressDCtx, zstd-mt_decompress.c:721-759)
    uint8_t first[16]; size_t have = 0, got = 0;
    bool hdr_pending = false;                 // first 12-byte header already (partly) read into `first`
    size_t first_payload_have = 0;            // zstd pzstd-style: 4 payload bytes already read
    if (c->codec == CODEC_LZ4) {
        size_t e = read_some(E, rw, first, 4, &got); if (e) return e;
        if (got != 4) return E.data_error;
        if (zf_rd32(first) != ZMT_CONTAINER_MAGIC) {
            if (zf_rd32(first) != ZMT_LZ4F_MAGIC) return E.data_error;
            return decompress_single_stream(c, rw, first, 4);          // plain .lz4 stream (st_decompress, lz4-mt_decompress.c:512-520)
        }
        e = read_some(E, rw, first + 4, 8, &got); if (e) return e;
        if (got != 8) return E.read_fail;
        have = 12; hdr_pending = true;
    } else {
        size_t e = read_some(E, rw, first, 16, &got); if (e) return e;
        have = got;
        auto is_zstd = [](const uint8_t* p) { uint32_t m = zf_rd32(p); return m >= 0xFD2FB522u && m <= ZMT_ZSTD_MAGIC; };
        auto is_skip = [](const uint8_t* p) { return zf_rd32(p) == ZMT_CONTAINER_MAGIC && zf_rd32(p + 4) == 4; };
        if (have < 16) {
            if (have < 4 || !is_zstd(first)) return E.data_error;
            if (have == 9) return 0;                                   // empty file (zstd-mt_decompress.c:735-740)
            return decompress_single_stream(c, rw, first, have);       // short plain zstd stream
        }
        c->insize += 16;
        if (is_skip(first) && is_zstd(first + 12)) { hdr_pending = true; first_payload_have = 4; }          // pzstd style
        else if (is_zstd(first) && zf_rd32(first + 9) == ZMT_CONTAINER_MAGIC) {                                    // zstdmt style: 9-byte empty frame + 12-byte header
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
        if (c->devs.empty()) return frame_error(c, ZMT_ST_CUDA);
        const size_t base_slots = c->threads >= 4 ? 4 : c->threads >= 3 ? 3 : 2;       // see compress_run
        P.slots.resize(base_slots > c->devs.size() ? base_slots : c->devs.size());
        for (size_t i = 0; i < P.slots.size(); i++)
        {
            // zstd scratch: 16 B per sequence + the literals: ~2x the output on text, bounded at 3x + tables (the reader closes a batch early otherwise)
            const size_t wk = is_zstd ? zmt_zstdd_workspace_bytes((uint32_t)tab_cap, kBlkCap, 3 * (uint64_t)out_cap0) : zmt_lz4d_workspace_bytes((uint32_t)tab_cap, lz4_slot_cap(out_cap0, tab_cap), in_cap0);
            if (!slot_alloc(P.slots[i], c->devs[i % c->devs.size()], in_cap0, out_cap0, wk, tab_cap, nullptr) || (is_zstd && !slot_ensure_blocks(P.slots[i], kBlkCap))) {
                ctx_release_slots(c); return E.mem;
            }
            P.slots[i].scr_cap = is_zstd ? 3 * (uint64_t)P.slots[i].out_cap : 0;
        }
    }

    double rd_scan = 0;
    bool eof = false;
    std::vector<uint8_t> carry;              // a frame that did not fit the previous slot
    PipeOps po;
    // pt_read, lz4-mt_decompress.c:192-281 / zstd-mt_decompress.c:209-369
    po.fill = [&](Slot& slot) -> bool {
        if (eof) return false;
        Slot* s = &slot;
        FrameList& fl = s->frames;           // the slot is reallocated in place by grow(), only while the list is empty
        fl.clear();
        size_t in_used = 0, stat_in = 0;
        bool failed = false;
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
            if (!slot_alloc(*s, dev, nin, nout, wk, tc, nullptr) || (is_zstd && !slot_ensure_blocks(*s, nb))) return false;
            s->scr_cap = nscr;
            return true;
        };
        // the zstd payload p[0..len) at `at` in the slot's input, as the next frame: the block-table rule, and the payload
        // must hold the frame and nothing else
        auto zstd_payload = [&](const uint8_t* p, size_t len, uint64_t at, bool count, ZWalk& w) -> int {
            const int zr = zstd_blocks(fl, p, len, at + 12, s->h_blk, s->blk_cap, count, w);
            return zr == ZMT_ST_OK && w.end != len ? ZMT_ST_TRAILING : zr;
        };
        // Put one whole frame (12-byte header + payload, held in `fr`) at the start of the empty slot, growing the slot
        // (input, output, zstd block table and entropy scratch) so that it fits.  Returns false after P.fail().
        auto place_first = [&](const std::vector<uint8_t>& fr) -> bool {
            const size_t len = fr.size() - 12;
            if (!grow(fr.size(), 0, 0, 0)) { P.fail(E.mem); return false; }
            uint64_t room = 0; ZWalk w;
            if (!is_zstd) {
                if (!lz4f_out_size(fr.data() + 12, len, &room)) { P.fail(frame_error(c, ZMT_ST_BAD_HEADER)); return false; }
                if (!grow(fr.size(), room, 0, 0)) { P.fail(E.mem); return false; }
            } else {
                int zr = zstd_payload(fr.data() + 12, len, 0, true, w);
                if (zr == ZMT_ST_DST_SMALL || (zr == ZMT_ST_OK && (w.room > s->out_cap || w.scratch > s->scr_cap))) {
                    // more blocks than descriptors (every block costs >= 3 bytes), output or scratch: grow, walk once more
                    if (!grow(fr.size(), w.room, w.scratch, zr == ZMT_ST_DST_SMALL ? (uint32_t)(len / 3 + 16) : 0)) { P.fail(E.mem); return false; }
                    zr = zstd_payload(fr.data() + 12, len, 0, false, w);
                }
                if (zr != ZMT_ST_OK) { P.fail(frame_error(c, zr)); return false; }
                room = w.room;
            }
            memcpy(s->h_in, fr.data(), fr.size());
            fl.push(0, is_zstd ? w.flags : (uint32_t)len, room, zstd_expect(w), w.nblk, w.scratch);
            in_used = fr.size();
            return true;
        };
        if (!carry.empty()) {
            if (!place_first(carry)) return false;
            carry.clear();
        }
        while (fl.n() < s->tab_cap) {
            uint8_t hdr[12]; size_t pre = 0;
            if (hdr_pending) { memcpy(hdr, first, 12); hdr_pending = false; pre = first_payload_have; }
            else {
                size_t g = 0; size_t e = read_some(E, rw, hdr, 12, &g);
                if (e) { P.fail(e); failed = true; break; }
                if (g == 0) { eof = true; break; }
                if (g != 12) { P.fail(E.read_fail); failed = true; break; }
                if (zf_rd32(hdr) != ZMT_CONTAINER_MAGIC) { P.fail(E.data_error); failed = true; break; }
                if (c->codec == CODEC_ZSTD) stat_in += 12;
            }
            if (zf_rd32(hdr + 4) != 4) { P.fail(E.data_error); failed = true; break; }
            if (c->codec == CODEC_LZ4) stat_in += 12;
            const size_t toRead = zf_rd32(hdr + 8);
            if (toRead < pre) { P.fail(E.data_error); failed = true; break; }
            // where to put it: the current slot if it fits behind the frames already there, else a temporary buffer
            // (first frame of a batch that needs a bigger slot, or a frame that moves to the next batch)
            uint8_t* dstp; bool to_tmp = false;
            if (in_used + 12 + toRead <= s->in_cap) dstp = s->h_in + in_used;
            else { carry.resize(12 + toRead); dstp = carry.data(); to_tmp = true; }
            memcpy(dstp, hdr, 12);
            if (pre) memcpy(dstp + 12, first + 12, pre);
            size_t g = 0; size_t e = read_some(E, rw, dstp + 12 + pre, toRead - pre, &g);
            if (e) { P.fail(e); failed = true; break; }
            if (g != toRead - pre) { P.fail(E.data_error); failed = true; break; }
            stat_in += g;
            if (to_tmp) {
                if (fl.n() > 0) break;                              // next batch starts with it
                if (!place_first(carry)) { failed = true; break; }
                carry.clear();
                continue;
            }
            uint64_t room = 0; ZWalk w;
            bool moves = false;                                     // does not fit behind the others: first frame of the next batch
            if (!is_zstd) {
                if (!lz4f_out_size(dstp + 12, toRead, &room)) { P.fail(frame_error(c, ZMT_ST_BAD_HEADER)); failed = true; break; }
            } else {
                // block table of this frame (descriptors are appended; dropped again if the frame moves to the next batch)
                const double ts0 = trace_now();
                const int zr = zstd_payload(dstp + 12, toRead, in_used, false, w);
                rd_scan += trace_now() - ts0;
                if (zr == ZMT_ST_DST_SMALL) moves = true;
                else if (zr != ZMT_ST_OK) { P.fail(frame_error(c, zr)); failed = true; break; }
                else if (w.scratch > s->scr_cap) moves = true;
                room = w.room;
            }
            if (!moves && room > s->out_cap - fl.out_end()) moves = true;
            if (moves) {
                carry.assign(dstp, dstp + 12 + toRead);
                if (fl.n() > 0) break;
                if (!place_first(carry)) { failed = true; break; }  // a single frame larger than the slot: grow the slot
                carry.clear();
                continue;
            }
            fl.push(in_used, is_zstd ? w.flags : (uint32_t)toRead, room, zstd_expect(w), w.nblk, w.scratch);
            in_used += 12 + toRead;
        }
        if (failed || fl.n() == 0) return false;
        s->in_used = in_used;
        c->insize += stat_in; c->frames += fl.n();
        return true;
    };
    po.submit = [&](Slot& s) -> int {
        if (cudaMemcpyAsync(s.d_in, s.h_in, s.in_used, cudaMemcpyHostToDevice, s.stream) != cudaSuccess) return ZMT_ST_CUDA;
        const int st = decode_step(is_zstd, s.frames, s.h_tab, s.d_tab, s.tab_cap, s.h_blk, s.d_blk, s.d_in, s.in_used, s.d_out, s.d_work, nullptr, nullptr, s.stream);
        if (st != ZMT_ST_OK) return st;
        return cudaEventRecord(s.ev, s.stream) == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
    };
    // pt_write, lz4-mt_decompress.c:165-187
    po.drain = [&](Slot& s) -> bool {
        const Tables T = tables_at(s.h_tab, s.tab_cap);
        const uint32_t n = s.frames.n();
        uint32_t issued = 0, ready = 0; int np_issued = 0, np_ready = 0;       // frames [0, issued) requested, [0, ready) landed
        auto issue_piece = [&]() -> bool {
            if (issued >= n) return true;
            uint32_t j = issued; uint64_t lo = T.out_off[j], hi = lo;
            while (j < n && hi - lo < kPieceBytes) { hi = T.out_off[j] + T.out_size[j]; j++; }
            if (hi > s.out_cap) hi = s.out_cap;
            if (hi > lo && cudaMemcpyAsync(s.h_out + lo, s.d_out + lo, (size_t)(hi - lo), cudaMemcpyDeviceToHost, s.stream) != cudaSuccess) return false;
            if (cudaEventRecord(s.evp[np_issued & 1], s.stream) != cudaSuccess) return false;
            np_issued++; issued = j;
            return true;
        };
        uint32_t piece_end[2] = { 0, 0 };
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t st = T.status[i];
            if (st != ZMT_ST_OK) { P.fail(frame_error(c, st)); return false; }
            if (i >= ready) {
                bool okp = true;
                if (np_issued == np_ready) { okp = issue_piece(); piece_end[(np_issued - 1) & 1] = issued; }
                if (okp && issued < n && np_issued == np_ready + 1) { okp = issue_piece(); piece_end[(np_issued - 1) & 1] = issued; }   // one ahead
                if (okp) okp = cudaEventSynchronize(s.evp[np_ready & 1]) == cudaSuccess;
                if (!okp) { P.fail(frame_error(c, ZMT_ST_CUDA)); return false; }
                ready = piece_end[np_ready & 1]; np_ready++;
            }
            GenBuffer b; b.buf = s.h_out + T.out_off[i]; b.size = (size_t)T.out_size[i]; b.allocated = b.size;
            int rv = rw->fn_write(rw->arg_write, &b);
            if (rv != 0) { P.fail(mt_error(E, rv)); return false; }
            c->outsize += b.size; c->curframe++;
        }
        return true;
    };
    po.name = "decompress"; po.batch_bytes = in_cap0; po.scan = &rd_scan;
    return run_pipeline(c, P.slots.size(), po);
}

// ------------------------------------------------------------------ context helpers
Ctx* ctx_new(int codec, int threads, int level, size_t inputsize)
{
    Ctx* c = new (std::nothrow) Ctx();
    if (!c) return nullptr;
    c->codec = codec; c->threads = threads; c->level = level; c->inputsize = inputsize;
    c->E = codec == CODEC_LZ4 ? &kErrLz4 : &kErrZstd;
    return c;
}
void ctx_delete(Ctx* c) { if (!c) return; const DeviceRestore restore_device; ctx_release_slots(c); delete c; }

// Levels.  LZ4 has two search classes on the device: the greedy single-probe parse of levels 1-2 (levels 3-9 run it
// too) and the high-compression class of levels 10-12 (chunk-wide hash chains, a lazy parse, linked blocks).  zstd has two: levels 1-5
// run the level-3 class (the LZ4 parse + Huffman / predefined-FSE entropy stage, "level 3 (predefined FSE tables)" in
// BASELINE terms), levels 6-12 the chunk-wide hash-chain class with a lazy parse and per-level parameters, and levels
// 13-22 that class with level 12's parameters.  A level above what its class implements is accepted — the CLI default
// for lz4 is 3 (programs/lz4-mt.c:19) and must keep working — and produces that class's stream; that is said once per
// codec and class on stderr (ZSTDMT_B200_QUIET=1 silences it) instead of silently, and ZSTDMT_B200_STRICT_LEVEL=1 turns
// it into the reference's own answer for a bad parameter (create returns NULL, lib/lz4-mt_compress.c:103-108).
bool level_ok(int codec, int level)
{
    int implemented = level >= 10 ? 12 : 2, cls = 0;
    if (codec != CODEC_LZ4) { implemented = level >= 6 ? 12 : 3; cls = level >= 6 ? 2 : 1; }
    if (level <= implemented) return true;
    if (getenv("ZSTDMT_B200_STRICT_LEVEL")) return false;
    static std::atomic<int> told[3];
    if (!getenv("ZSTDMT_B200_QUIET") && told[cls].exchange(1) == 0)
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
    case ZMT_ST_DICT_WRONG: return "ERROR_dictionary_wrong";
    }
    return nullptr;
}

const char* error_string(bool lz4, size_t code, size_t lib_errcode)
{
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
    return ctx_new(CODEC_LZ4, threads, level, inputsize ? (size_t)inputsize : (size_t)4 << 20);
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
    return ctx_new(CODEC_LZ4, threads, 0, inputsize ? (size_t)inputsize : (size_t)64 << 10);
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
    return ctx_new(CODEC_ZSTD, threads, level, chunk);
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
    return ctx_new(CODEC_ZSTD, threads, 0, inputsize ? (size_t)inputsize : (size_t)512 << 10);
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
