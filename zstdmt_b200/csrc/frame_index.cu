// frame_index.cu — the decoders' tables, built on the GPU from a stream that is already in HBM.
//
// zmt_lz4_decompress_device and zmt_zstd_decompress_device take per-frame tables (and, for zstd, a block table) that the
// host pipeline builds while its reader walks the headers.  A caller whose stream reaches HBM some other way (GPUDirect
// Storage, NCCL, our own device compressor) builds them here instead, and the host learns only a summary to size its
// allocations with.  Container-framed streams:
//   zidx_walk_kernel          one thread follows the chain of 12-byte container headers (one dependent load per frame)
//   zidx_lz4_frames_kernel    one thread per frame: the LZ4F room rule (lz4f_out_size) and the block-table slot count
//   zidx_zstd_frames_kernel   one thread per frame: the counting walk of zstd_frame_walk (blocks, scratch, content size, flags)
// Plain streams (.lz4 / .zst files: codec frames and skippable frames back to back), where a frame's end is only known
// by walking its block headers:
//   zidx_plain_walk_kernel    one thread walks the stream with the host plain path's rule (plain_frame_head, then
//                             lz4f_plain_frame or the counting walk of zstd_frame_walk) and writes every per-frame entry
//   zidx_plain_tail_kernel    one thread per entry: zeroes the entries behind the stored frames for the scans
// Both then share:
//   cub::DeviceScan           exclusive sums in place: output offsets, first block, scratch bases, slots
//   zidx_summary_kernel       one thread: the first failure in stream order and the totals (zmt_frame_index)
//   zidx_zstd_blocks_kernel   one thread per frame: the writing walk of zstd_frame_walk fills the ZBlk table
// The header formats live in frame_format.h, shared with the host walkers, so both sources of tables agree byte for byte.
// The zstd kernels take a template flag D: D = true walks against the loaded dictionary dd (the *_dict_device calls),
// D = false is the walk without one and never reads dd.
#include <stdint.h>
#include "cub_scan.h"
#include "frame_format.h"
#include "launch.h"

namespace {

constexpr uint32_t kThreads = 128;
constexpr uint64_t kMaxIndexBytes = 3ull * 0xFFFFFFFFull;     // frames (>= 9 B), zstd blocks (>= 3 B) and LZ4 slots then fit in 32 bits

struct IdxCtl {
    uint32_t nframes;       // frames the walk accepted
    uint32_t cstatus;       // ZMT_ST_* of the walk
    uint32_t first_bad;     // lowest frame index whose per-frame pass failed (~0: none)
    uint32_t pad;
    uint64_t coff;          // stream offset where the walk stopped (on failure: where in the failing frame)
    uint64_t max_off;       // offset of frame max_frames' header (the first one not stored)
};

struct IdxWork { IdxCtl* ctl; uint32_t* fstat; uint64_t* fstop; uint64_t* slots; void* tmp; size_t tmp_bytes; };

// workspace (ZmtCarve, launch.h): ctl | per-frame status | per-frame stop offset | LZ4 slots (max_frames + 1) | cub scan
// storage.  Returns its size, 0 when cub cannot size its scans.
size_t carve(void* d_work, uint32_t max_frames, IdxWork* k)
{
    ZmtCarve c{(uint8_t*)d_work, 0};
    k->ctl = c.take<IdxCtl>(256);
    k->fstat = c.take<uint32_t>(a256((uint64_t)max_frames * 4));
    k->fstop = c.take<uint64_t>(a256((uint64_t)max_frames * 8));
    k->slots = c.take<uint64_t>(a256(((uint64_t)max_frames + 1) * 8));
    k->tmp_bytes = scan_tmp_bytes(max_frames + 1);
    k->tmp = c.take<void>(k->tmp_bytes);
    return k->tmp_bytes ? (size_t)c.off : 0;
}

__global__ void zidx_walk_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t max_frames, uint64_t* __restrict__ frame_off,
                                 uint32_t* __restrict__ frame_csize, IdxCtl* __restrict__ ctl)
{
    uint64_t pos = 0, max_off = 0;
    uint32_t n = 0, st = ZMT_ST_OK;
    while (pos < in_bytes) {
        if (in_bytes - pos < 12) { st = ZMT_ST_TRUNCATED; break; }
        const uint8_t* h = in + pos;
        if (zf_rd32(h) != ZMT_CONTAINER_MAGIC || zf_rd32(h + 4) != 4) { st = ZMT_ST_BAD_MAGIC; break; }
        const uint32_t cs = zf_rd32(h + 8);
        if (in_bytes - pos - 12 < cs) { st = ZMT_ST_TRUNCATED; break; }
        if (n < max_frames) { frame_off[n] = pos; frame_csize[n] = cs; }
        else if (n == max_frames) max_off = pos;
        n++; pos += 12 + (uint64_t)cs;
    }
    ctl->nframes = n; ctl->cstatus = st; ctl->first_bad = 0xFFFFFFFFu; ctl->coff = pos; ctl->max_off = max_off;
}

__device__ __forceinline__ void zidx_fail(IdxWork k, uint32_t f, uint32_t st, uint64_t at)
{
    k.fstat[f] = st; k.fstop[f] = at;
    atomicMin(&k.ctl->first_bad, f);
}

// f in [0, max_frames]: the entries behind the stored frames are zeroed, so the scans over max_frames + 1 entries leave
// the totals at index min(nframes, max_frames)
__global__ void __launch_bounds__(kThreads)
zidx_lz4_frames_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ frame_off, const uint32_t* __restrict__ frame_csize,
                       uint64_t* __restrict__ out_off, IdxWork k, uint32_t max_frames)
{
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    if (f > max_frames) return;
    const uint32_t stored = min(k.ctl->nframes, max_frames);
    uint64_t room = 0, slots = 0;
    if (f < stored) {
        const uint64_t p = frame_off[f] + 12;
        if (lz4f_out_size(in + p, frame_csize[f], &room)) slots = lz4_frame_slots(room);
        else { room = 0; zidx_fail(k, f, ZMT_ST_BAD_HEADER, p); }
    }
    out_off[f] = room; k.slots[f] = slots;
}

template <bool D>
__global__ void __launch_bounds__(kThreads)
zidx_zstd_frames_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ frame_off, const uint32_t* __restrict__ frame_csize,
                        uint32_t* __restrict__ first_blk, uint64_t* __restrict__ frame_scratch, uint64_t* __restrict__ expect,
                        uint32_t* __restrict__ frame_seq, uint64_t* __restrict__ out_off, IdxWork k, uint32_t max_frames, const ZDDict* __restrict__ dd)
{
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    if (f > max_frames) return;
    const uint32_t stored = min(k.ctl->nframes, max_frames);
    uint32_t nb = 0, flags = 0; uint64_t scr = 0, cs = 0;
    if (f < stored) {
        const uint64_t p = frame_off[f] + 12;
        const uint32_t n = frame_csize[f];
        size_t end = 0;
        int r = zstd_frame_walk<false, D>(in + p, n, p, f, nullptr, &nb, 0xFFFFFFFFu, &scr, &cs, &flags, &end, D ? &dd->info : nullptr);
        if (r == ZMT_ST_OK && end != n) r = ZMT_ST_TRAILING;
        if (r != ZMT_ST_OK) { nb = 0; scr = 0; cs = 0; flags = 0; zidx_fail(k, f, (uint32_t)r, p + end); }
    }
    first_blk[f] = nb; frame_scratch[f] = scr; out_off[f] = cs;
    if (f < max_frames) { expect[f] = (flags & ZF_NO_SIZE) ? ~0ull : cs; frame_seq[f] = flags; }
}

// The plain stream in[0..in_bytes): skippable frames are stepped over, every codec frame is decided by the host plain
// path's rule, and the first failure ends the walk (the next frame's start is not known behind it).  Frame f < max_frames
// gets its offset, length, room and (LZ4) slot count or (zstd) block count, scratch, expect and flags; the scans make the
// counts bases.  The decode calls take frame_csize as 32 bits: a frame of 2^32 bytes or more is ZMT_ST_UNSUPPORTED.
template <bool Z, bool D>
__global__ void zidx_plain_walk_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t max_frames, uint64_t* __restrict__ frame_off,
                                       uint32_t* __restrict__ frame_csize, uint64_t* __restrict__ out_off, uint64_t* __restrict__ slots,
                                       uint32_t* __restrict__ first_blk, uint64_t* __restrict__ frame_scratch, uint64_t* __restrict__ expect,
                                       uint32_t* __restrict__ frame_seq, IdxCtl* __restrict__ ctl, const ZDDict* __restrict__ dd)
{
    uint64_t pos = 0, max_off = 0, at = 0;
    uint32_t n = 0, st = ZMT_ST_OK;
    while (pos < in_bytes) {
        const uint8_t* p = in + pos;
        const uint64_t rem = in_bytes - pos;
        uint64_t skip = 0;
        st = (uint32_t)plain_frame_head(p, rem, Z, &skip);
        if (st != ZMT_ST_OK) { at = pos; break; }
        if (skip) { pos += skip; continue; }
        uint64_t len = 0, room = 0, scr = 0;
        uint32_t nb = 0, flags = 0;
        if (Z) {
            size_t end = 0;
            st = (uint32_t)zstd_frame_walk<false, D>(p, rem, 0, 0, nullptr, &nb, 0xFFFFFFFFu, &scr, &room, &flags, &end, D ? &dd->info : nullptr);
            len = end; at = pos + end;
        } else {
            uint64_t stop = 0;
            st = (uint32_t)lz4f_plain_frame(p, rem, &len, &room, &stop);
            at = pos + stop;
        }
        if (st != ZMT_ST_OK) break;
        if (len > 0xFFFFFFFFull) { st = ZMT_ST_UNSUPPORTED; at = pos; break; }
        if (n < max_frames) {
            frame_off[n] = pos; frame_csize[n] = (uint32_t)len; out_off[n] = room;
            if (Z) { first_blk[n] = nb; frame_scratch[n] = scr; expect[n] = (flags & ZF_NO_SIZE) ? ~0ull : room; frame_seq[n] = flags; }
            else slots[n] = lz4_frame_slots(room);
        } else if (n == max_frames) max_off = pos;
        n++; pos += len;
    }
    ctl->nframes = n; ctl->cstatus = st; ctl->first_bad = 0xFFFFFFFFu; ctl->coff = st == ZMT_ST_OK ? pos : at; ctl->max_off = max_off;
}

// f in [min(nframes, max_frames), max_frames]: the entries behind the stored frames are zeroed, as the frame passes of
// the container path do, so the scans over max_frames + 1 entries leave the totals at index min(nframes, max_frames)
__global__ void __launch_bounds__(kThreads)
zidx_plain_tail_kernel(IdxWork k, uint32_t max_frames, uint64_t* __restrict__ out_off, uint32_t* __restrict__ first_blk, uint64_t* __restrict__ frame_scratch)
{
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    if (f > max_frames || f < min(k.ctl->nframes, max_frames)) return;
    out_off[f] = 0;
    if (first_blk) { first_blk[f] = 0; frame_scratch[f] = 0; }
    else k.slots[f] = 0;
}

__global__ void zidx_summary_kernel(IdxWork k, uint32_t max_frames, const uint64_t* __restrict__ out_off, const uint32_t* __restrict__ first_blk,
                                    const uint64_t* __restrict__ frame_scratch, zmt_frame_index* __restrict__ info)
{
    const IdxCtl c = *k.ctl;
    const uint32_t stored = min(c.nframes, max_frames);
    zmt_frame_index r;
    r.status = c.cstatus; r.bad_frame = c.nframes; r.bad_offset = c.cstatus == ZMT_ST_OK ? 0 : c.coff;
    if (c.nframes > max_frames) { r.status = ZMT_ST_DST_SMALL; r.bad_frame = max_frames; r.bad_offset = c.max_off; }
    if (c.first_bad < stored) { r.status = k.fstat[c.first_bad]; r.bad_frame = c.first_bad; r.bad_offset = k.fstop[c.first_bad]; }
    r.nframes = c.nframes;
    r.out_bytes = out_off[stored];
    if (first_blk) { r.nblocks = first_blk[stored]; r.scratch_bytes = frame_scratch[stored]; }
    else { r.nblocks = (uint32_t)k.slots[stored]; r.scratch_bytes = 0; }
    *info = r;
}

template <bool D>
__global__ void __launch_bounds__(kThreads)
zidx_zstd_blocks_kernel(const uint8_t* __restrict__ in, uint32_t nframes, const uint64_t* __restrict__ frame_off, const uint32_t* __restrict__ frame_csize,
                        const uint32_t* __restrict__ first_blk, const uint64_t* __restrict__ frame_scratch, ZBlk* __restrict__ blocks, uint32_t nblocks,
                        const ZDDict* __restrict__ dd)
{
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    if (f >= nframes) return;
    const uint64_t p = frame_off[f] + 12;
    uint32_t nb = first_blk[f], flags = 0;
    const uint32_t lim = min(first_blk[f + 1], nblocks);
    uint64_t scr = frame_scratch[f], cs = 0;
    size_t end = 0;
    zstd_frame_walk<true, D>(in + p, frame_csize[f], p, f, blocks, &nb, lim, &scr, &cs, &flags, &end, D ? &dd->info : nullptr);
}

// The common part of the index calls: the walk, the per-frame pass, scans, summary.  walk(k) enqueues the walk,
// pass(grid, k) the per-frame pass over max_frames + 1 entries.
template <typename Walk, typename FramePass>
int index_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize, uint64_t* d_out_off,
                 uint32_t* d_first_blk, uint64_t* d_frame_scratch, zmt_frame_index* d_info, void* d_work, cudaStream_t stream, Walk walk, FramePass pass)
{
    if (in_bytes > kMaxIndexBytes || max_frames >= 0x7FFFFFFFu || !d_info || !d_work || !d_out_off || (max_frames && (!d_frame_off || !d_frame_csize)))
        return ZMT_ST_BAD_ARG;
    IdxWork k;
    if (!carve(d_work, max_frames, &k)) return ZMT_ST_CUDA;
    const uint64_t n = (uint64_t)max_frames + 1;
    ZmtProfScope ps(ZMT_K_FRAME_INDEX, stream);
    walk(k);
    pass((max_frames + kThreads) / kThreads, k);
    bool ok = exclusive_sum(k, d_out_off, n, stream);
    if (d_first_blk) ok = ok && exclusive_sum(k, d_first_blk, n, stream) && exclusive_sum(k, d_frame_scratch, n, stream);
    else ok = ok && exclusive_sum(k, k.slots, n, stream);
    zidx_summary_kernel<<<1, 1, 0, stream>>>(k, max_frames, d_out_off, d_first_blk, d_frame_scratch, d_info);
    return ok && cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

void container_walk(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize, IdxWork k, cudaStream_t stream)
{
    zidx_walk_kernel<<<1, 1, 0, stream>>>((const uint8_t*)d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, k.ctl);
}

}  // namespace

extern "C" size_t zmt_index_workspace_bytes(uint32_t max_frames)
{
    if (max_frames >= 0x7FFFFFFFu) return 0;
    IdxWork k;
    return carve(nullptr, max_frames, &k);
}

extern "C" int zmt_lz4_index_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                    uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    return index_device(d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_out_off, nullptr, nullptr, d_info, d_work, stream,
                        [&](IdxWork k) { container_walk(d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, k, stream); },
                        [&](uint32_t grid, IdxWork k) {
                            zidx_lz4_frames_kernel<<<grid, kThreads, 0, stream>>>((const uint8_t*)d_in, d_frame_off, d_frame_csize, d_out_off, k, max_frames);
                        });
}

// The zstd index calls: container (plain = false) or plain stream, against the dictionary dd or without one.
static int zstd_index(bool plain, const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
               uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq, uint64_t* d_out_off,
               zmt_frame_index* d_info, void* d_work, cudaStream_t stream, const ZDDict* dd)
{
    if (!d_frame_first_blk || !d_frame_scratch || (max_frames && (!d_expect || !d_frame_seq))) return ZMT_ST_BAD_ARG;
    return index_device(d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_out_off, d_frame_first_blk, d_frame_scratch, d_info, d_work, stream,
                        [&](IdxWork k) {
                            if (!plain) container_walk(d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, k, stream);
                            else (dd ? zidx_plain_walk_kernel<true, true> : zidx_plain_walk_kernel<true, false>)<<<1, 1, 0, stream>>>(
                                (const uint8_t*)d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_out_off, k.slots, d_frame_first_blk,
                                d_frame_scratch, d_expect, d_frame_seq, k.ctl, dd);
                        },
                        [&](uint32_t grid, IdxWork k) {
                            if (plain) zidx_plain_tail_kernel<<<grid, kThreads, 0, stream>>>(k, max_frames, d_out_off, d_frame_first_blk, d_frame_scratch);
                            else if (dd) zidx_zstd_frames_kernel<true><<<grid, kThreads, 0, stream>>>(
                                (const uint8_t*)d_in, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_expect, d_frame_seq, d_out_off,
                                k, max_frames, dd);
                            else zidx_zstd_frames_kernel<false><<<grid, kThreads, 0, stream>>>(
                                (const uint8_t*)d_in, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_expect, d_frame_seq, d_out_off,
                                k, max_frames, nullptr);
                        });
}

extern "C" int zmt_zstd_index_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                     uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                                     uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream)
{
    return zstd_index(false, d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_expect, d_frame_seq,
                      d_out_off, d_info, d_work, (cudaStream_t)stream, nullptr);
}

extern "C" int zmt_zstd_index_dict_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                          uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                                          uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream, const void* d_ddict)
{
    return zstd_index(false, d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_expect, d_frame_seq,
                      d_out_off, d_info, d_work, (cudaStream_t)stream, (const ZDDict*)d_ddict);
}

extern "C" int zmt_lz4_index_plain_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                          uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    return index_device(d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_out_off, nullptr, nullptr, d_info, d_work, stream,
                        [&](IdxWork k) {
                            zidx_plain_walk_kernel<false, false><<<1, 1, 0, stream>>>((const uint8_t*)d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_out_off,
                                                                               k.slots, nullptr, nullptr, nullptr, nullptr, k.ctl, nullptr);
                        },
                        [&](uint32_t grid, IdxWork k) { zidx_plain_tail_kernel<<<grid, kThreads, 0, stream>>>(k, max_frames, d_out_off, nullptr, nullptr); });
}

extern "C" int zmt_zstd_index_plain_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                           uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                                           uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream)
{
    return zstd_index(true, d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_expect, d_frame_seq,
                      d_out_off, d_info, d_work, (cudaStream_t)stream, nullptr);
}

extern "C" int zmt_zstd_index_plain_dict_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                                uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                                                uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream, const void* d_ddict)
{
    return zstd_index(true, d_in, in_bytes, max_frames, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_expect, d_frame_seq,
                      d_out_off, d_info, d_work, (cudaStream_t)stream, (const ZDDict*)d_ddict);
}

extern "C" int zmt_zstd_blocks_dict_device(const void* d_in, uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                                           const uint32_t* d_frame_first_blk, const uint64_t* d_frame_scratch, void* d_blocks, uint32_t nblocks, void* stream_,
                                           const void* d_ddict)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    if (nframes == 0 || nblocks == 0) return ZMT_ST_OK;
    if (!d_in || !d_frame_off || !d_frame_csize || !d_frame_first_blk || !d_frame_scratch || !d_blocks) return ZMT_ST_BAD_ARG;
    const ZDDict* dd = (const ZDDict*)d_ddict;
    ZmtProfScope ps(ZMT_K_FRAME_INDEX, stream);
    (dd ? zidx_zstd_blocks_kernel<true> : zidx_zstd_blocks_kernel<false>)<<<(nframes + kThreads - 1) / kThreads, kThreads, 0, stream>>>(
        (const uint8_t*)d_in, nframes, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, (ZBlk*)d_blocks, nblocks, dd);
    return cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

extern "C" int zmt_zstd_blocks_device(const void* d_in, uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                                      const uint32_t* d_frame_first_blk, const uint64_t* d_frame_scratch, void* d_blocks, uint32_t nblocks, void* stream)
{
    return zmt_zstd_blocks_dict_device(d_in, nframes, d_frame_off, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_blocks, nblocks, stream, nullptr);
}
