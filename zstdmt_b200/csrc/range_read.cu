// range_read.cu — byte ranges of a compressed stream in HBM, decoding only the frames that hold them.
//
// A frame is the unit of access: its content position comes from the content sizes of the frames before it, and its
// bytes only from decoding it whole.  So a batch of ranges maps to a set of frames, each decoded once by the existing
// decoders, and a gather copies the ranges out of their content.  On top of the device frame index (frame_index.cu):
//   content table  rr_content_kernel     one thread per frame: the content size its header states (frame_format.h)
//                  cub::DeviceScan       exclusive sum in place: d_content_off
//                  rr_content_summary    one thread: the first frame without a usable size, the total
//   plan           rr_ranges_kernel      one thread per range: validation, binary search for the first and last frame it
//                                        touches, +1 / -1 at the ends of that span, its length and gather pieces
//                  cub::DeviceScan       exclusive sum of the +1 / -1 marks: how many ranges touch each frame
//                  rr_frames_kernel      one thread per frame: selected or not, and what a selected frame adds to the
//                                        selection's tables (content, packed bytes, LZ4 slots or zstd blocks, scratch)
//                  cub::DeviceScan       exclusive sums: selected index, content, packed offset, units, scratch, dst_off,
//                                        pieces
//                  rr_compact_kernel     one thread per frame: the selected frames' decode tables, in stream order
//                  rr_plan_summary       one thread: the zmt_range_plan the host reads back
//   read           rr_pack_kernel        LZ4: the selected frames back to back in a staging buffer, a CTA per 128 KiB piece
//                  rr_select_kernel      zstd: the selected frames' offsets, sizes and flags from the index tables
//                  the decoders          zmt_lz4_decompress_device / zmt_zstd_blocks_device + zmt_zstd_decompress_device
//                  rr_fail_kernel, scan  which selected frames failed, as a prefix count
//                  rr_status_kernel      one thread per range: its status (a search over the failure prefix) and source
//                  rr_gather_kernel      a CTA per piece of at most 64 KiB: the range's bytes to dst + dst_off[r]
#include <stdint.h>
#include "cub_scan.h"
#include "frame_format.h"
#include "launch.h"

namespace {

constexpr uint32_t kThreads = 128;
constexpr uint32_t kCopyThreads = 256;                  // CTA of the pack and gather kernels: 8 warps
constexpr uint64_t kPiece = 64 * 1024;                  // gather piece: the most one CTA copies of one range
constexpr uint64_t kPackPiece = 128 * 1024;             // pack: the most one CTA copies of one frame
constexpr uint64_t kMaxExpand = 32768;                  // content bytes per compressed byte no frame can exceed (zstd RLE: 4 B -> 128 KiB)

__host__ __device__ inline uint64_t a16(uint64_t x) { return (x + 15) & ~15ull; }

struct RangeCtl {
    uint32_t first_bad_frame;   // content table: lowest frame without a usable content size (~0: none)
    uint32_t pad0;
    uint32_t first_bad_range;   // plan: lowest bad range (~0: none)
    uint32_t pad;
};

// The plan's workspace, carved the same way by the plan and the read call from (nframes, nranges).  F = nframes + 1
// entries per frame array (entry nframes holds the totals after the scans), R = nranges + 1 per range array.
struct RangeWork {
    RangeCtl* ctl;
    uint32_t* cover;        // +1 / -1 marks (mod 2^32), then their exclusive prefix: cover[f + 1] = the ranges touching frame f
    uint32_t* selx;         // 1 for a selected frame, then its index among the selected
    uint64_t* f_out;        // a selected frame's content size, then its offset in the scratch
    uint64_t* f_pack;       // LZ4: a selected frame's packed size (16 + its payload, 16-aligned), then its packed offset
    uint32_t* f_units;      // a selected frame's LZ4 slots / zstd blocks, then their base
    uint64_t* f_scr;        // zstd: a selected frame's entropy scratch, then its base
    // the selected frames' decode tables (index s < nsel; entry nsel holds the totals)
    uint32_t* sel_src;      // the frame of the stream
    uint64_t* sel_frame_off;
    uint32_t* sel_csize;
    uint64_t* sel_out_off;
    uint32_t* sel_first_blk;
    uint64_t* sel_scratch;
    uint64_t* sel_expect;
    uint32_t* sel_seq;
    uint64_t* sel_out_size;
    uint32_t* sel_status;
    uint32_t* sel_fail;     // 1 for a failed selected frame, then the number of failures before it
    // per range
    uint32_t* r_fa;         // first and last frame it touches
    uint32_t* r_fb;
    uint64_t* r_skip;       // its start's offset in frame r_fa's content
    uint64_t* r_len;        // its length (0 for a bad range)
    uint32_t* r_st;         // ZMT_ST_OK or ZMT_ST_BAD_ARG
    uint64_t* r_src;        // read: its start in the scratch
    uint64_t* r_piece;      // its gather pieces, then their base
    void*     tmp;
    size_t    tmp_bytes;
};

template <typename T>
T* take(ZmtCarve& w, uint64_t n) { return w.take<T>(a256(n * sizeof(T))); }

// returns the workspace's size (ZmtCarve, launch.h), 0 when cub cannot size its scans
size_t carve(void* d_work, uint32_t nframes, uint32_t nranges, RangeWork* k)
{
    ZmtCarve w{(uint8_t*)d_work, 0};
    const uint64_t F = (uint64_t)nframes + 1, R = (uint64_t)nranges + 1;
    k->ctl = take<RangeCtl>(w, 1);
    k->cover = take<uint32_t>(w, F); k->selx = take<uint32_t>(w, F); k->f_out = take<uint64_t>(w, F); k->f_pack = take<uint64_t>(w, F);
    k->f_units = take<uint32_t>(w, F); k->f_scr = take<uint64_t>(w, F);
    k->sel_src = take<uint32_t>(w, F); k->sel_frame_off = take<uint64_t>(w, F); k->sel_csize = take<uint32_t>(w, F);
    k->sel_out_off = take<uint64_t>(w, F); k->sel_first_blk = take<uint32_t>(w, F); k->sel_scratch = take<uint64_t>(w, F);
    k->sel_expect = take<uint64_t>(w, F); k->sel_seq = take<uint32_t>(w, F); k->sel_out_size = take<uint64_t>(w, F);
    k->sel_status = take<uint32_t>(w, F); k->sel_fail = take<uint32_t>(w, F);
    k->r_fa = take<uint32_t>(w, R); k->r_fb = take<uint32_t>(w, R); k->r_skip = take<uint64_t>(w, R); k->r_len = take<uint64_t>(w, R);
    k->r_st = take<uint32_t>(w, R); k->r_src = take<uint64_t>(w, R); k->r_piece = take<uint64_t>(w, R);
    k->tmp_bytes = scan_tmp_bytes((uint32_t)(F > R ? F : R));
    k->tmp = w.take<void>(k->tmp_bytes);
    return k->tmp_bytes ? (size_t)w.off : 0;
}

bool too_many(uint32_t nframes, uint32_t nranges) { return nframes >= 0x7FFFFFFFu || nranges >= 0x7FFFFFFFu; }

// ---------------------------------------------------------------- content table
// f < nframes: frame f's content size (LZ4: from its LZ4F header; zstd: the index's d_expect, ~0 without a size), or 0
// and a failure; f == nframes: 0, so the exclusive scan leaves the total there
template <bool Z>
__global__ void __launch_bounds__(kThreads)
rr_content_kernel(const uint8_t* __restrict__ in, uint32_t nframes, const uint64_t* __restrict__ frame_off, const uint32_t* __restrict__ frame_csize,
                  const uint64_t* __restrict__ expect, uint64_t* __restrict__ content_off, uint32_t* __restrict__ fstat, RangeCtl* __restrict__ ctl)
{
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    if (f > nframes) return;
    uint64_t cs = 0;
    uint32_t st = ZMT_ST_OK;
    if (f < nframes) {
        const uint32_t n = frame_csize[f];
        bool has;
        if (Z) { cs = expect[f]; has = cs != ~0ull; }
        else has = lz4f_known_content_size(in + frame_off[f] + 12, n, &cs);
        if (!has) st = ZMT_ST_UNSUPPORTED;
        else if (cs > (uint64_t)n * kMaxExpand) st = ZMT_ST_CONTENT_SIZE;
        if (st != ZMT_ST_OK) { cs = 0; fstat[f] = st; atomicMin(&ctl->first_bad_frame, f); }
    }
    content_off[f] = cs;
}

__global__ void rr_content_summary(uint32_t nframes, const uint64_t* __restrict__ frame_off, const uint64_t* __restrict__ content_off,
                                   const uint32_t* __restrict__ fstat, const RangeCtl* __restrict__ ctl, zmt_frame_index* __restrict__ info)
{
    const uint32_t bad = ctl->first_bad_frame;
    zmt_frame_index r;
    r.status = bad < nframes ? fstat[bad] : ZMT_ST_OK;
    r.bad_frame = bad < nframes ? bad : nframes;
    r.bad_offset = bad < nframes ? frame_off[bad] : 0;
    r.nframes = nframes; r.nblocks = 0;
    r.out_bytes = content_off[nframes]; r.scratch_bytes = 0;
    *info = r;
}

template <bool Z>
int content_offsets(const void* d_in, uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, const uint64_t* d_expect,
                    uint64_t* d_content_off, zmt_frame_index* d_info, void* d_work, cudaStream_t stream)
{
    if (too_many(nframes, 0) || !d_content_off || !d_info || !d_work) return ZMT_ST_BAD_ARG;
    if (nframes && (!d_frame_off || !d_frame_csize || (Z ? !d_expect : !d_in))) return ZMT_ST_BAD_ARG;
    RangeWork k;
    if (!carve(d_work, nframes, 0, &k)) return ZMT_ST_CUDA;
    ZmtProfScope ps(ZMT_K_FRAME_INDEX, stream);
    cudaMemsetAsync(k.ctl, 0xFF, sizeof(RangeCtl), stream);
    rr_content_kernel<Z><<<(nframes + kThreads) / kThreads, kThreads, 0, stream>>>((const uint8_t*)d_in, nframes, d_frame_off, d_frame_csize,
                                                                                  d_expect, d_content_off, k.selx, k.ctl);
    const bool ok = exclusive_sum(k, d_content_off, (uint64_t)nframes + 1, stream);
    rr_content_summary<<<1, 1, 0, stream>>>(nframes, d_frame_off, d_content_off, k.selx, k.ctl, d_info);
    return ok && cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

// ---------------------------------------------------------------- plan
// first index i in [lo, hi) with a[i] > v (hi if none)
__device__ __forceinline__ uint32_t upper_bound(const uint64_t* __restrict__ a, uint32_t lo, uint32_t hi, uint64_t v)
{
    while (lo < hi) { const uint32_t m = lo + (hi - lo) / 2; if (a[m] > v) hi = m; else lo = m + 1; }
    return lo;
}

// r < nranges: range r validated; a good non-empty range [start, end) touches the frames fa..fb, fa the first whose content
// ends past start, fb the last whose content starts before end (the zero-size frames between them included), and marks
// them +1 at fa, -1 at fb + 1.  r == nranges: the zero entries behind the ranges for the scans.
__global__ void __launch_bounds__(kThreads)
rr_ranges_kernel(uint32_t nframes, const uint64_t* __restrict__ content_off, const uint64_t* __restrict__ ranges, uint32_t nranges,
                 uint64_t* __restrict__ dst_off, RangeWork k)
{
    const uint32_t r = blockIdx.x * kThreads + threadIdx.x;
    if (r > nranges) return;
    uint64_t len = 0, pieces = 0, skip = 0;
    uint32_t st = ZMT_ST_OK, fa = 0, fb = 0;
    if (r < nranges) {
        const uint64_t start = ranges[2 * (uint64_t)r], n = ranges[2 * (uint64_t)r + 1], end = start + n;
        if (end < start || end > content_off[nframes]) {
            st = ZMT_ST_BAD_ARG;
            atomicMin(&k.ctl->first_bad_range, r);
        } else if (n) {
            fa = upper_bound(content_off, 1, nframes + 1, start) - 1;
            fb = upper_bound(content_off, fa + 1, nframes + 1, end - 1) - 1;
            skip = start - content_off[fa];
            len = n; pieces = (n + kPiece - 1) / kPiece;
            atomicAdd(&k.cover[fa], 1u);
            atomicSub(&k.cover[fb + 1], 1u);
        }
        k.r_fa[r] = fa; k.r_fb[r] = fb; k.r_skip[r] = skip; k.r_len[r] = len; k.r_st[r] = st;
    }
    dst_off[r] = len; k.r_piece[r] = pieces;
}

// f <= nframes: what frame f adds to the selection (0 unless it is selected; entry nframes stays 0 for the totals)
template <bool Z>
__global__ void __launch_bounds__(kThreads)
rr_frames_kernel(uint32_t nframes, const uint32_t* __restrict__ frame_csize, const uint32_t* __restrict__ first_blk,
                 const uint64_t* __restrict__ frame_scratch, const uint64_t* __restrict__ content_off, RangeWork k)
{
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    if (f > nframes) return;
    const bool sel = f < nframes && k.cover[f + 1] != 0;
    uint64_t out = 0, pack = 0, scr = 0;
    uint32_t units = 0;
    if (sel) {
        out = content_off[f + 1] - content_off[f];
        if (Z) { units = first_blk[f + 1] - first_blk[f]; scr = frame_scratch[f + 1] - frame_scratch[f]; }
        else { units = (uint32_t)lz4_frame_slots(out); pack = 16 + a16(frame_csize[f]); }
    }
    k.selx[f] = sel ? 1u : 0u; k.f_out[f] = out; k.f_pack[f] = pack; k.f_units[f] = units; k.f_scr[f] = scr;
}

// The selected frames' tables at their index s = selx[f]; frame nframes writes the totals at s = nsel.  LZ4: the packed
// stream holds selected frame s's container header at f_pack + 4 and its payload at f_pack + 16 (16-aligned), so its
// frame_off in the packed stream is f_pack + 4.
template <bool Z>
__global__ void __launch_bounds__(kThreads)
rr_compact_kernel(uint32_t nframes, const uint32_t* __restrict__ frame_csize, RangeWork k)
{
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    if (f > nframes) return;
    if (f < nframes && k.selx[f + 1] == k.selx[f]) return;
    const uint32_t s = k.selx[f];
    k.sel_out_off[s] = k.f_out[f]; k.sel_first_blk[s] = k.f_units[f]; k.sel_scratch[s] = k.f_scr[f];
    if (f == nframes) return;
    k.sel_src[s] = f; k.sel_csize[s] = frame_csize[f];
    if (!Z) k.sel_frame_off[s] = k.f_pack[f] + 4;
}

__global__ void rr_plan_summary(uint32_t nframes, uint32_t nranges, const uint64_t* __restrict__ dst_off, RangeWork k, zmt_range_plan* __restrict__ plan)
{
    zmt_range_plan p;
    const uint32_t bad = k.ctl->first_bad_range;
    p.status = bad < nranges ? ZMT_ST_BAD_ARG : ZMT_ST_OK;
    p.bad_range = bad < nranges ? bad : nranges;
    p.nframes = nframes; p.nranges = nranges;
    p.nsel = k.selx[nframes]; p.nunits = k.f_units[nframes];
    p.packed_bytes = k.f_pack[nframes]; p.scratch_bytes = k.f_out[nframes]; p.dec_scratch = k.f_scr[nframes];
    p.dst_bytes = dst_off[nranges]; p.npieces = k.r_piece[nranges];
    *plan = p;
}

template <bool Z>
int range_plan(uint32_t nframes, const uint32_t* d_frame_csize, const uint32_t* d_first_blk, const uint64_t* d_frame_scratch,
               const uint64_t* d_content_off, const uint64_t* d_ranges, uint32_t nranges, uint64_t* d_dst_off, zmt_range_plan* d_plan,
               void* d_work, cudaStream_t stream)
{
    if (too_many(nframes, nranges) || !d_content_off || !d_dst_off || !d_plan || !d_work || (nranges && !d_ranges)) return ZMT_ST_BAD_ARG;
    if (nframes && (!d_frame_csize || (Z && (!d_first_blk || !d_frame_scratch)))) return ZMT_ST_BAD_ARG;
    RangeWork k;
    if (!carve(d_work, nframes, nranges, &k)) return ZMT_ST_CUDA;
    const uint64_t F = (uint64_t)nframes + 1, R = (uint64_t)nranges + 1;
    ZmtProfScope ps(ZMT_K_FRAME_INDEX, stream);
    cudaMemsetAsync(k.ctl, 0xFF, sizeof(RangeCtl), stream);
    cudaMemsetAsync(k.cover, 0, F * sizeof(uint32_t), stream);
    rr_ranges_kernel<<<(nranges + kThreads) / kThreads, kThreads, 0, stream>>>(nframes, d_content_off, d_ranges, nranges, d_dst_off, k);
    bool ok = exclusive_sum(k, k.cover, F, stream);
    rr_frames_kernel<Z><<<(nframes + kThreads) / kThreads, kThreads, 0, stream>>>(nframes, d_frame_csize, d_first_blk, d_frame_scratch, d_content_off, k);
    ok = ok && exclusive_sum(k, k.selx, F, stream) && exclusive_sum(k, k.f_out, F, stream) && exclusive_sum(k, k.f_units, F, stream);
    ok = ok && (Z ? exclusive_sum(k, k.f_scr, F, stream) : exclusive_sum(k, k.f_pack, F, stream));
    ok = ok && exclusive_sum(k, d_dst_off, R, stream) && exclusive_sum(k, k.r_piece, R, stream);
    rr_compact_kernel<Z><<<(nframes + kThreads) / kThreads, kThreads, 0, stream>>>(nframes, d_frame_csize, k);
    rr_plan_summary<<<1, 1, 0, stream>>>(nframes, nranges, d_dst_off, k, d_plan);
    return ok && cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

// ---------------------------------------------------------------- read
// Bytes [sh, sh + 16) of the 32 bytes a || b (little endian), 0 < sh < 16.
__device__ __forceinline__ uint4 byte_window(const uint4 a, const uint4 b, uint32_t sh)
{
    const uint32_t r = (sh & 3) * 8;
    uint32_t w0, w1, w2, w3, w4;
    switch (sh >> 2) {
        case 0: w0 = a.x; w1 = a.y; w2 = a.z; w3 = a.w; w4 = b.x; break;
        case 1: w0 = a.y; w1 = a.z; w2 = a.w; w3 = b.x; w4 = b.y; break;
        case 2: w0 = a.z; w1 = a.w; w2 = b.x; w3 = b.y; w4 = b.z; break;
        default: w0 = a.w; w1 = b.x; w2 = b.y; w3 = b.z; w4 = b.w; break;
    }
    return make_uint4(__funnelshift_r(w0, w1, r), __funnelshift_r(w1, w2, r), __funnelshift_r(w2, w3, r), __funnelshift_r(w3, w4, r));
}

// One warp copies n bytes, any alignment of either side: bytes up to a 16-aligned dst one per lane, then 16-byte stores,
// each from two aligned 16-byte loads when src is not aligned with dst (both loaded words hold a source byte, so no
// load leaves the source's allocation), then the tail one byte per lane.
__device__ __forceinline__ void warp_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint64_t n, uint32_t lane)
{
    uint64_t head = (16 - ((uintptr_t)dst & 15)) & 15;
    if (head > n) head = n;
    if (lane < head) dst[lane] = src[lane];
    dst += head; src += head; n -= head;
    const uint64_t nv = n / 16;
    const uint32_t sh = (uint32_t)((uintptr_t)src & 15);
    uint4* d4 = (uint4*)dst;
    const uint4* s4 = (const uint4*)(src - sh);
    if (sh == 0) {
#pragma unroll 4
        for (uint64_t i = lane; i < nv; i += 32) d4[i] = s4[i];
    } else {
#pragma unroll 4
        for (uint64_t i = lane; i < nv; i += 32) d4[i] = byte_window(s4[i], s4[i + 1], sh);
    }
    for (uint64_t i = nv * 16 + lane; i < n; i += 32) dst[i] = src[i];
}

// The warps of a CTA share n bytes in 16-byte multiples, each copying its own contiguous part.
__device__ __forceinline__ void cta_copy(uint8_t* dst, const uint8_t* src, uint64_t n)
{
    constexpr uint32_t kWarps = kCopyThreads / 32;
    const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x & 31;
    const uint64_t share = a16((n + kWarps - 1) / kWarps);
    const uint64_t a = min(n, warp * share), b = min(n, a + share);
    if (a < b) warp_copy(dst + a, src + a, b - a, lane);
}

// LZ4: CTA (s, y) copies the 128 KiB pieces y, y + gridDim.y, ... of selected frame s's payload to its packed place;
// CTA (s, 0) also writes the frame's container header in front of it.
__global__ void __launch_bounds__(kCopyThreads)
rr_pack_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ frame_off, uint8_t* __restrict__ packed, RangeWork k)
{
    const uint32_t s = blockIdx.x;
    const uint64_t n = k.sel_csize[s];
    uint8_t* d = packed + k.sel_frame_off[s];
    const uint8_t* src = in + frame_off[k.sel_src[s]] + 12;
    if (blockIdx.y == 0 && threadIdx.x == 0) {
        uint32_t* h = (uint32_t*)d;                          // 4-aligned: f_pack + 4
        h[0] = ZMT_CONTAINER_MAGIC; h[1] = 4; h[2] = (uint32_t)n;
    }
    for (uint64_t a = (uint64_t)blockIdx.y * kPackPiece; a < n; a += (uint64_t)gridDim.y * kPackPiece)
        cta_copy(d + 12 + a, src + a, min(kPackPiece, n - a));
}

// zstd: the selected frames' own offsets (the decode runs in place in d_in), sizes, expected content and flags
__global__ void __launch_bounds__(kThreads)
rr_select_kernel(uint32_t nsel, const uint64_t* __restrict__ frame_off, const uint64_t* __restrict__ expect, const uint32_t* __restrict__ frame_seq, RangeWork k)
{
    const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
    if (s >= nsel) return;
    const uint32_t f = k.sel_src[s];
    k.sel_frame_off[s] = frame_off[f]; k.sel_expect[s] = expect[f]; k.sel_seq[s] = frame_seq[f];
}

__global__ void __launch_bounds__(kThreads)
rr_fail_kernel(uint32_t nsel, RangeWork k)
{
    const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
    if (s <= nsel) k.sel_fail[s] = s < nsel && k.sel_status[s] != ZMT_ST_OK ? 1u : 0u;
}

// A good range touches the selected frames a..b; its status is that of the first failed one among them: the first s
// with sel_fail[s + 1] > sel_fail[a] (sel_fail is the exclusive prefix of the failure flags).
__global__ void __launch_bounds__(kThreads)
rr_status_kernel(uint32_t nranges, uint32_t* __restrict__ range_status, RangeWork k)
{
    const uint32_t r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= nranges) return;
    uint32_t st = k.r_st[r];
    if (st == ZMT_ST_OK && k.r_len[r]) {
        const uint32_t a = k.selx[k.r_fa[r]], b = k.selx[k.r_fb[r]];
        const uint32_t f0 = k.sel_fail[a];
        if (k.sel_fail[b + 1] > f0) {
            uint32_t lo = a, hi = b;                         // the answer lies in [lo, hi]
            while (lo < hi) { const uint32_t m = lo + (hi - lo) / 2; if (k.sel_fail[m + 1] > f0) hi = m; else lo = m + 1; }
            st = k.sel_status[lo];
        }
        k.r_src[r] = k.sel_out_off[a] + k.r_skip[r];
    }
    range_status[r] = st;
}

// CTA p copies gather piece p: piece p - r_piece[r] of the range r whose pieces hold p
__global__ void __launch_bounds__(kCopyThreads)
rr_gather_kernel(uint32_t nranges, const uint8_t* __restrict__ scratch, uint8_t* __restrict__ dst, const uint64_t* __restrict__ dst_off,
                 const uint32_t* __restrict__ range_status, RangeWork k)
{
    const uint64_t p = blockIdx.x;
    uint32_t lo = 0, hi = nranges;                            // the last r with r_piece[r] <= p
    while (hi - lo > 1) { const uint32_t m = lo + (hi - lo) / 2; if (k.r_piece[m] <= p) lo = m; else hi = m; }
    const uint32_t r = lo;
    if (range_status[r] != ZMT_ST_OK) return;
    const uint64_t a = (p - k.r_piece[r]) * kPiece;
    cta_copy(dst + dst_off[r] + a, scratch + k.r_src[r] + a, min(kPiece, k.r_len[r] - a));
}

bool plan_ok(const zmt_range_plan* plan) { return plan && !too_many(plan->nframes, plan->nranges) && plan->nsel <= plan->nframes; }

// The steps after the decode, shared by both codecs: failure prefix, per-range status, gather.
bool finish_read(const zmt_range_plan* plan, const RangeWork& k, void* d_dst, const uint64_t* d_dst_off, uint32_t* d_range_status,
                 const void* d_scratch, cudaStream_t stream)
{
    ZmtProfScope ps(ZMT_K_FRAME_INDEX, stream);
    rr_fail_kernel<<<(plan->nsel + kThreads) / kThreads, kThreads, 0, stream>>>(plan->nsel, k);
    const bool ok = exclusive_sum(k, k.sel_fail, (uint64_t)plan->nsel + 1, stream);
    if (plan->nranges) rr_status_kernel<<<(plan->nranges + kThreads - 1) / kThreads, kThreads, 0, stream>>>(plan->nranges, d_range_status, k);
    if (plan->npieces) rr_gather_kernel<<<(uint32_t)plan->npieces, kCopyThreads, 0, stream>>>(plan->nranges, (const uint8_t*)d_scratch, (uint8_t*)d_dst,
                                                                                              d_dst_off, d_range_status, k);
    return ok;
}

}  // namespace

extern "C" size_t zmt_range_workspace_bytes(uint32_t nframes, uint32_t nranges)
{
    if (too_many(nframes, nranges)) return 0;
    RangeWork k;
    return carve(nullptr, nframes, nranges, &k);
}

extern "C" int zmt_lz4_content_offsets_device(const void* d_in, uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                                              uint64_t* d_content_off, zmt_frame_index* d_info, void* d_work, void* stream)
{
    return content_offsets<false>(d_in, nframes, d_frame_off, d_frame_csize, nullptr, d_content_off, d_info, d_work, (cudaStream_t)stream);
}

extern "C" int zmt_zstd_content_offsets_device(uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, const uint64_t* d_expect,
                                               uint64_t* d_content_off, zmt_frame_index* d_info, void* d_work, void* stream)
{
    return content_offsets<true>(nullptr, nframes, d_frame_off, d_frame_csize, d_expect, d_content_off, d_info, d_work, (cudaStream_t)stream);
}

extern "C" int zmt_lz4_range_plan_device(uint32_t nframes, const uint32_t* d_frame_csize, const uint64_t* d_content_off, const uint64_t* d_ranges,
                                         uint32_t nranges, uint64_t* d_dst_off, zmt_range_plan* d_plan, void* d_work, void* stream)
{
    return range_plan<false>(nframes, d_frame_csize, nullptr, nullptr, d_content_off, d_ranges, nranges, d_dst_off, d_plan, d_work, (cudaStream_t)stream);
}

extern "C" int zmt_zstd_range_plan_device(uint32_t nframes, const uint32_t* d_frame_csize, const uint32_t* d_frame_first_blk, const uint64_t* d_frame_scratch,
                                          const uint64_t* d_content_off, const uint64_t* d_ranges, uint32_t nranges, uint64_t* d_dst_off,
                                          zmt_range_plan* d_plan, void* d_work, void* stream)
{
    return range_plan<true>(nframes, d_frame_csize, d_frame_first_blk, d_frame_scratch, d_content_off, d_ranges, nranges, d_dst_off, d_plan, d_work,
                            (cudaStream_t)stream);
}

extern "C" size_t zmt_lz4_range_read_workspace_bytes(const zmt_range_plan* plan)
{
    if (!plan_ok(plan)) return 0;
    return (size_t)a256(plan->packed_bytes) + zmt_lz4d_workspace_bytes(plan->nsel, plan->nunits, plan->packed_bytes);
}

extern "C" size_t zmt_zstd_range_read_workspace_bytes(const zmt_range_plan* plan)
{
    if (!plan_ok(plan)) return 0;
    return (size_t)a256((uint64_t)plan->nunits * sizeof(ZBlk)) + zmt_zstdd_workspace_bytes(plan->nsel, plan->nunits, plan->dec_scratch);
}

extern "C" int zmt_lz4_range_read_device(const void* d_in, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, const zmt_range_plan* plan,
                                         void* d_dst, const uint64_t* d_dst_off, uint32_t* d_range_status, void* d_scratch, void* d_read_work,
                                         void* d_work, void* stream_)
{
    (void)d_frame_csize;                                      // the plan copied the selected frames' sizes
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!plan_ok(plan) || !d_work || (plan->nranges && (!d_dst_off || !d_range_status)) || (plan->npieces && !d_dst) ||
        (plan->nsel && (!d_in || !d_frame_off || !d_read_work || !d_scratch)))
        return ZMT_ST_BAD_ARG;
    RangeWork k;
    if (!carve(d_work, plan->nframes, plan->nranges, &k)) return ZMT_ST_CUDA;
    int rc = ZMT_ST_OK;
    if (plan->nsel) {
        uint8_t* packed = (uint8_t*)d_read_work;
        void* dec_work = packed + a256(plan->packed_bytes);
        // pieces of the average selected frame: frames cut from one input at one chunk size get a CTA per piece
        const uint64_t ys = (plan->packed_bytes / plan->nsel + kPackPiece - 1) / kPackPiece;
        { ZmtProfScope ps(ZMT_K_FRAME_INDEX, stream);
        rr_pack_kernel<<<dim3(plan->nsel, (uint32_t)(ys < 1 ? 1 : ys > 65535 ? 65535 : ys)), kCopyThreads, 0, stream>>>((const uint8_t*)d_in, d_frame_off, packed, k); }
        rc = zmt_lz4_decompress_device(packed, plan->packed_bytes, k.sel_frame_off, k.sel_csize, plan->nsel, plan->nunits, d_scratch,
                                       k.sel_out_off, k.sel_out_size, k.sel_status, dec_work, stream);
    }
    const bool ok = finish_read(plan, k, d_dst, d_dst_off, d_range_status, d_scratch, stream);
    if (rc != ZMT_ST_OK) return rc;
    return ok && cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}

extern "C" int zmt_zstd_range_read_device(const void* d_in, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, const uint64_t* d_expect,
                                          const uint32_t* d_frame_seq, const zmt_range_plan* plan, void* d_dst, const uint64_t* d_dst_off,
                                          uint32_t* d_range_status, void* d_scratch, void* d_read_work, void* d_work, void* stream_)
{
    (void)d_frame_csize;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!plan_ok(plan) || !d_work || (plan->nranges && (!d_dst_off || !d_range_status)) || (plan->npieces && !d_dst) ||
        (plan->nsel && (!d_in || !d_frame_off || !d_expect || !d_frame_seq || !d_read_work || !d_scratch)))
        return ZMT_ST_BAD_ARG;
    RangeWork k;
    if (!carve(d_work, plan->nframes, plan->nranges, &k)) return ZMT_ST_CUDA;
    int rc = ZMT_ST_OK;
    if (plan->nsel) {
        uint8_t* blocks = (uint8_t*)d_read_work;
        void* dec_work = blocks + a256((uint64_t)plan->nunits * sizeof(ZBlk));
        rr_select_kernel<<<(plan->nsel + kThreads - 1) / kThreads, kThreads, 0, stream>>>(plan->nsel, d_frame_off, d_expect, d_frame_seq, k);
        rc = zmt_zstd_blocks_device(d_in, plan->nsel, k.sel_frame_off, k.sel_csize, k.sel_first_blk, k.sel_scratch, blocks, plan->nunits, stream);
        if (rc == ZMT_ST_OK)
            rc = zmt_zstd_decompress_device(d_in, blocks, plan->nunits, k.sel_first_blk, k.sel_expect, k.sel_seq, plan->nsel, d_scratch,
                                            k.sel_out_off, k.sel_out_size, k.sel_status, dec_work, stream);
    }
    const bool ok = finish_read(plan, k, d_dst, d_dst_off, d_range_status, d_scratch, stream);
    if (rc != ZMT_ST_OK) return rc;
    return ok && cudaGetLastError() == cudaSuccess ? ZMT_ST_OK : ZMT_ST_CUDA;
}
