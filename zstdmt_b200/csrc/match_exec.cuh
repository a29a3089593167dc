// match_exec.cuh — what the two decoders' last passes share (DESIGN.md §3.2): lz4_exec_blocks_kernel (lz4_decode.cuh)
// and zx_block / zstd_execute_kernel (zstd_decode.cu) both give one warp a block by ticket and run its matches in steps.
// Here: the ticket order, the step constants, the dependency test and the copies.  Record formats, literals, validation
// and the waits on earlier blocks stay with the callers; nothing here knows which codec calls it.
#pragma once
#include "launch.h"

#define MX_STEP     32u           // match records per step: one per lane
#define MX_SPAN     2048u         // bytes of output a step may span: staged in shared memory
#define MX_OWN      32u           // an independent match up to this length is copied by its own lane, a longer one by the warp
#define MX_PERIOD   32u           // an overlapping match with a shorter period (offset) is copied modulo the offset
#define MX_INACTIVE 0x7FFFFFFF    // destination start / end of a lane without a match in the dependency search
#define MX_TICKET_WIN 16384u      // frames per ticket window

// ---------------------------------------------------------------- ticket order
// A unit is one block: unit first[f] + b is block b of frame f (first[]: nframes + 1 entries).  Blocks of one frame form a
// dependency chain wherever matches reach below their block (the first matches of a linked LZ4 block usually read the
// tail of the previous one), so tickets must not put the blocks of one frame on neighbouring warps: within a window of
// MX_TICKET_WIN frames the order is block-index-major — block 0 of every frame of the window, then block 1 of every
// frame, ... — which keeps as many independent chains in flight as there are frames in the window, and by the time block
// b+1 of a frame comes up its block b has long finished.  A warp may wait for earlier blocks of its frame only: unit
// (f, b-1) always holds a lower ticket than (f, b), and tickets are taken only by warps that are already running, so the
// wait cannot deadlock whatever order the hardware schedules CTAs in.
// A window whose frames have very different block counts would mostly hand out empty tickets; it falls back to
// frame-major order (flag in the top bit of its base).
#define MX_FRAME_MAJOR (1ull << 63)
// bytes of the window-base table wbase[] in a workspace (one entry per window and the total, rounded to 256)
static inline size_t ticket_table_bytes(uint32_t nframes) { return (size_t)a256(((uint64_t)nframes / MX_TICKET_WIN + 2) * 8); }

template <typename Idx>
__global__ void __launch_bounds__(256)
ticket_windows_kernel(const Idx* __restrict__ first, uint32_t nframes, unsigned long long* __restrict__ wbase)
{
    __shared__ uint32_t red[256];
    const uint32_t nwin = (nframes + MX_TICKET_WIN - 1) / MX_TICKET_WIN;
    unsigned long long base = 0;
    for (uint32_t w = 0; w < nwin; w++) {
        const uint32_t f0 = w * MX_TICKET_WIN, f1 = f0 + MX_TICKET_WIN < nframes ? f0 + MX_TICKET_WIN : nframes;
        uint32_t mx = 0;
        for (uint32_t f = f0 + threadIdx.x; f < f1; f += 256) { const uint32_t c = (uint32_t)(first[f + 1] - first[f]); mx = c > mx ? c : mx; }
        red[threadIdx.x] = mx;
        __syncthreads();
        for (uint32_t d = 128; d > 0; d >>= 1) { if (threadIdx.x < d && red[threadIdx.x + d] > red[threadIdx.x]) red[threadIdx.x] = red[threadIdx.x + d]; __syncthreads(); }
        mx = red[0];
        __syncthreads();
        const unsigned long long real = first[f1] - first[f0], grid = (unsigned long long)(f1 - f0) * mx;
        const bool frame_major = grid > 8 * real + 65536;
        if (threadIdx.x == 0) wbase[w] = base | (frame_major ? MX_FRAME_MAJOR : 0ull);
        base += frame_major ? real : grid;
    }
    if (threadIdx.x == 0) wbase[nwin] = base;
}

struct MxTickets { const unsigned long long* wbase; uint32_t nframes, nwin; unsigned long long count; };
__device__ __forceinline__ MxTickets mx_tickets(const unsigned long long* __restrict__ wbase, uint32_t nframes)
{
    MxTickets T; T.wbase = wbase; T.nframes = nframes;
    T.nwin = (nframes + MX_TICKET_WIN - 1) / MX_TICKET_WIN;
    T.count = wbase[T.nwin] & ~MX_FRAME_MAJOR;
    return T;
}

// the warp's next ticket (all tickets are handed out once it reaches T.count)
__device__ __forceinline__ unsigned long long mx_take_ticket(unsigned long long* ticket, uint32_t lane)
{
    unsigned long long tk = 0;
    if (lane == 0) tk = atomicAdd(ticket, 1ull);
    return __shfl_sync(ZMT_FULL_MASK, tk, 0);
}

// ticket -> window (binary search over the window bases) -> (frame, block) -> unit; false: an empty ticket (the frame
// has fewer blocks than the widest of its window)
template <typename Idx>
__device__ __forceinline__ bool mx_ticket_unit(const MxTickets& T, unsigned long long tk, const Idx* __restrict__ first, Idx& unit)
{
    uint32_t lo = 0, hi = T.nwin;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if ((T.wbase[mid] & ~MX_FRAME_MAJOR) <= tk) lo = mid; else hi = mid; }
    const unsigned long long wb = T.wbase[lo];
    const unsigned long long tl = tk - (wb & ~MX_FRAME_MAJOR);
    const uint32_t f0 = lo * MX_TICKET_WIN, wn = (f0 + MX_TICKET_WIN < T.nframes ? MX_TICKET_WIN : T.nframes - f0);
    if (wb >> 63) { unit = first[f0] + (Idx)tl; return true; }          // frame-major window
    const uint32_t fb = (uint32_t)(tl / wn), ff = f0 + (uint32_t)(tl % wn);
    const Idx s0 = first[ff];
    unit = s0 + fb;
    return fb < first[ff + 1] - s0;                                     // false: this frame has fewer blocks
}

// ---------------------------------------------------------------- dependency test
// Which matches of a step must wait for an earlier match of this very step?  Lane k holds match k: destination
// [dst, dst + ml), source dst - off (block-relative, may be negative); act = the lane holds a match.  Only the
// destinations of matches j < k matter, and they are sorted and disjoint: a = first j whose destination ends above my
// source start (binary search over the lanes by shuffle); my source touches a destination of the step iff that j lies
// before me and starts below my source end.  A match that overlaps its own destination (off < ml) is not independent
// either.  Exact: it gives the pairwise overlap's answer.
__device__ __forceinline__ bool mx_independent(uint32_t lane, bool act, uint32_t dst, uint32_t ml, uint32_t off)
{
    const int32_t sp = (int32_t)dst - (int32_t)off;
    const int32_t e_end = act ? (int32_t)(dst + ml) : MX_INACTIVE, d_beg = act ? (int32_t)dst : MX_INACTIVE;
    uint32_t a = 0;
#pragma unroll
    for (uint32_t stp = 16; stp > 0; stp >>= 1) {
        const int32_t v = __shfl_sync(ZMT_FULL_MASK, e_end, (a + stp - 1) & 31);
        if (v <= sp) a += stp;                                  // e_j <= sp: destination j lies entirely below my source
    }
    const int32_t da = __shfl_sync(ZMT_FULL_MASK, d_beg, a & 31);
    return act && off >= ml && !(a < lane && da < sp + (int32_t)ml);
}

// ---------------------------------------------------------------- the step window and the copies
// Every byte a step regenerates is written to global memory AND to the window; a source byte at or above the step's
// first output byte is read from the window.  A chain of matches that feed each other then runs at shared-memory
// latency instead of one L2 round trip per link.
// A prefix region below the frame: content that precedes the frame's output without being part of it (a dictionary's
// content).  The copies below take it when instantiated with PRE = true: a source byte at block position q below the
// frame's first byte fs reads pre_end[q - fs], the region's tail, and a copy that straddles fs is split there.  The
// caller bounds every source by the frame's output so far plus the region.  PRE = false never reads pre_end / fs.
struct MxWin {
    uint8_t* dst;             // the block's output in global memory
    uint8_t* S;               // S[wb + p] = window byte of block position p, lo <= p < lo + MX_SPAN
    int32_t wb, lo;           // lo = block position of the step's first output byte
    const uint8_t* pre_end;   // PRE: one past the prefix region's last byte
    int32_t fs;               // PRE: block position of the frame's first byte (<= 0)
};

template <bool PRE = false>
__device__ __forceinline__ uint8_t mx_src_byte(const MxWin& W, int32_t q)
{
    return q >= W.lo ? W.S[W.wb + q] : (PRE && q < W.fs) ? W.pre_end[q - W.fs] : W.dst[q];
}
// One lane: bytes [k0, n) of src to d (global memory) and dw (window), loads first, stores after, 8 bytes at a time — a
// byte-wise load -> store loop pays one L2 latency per byte, this one per 8 bytes.
__device__ __forceinline__ void mx_lane_copy(uint8_t* d, uint8_t* dw, const uint8_t* src, uint32_t k0, uint32_t n)
{
    for (uint32_t k = k0; k < n; k += 8) {
        uint8_t x[8];
#pragma unroll
        for (int j = 0; j < 8; j++) x[j] = (k + j < n) ? src[k + j] : (uint8_t)0;
#pragma unroll
        for (int j = 0; j < 8; j++) if (k + j < n) { d[k + j] = x[j]; dw[k + j] = x[j]; }
    }
}

// bytes of the source [sp, sp + ml) that lie below the window (with PRE: the prefix region's among them too)
__device__ __forceinline__ int32_t mx_nlow(const MxWin& W, int32_t sp, uint32_t ml)
{
    return sp >= W.lo ? 0 : (W.lo - sp < (int32_t)ml ? W.lo - sp : (int32_t)ml);
}

// One lane copies its own independent match of at most MX_OWN bytes: the nlow source bytes below the window come from
// global memory (those below k0 the caller has copied already), the rest out of the window.
template <bool PRE = false>
__device__ __forceinline__ void mx_own_match(const MxWin& W, uint32_t dst, uint32_t ml, uint32_t off, int32_t nlow, int32_t k0)
{
    const int32_t sp = (int32_t)dst - (int32_t)off;
    uint8_t* d = W.dst + dst; uint8_t* dw = W.S + (W.wb + (int32_t)dst);
    if (PRE && sp < W.fs) {                                     // the first np source bytes lie in the prefix region
        const int32_t np = W.fs - sp < nlow ? W.fs - sp : nlow;
        mx_lane_copy(d, dw, W.pre_end + (sp - W.fs), (uint32_t)k0, (uint32_t)np);
        mx_lane_copy(d, dw, W.dst + sp, (uint32_t)(k0 > np ? k0 : np), (uint32_t)nlow);
    } else
        mx_lane_copy(d, dw, W.dst + sp, (uint32_t)k0, (uint32_t)nlow);
    for (int32_t k = nlow; k < (int32_t)ml; k++) { const uint8_t x = W.S[W.wb + sp + k]; d[k] = x; dw[k] = x; }
}

// The whole warp copies one match through the window; called for the matches of a step in order, so the source may be a
// match of this very step, or the match itself (off < ml).
template <bool PRE = false>
__device__ __forceinline__ void mx_warp_match(const MxWin& W, uint32_t dst, uint32_t ml, uint32_t off, uint32_t lane)
{
    const int32_t qs = (int32_t)dst - (int32_t)off;
    uint8_t* d = W.dst + dst; uint8_t* dw = W.S + (W.wb + (int32_t)dst);
    if (off >= ml) {
        for (uint32_t k = lane; k < ml; k += 32) { const uint8_t x = mx_src_byte<PRE>(W, qs + (int32_t)k); d[k] = x; dw[k] = x; }
    } else if (off >= MX_PERIOD) {                              // overlapping, period >= warp width: 32-byte waves
        for (uint32_t k = 0; k < ml; k += 32) {
            if (k + lane < ml) { const uint8_t x = mx_src_byte<PRE>(W, qs + (int32_t)(k + lane)); d[k + lane] = x; dw[k + lane] = x; }
            __syncwarp();
        }
    } else {                                                    // short period: replicate the pattern
        for (uint32_t k = lane; k < ml; k += 32) { const uint8_t x = mx_src_byte<PRE>(W, qs + (int32_t)(k % off)); d[k] = x; dw[k] = x; }
    }
    __syncwarp();
}

// The whole warp copies one match straight in global memory (no window): a lone match longer than MX_SPAN, and every
// match of the LZ4 sequential fallback.  The caller has made the source visible to all lanes.
__device__ __forceinline__ void mx_warp_match_global(uint8_t* d, uint32_t ml, uint32_t off, uint32_t lane)
{
    const uint8_t* m = d - off;
    if (off >= ml) { for (uint32_t k = lane; k < ml; k += 32) d[k] = m[k]; }
    else if (off >= MX_PERIOD) { for (uint32_t k = 0; k < ml; k += 32) { if (k + lane < ml) d[k + lane] = m[k + lane]; __syncwarp(); } }
    else { for (uint32_t k = lane; k < ml; k += 32) d[k] = m[k % off]; }
    __syncwarp();
}

// mx_warp_match_global with a prefix region: `below` = the frame's output below d; a source that starts further back takes
// its first off - below bytes from the region's tail [pre_end - (off - below), pre_end).
__device__ __forceinline__ void mx_warp_match_global_pre(uint8_t* d, uint32_t ml, uint32_t off, uint32_t lane, const uint8_t* pre_end, uint64_t below)
{
    if (off <= below) { mx_warp_match_global(d, ml, off, lane); return; }
    const uint8_t* m = d - off;
    const uint32_t np = (uint32_t)(off - below);
    const uint8_t* pm = pre_end - np;
    auto at = [&](uint32_t i) -> uint8_t { return i < np ? pm[i] : m[i]; };
    if (off >= ml) { for (uint32_t k = lane; k < ml; k += 32) d[k] = at(k); }
    else if (off >= MX_PERIOD) { for (uint32_t k = 0; k < ml; k += 32) { if (k + lane < ml) d[k + lane] = at(k + lane); __syncwarp(); } }
    else { for (uint32_t k = lane; k < ml; k += 32) d[k] = at(k % off); }
    __syncwarp();
}
