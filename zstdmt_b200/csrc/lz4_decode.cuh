// lz4_decode.cuh — LZ4F frame decoder (included by lz4_kernels.cu).
//
// Replaces the arithmetic of LZ4F_decompress as the reference calls it per frame
// (lib/lz4-mt_decompress.c:349-351), for whole batches of frames at once.
//
// Work unit = one warp per LZ4F block (64 KiB .. 4 MiB of output), two passes over every block:
//
//   lz4_scan_frames_kernel   one thread per frame: header + header checksum, walks the block headers and
//                            fills the block table (one LzBlk per "slot"; frame f owns the slots
//                            first_slot[f] .. first_slot[f+1], one per blockMaxSize of output room).
//   lz4_parse_blocks_kernel  pass A, history-free, fully parallel over blocks: the token stream of a block is
//                            parsed 32 sequences at a time — every lane classifies 8 byte positions of a
//                            256-byte stretch as "if a token starts here, the next one starts at +d" (one byte
//                            of shared memory per position), the warp then follows the chain from the known
//                            start (one dependent LDS per sequence) and lane k keeps the k-th sequence.  Output
//                            positions come from a warp scan; every lane copies its own literal run to its final
//                            place and appends a match record {dst, length, offset} to the block's record list.
//   lz4_exec_blocks_kernel   pass B, persistent grid, blocks handed out by a ticket counter in frame order:
//                            32 match records per step; matches whose source lies entirely below the step's
//                            first destination are copied lane-parallel, the others (overlapping or reading a
//                            match of the same step) in order by the whole warp.  A match that reaches into the
//                            previous block of a linked-block frame (what liblz4 emits for the reference,
//                            lz4-mt_compress.c:141-146) waits on that block's published progress counter; the
//                            previous block always holds a lower ticket, so the wait cannot deadlock.
//   lz4_decode_frames_seq_kernel   fallback, one warp per flagged frame, blocks in order: frames whose non-last
//                            blocks do not regenerate exactly blockMaxSize bytes (LZ4F_compressUpdate + flush
//                            streams), where the output position of a block is not known before decoding.
#pragma once

#define LZD_WARPS 8
#define LZD_WIN   512u        // compressed bytes staged per step and warp (one 16-byte load per lane)
#define LZD_NJ    256u        // token-start candidates examined per step
#define LZD_LONG  32u         // matches longer than this are copied by the whole warp
#define LZD_LONGLIT 16u       // literal runs longer than this are copied by the whole warp (pass A: few lanes hold long runs)
#define LZD_ERR   0xFFFFFFFFu
#define LZD_DONE  0xFFFFFFFFu // progress value of a finished block

#define LZB_LINKED 1u         // block may copy from the previous block of its frame
#define LZB_LAST   2u         // last block of its frame
#define LZB_BCHK   4u         // an XXH32 of the block's stored bytes follows them (FLG.BC)

struct LzBlk {
    uint32_t src;             // offset of the block data inside the LZ4F frame
    uint32_t csize;           // compressed size, bit 31 = stored; 0 = empty slot
    uint32_t flags;           // LZB_* | log2(blockMaxSize) << 8
    uint32_t nrec;            // match records written by pass A
    uint32_t frame;
};

// first error wins; bit 8 (ZMT_ST_HAS_CHK, set by the scan) is preserved
__device__ __forceinline__ void d_fail(uint32_t* status, uint32_t f, uint32_t code, uint32_t lane)
{
    if (lane == 0) {
        uint32_t old = status[f];
        while ((old & 0xFF) == 0) { const uint32_t was = atomicCAS(&status[f], old, old | code); if (was == old) break; old = was; }
    }
}

// whole-warp copy; long runs go through the 16-byte-store copier of common.cuh (re-aligns the source with funnel shifts;
// may read up to 4 bytes past src + n: every source here is followed by at least an end mark or lies inside the output)
__device__ __forceinline__ void warp_copy_lit(uint8_t* dst, const uint8_t* src, uint32_t n, uint32_t lane)
{
    if (n >= 64) coop_copy_g2g(dst, src, n, lane, 32);
    else for (uint32_t i = lane; i < n; i += 32) dst[i] = src[i];
}

// ---------------------------------------------------------------- frame scan
// slots per frame = max(1, ceil(room / 64 KiB)) (64 KiB is the smallest blockMaxSize): an upper bound of its block count
__global__ void lz4_slot_counts_kernel(const uint64_t* __restrict__ out_off, uint32_t nframes, uint64_t* __restrict__ cnt)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint64_t room = out_off[f + 1] - out_off[f];
    const uint64_t n = (room + 65535) >> 16;
    cnt[f] = n ? n : 1;
}

__global__ void lz4_scan_frames_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ frame_off, const uint32_t* __restrict__ frame_csize,
                                       const uint64_t* __restrict__ out_off, const uint64_t* __restrict__ first_slot, uint32_t slot_cap,
                                       LzBlk* __restrict__ tab, uint32_t* __restrict__ prog, uint32_t* __restrict__ status,
                                       uint32_t* __restrict__ stored_chk, uint32_t* __restrict__ needs_seq, uint32_t* __restrict__ any_bchk,
                                       uint32_t nframes)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const uint64_t s0 = first_slot[f], s1 = first_slot[f + 1];
    if (s1 > slot_cap) { status[f] = ZMT_ST_BAD_ARG; return; }                 // table too small for this batch (caller's slot count is wrong)
    const uint32_t nslot = (uint32_t)(s1 - s0);
    LzBlk* T = tab + s0;
    for (uint32_t s = 0; s < nslot; s++) { LzBlk e; e.src = 0; e.csize = 0; e.flags = 0; e.nrec = 0; e.frame = f; T[s] = e; prog[s0 + s] = 0; }
    const uint8_t* p = in + frame_off[f] + 12;              // LZ4F frame (after the skippable header)
    const uint32_t fs = frame_csize[f];
    const uint64_t cap = out_off[f + 1] - out_off[f];
    uint32_t err = 0;
    if (fs < 7 + 4) err = ZMT_ST_TRUNCATED;
    else if (ldg_le32(p) != 0x184D2204u) err = ZMT_ST_BAD_MAGIC;
    if (err) { status[f] = err; return; }
    const uint32_t flg = p[4], bd = p[5];
    if ((flg >> 6) != 1 || (flg & 2) || (bd & 0x8F) || ((bd >> 4) & 7) < 4) { status[f] = ZMT_ST_BAD_HEADER; return; }
    const uint32_t indep = (flg >> 5) & 1, bchk = (flg >> 4) & 1, csz = (flg >> 3) & 1, cchk = (flg >> 2) & 1, did = flg & 1;
    const uint32_t blklog = 8 + 2 * ((bd >> 4) & 7), blkmax = 1u << blklog;
    const uint32_t hl = 2 + (csz ? 8 : 0) + (did ? 4 : 0);
    if (fs < 4 + hl + 1 + 4) { status[f] = ZMT_ST_TRUNCATED; return; }
    {
        uint8_t h[14];
        for (uint32_t i = 0; i < hl; i++) h[i] = p[4 + i];
        if (((xxh32_small(h, hl, 0) >> 8) & 0xFF) != p[4 + hl]) { status[f] = ZMT_ST_HDR_CHECKSUM; return; }
    }
    uint32_t ip = 4 + hl + 1, b = 0;
    bool seq = false;
    for (;;) {
        if (fs - ip < 4) { err = ZMT_ST_TRUNCATED; break; }
        const uint32_t bh = ldg_le32(p + ip);
        if (bh == 0) break;
        ip += 4;
        const uint32_t bs = bh & 0x7FFFFFFFu;
        if (bs > blkmax) { err = ZMT_ST_BLOCK; break; }
        if (fs - ip < bs + (bchk ? 4 : 0) || fs - ip - bs - (bchk ? 4 : 0) < 4) { err = ZMT_ST_TRUNCATED; break; }
        // a block beyond the slots, or one that would start past the room: partial blocks or an overlong frame —
        // the sequential pass decodes it block after block and reports what is wrong, if anything
        if (b >= nslot || (uint64_t)b * blkmax > cap) { seq = true; }
        else {
            LzBlk e; e.src = ip; e.csize = bh; e.flags = ((!indep && b > 0) ? LZB_LINKED : 0u) | (bchk ? LZB_BCHK : 0u) | (blklog << 8); e.nrec = 0; e.frame = f;
            if (bs == 0) e.csize = 0;                      // a zero-sized stored block regenerates nothing (bit 31 set, size 0)
            if (bs == 0) seq = true;                       // ... and breaks the fixed block addressing
            T[b] = e;
        }
        ip += bs + (bchk ? 4 : 0); b++;
    }
    if (!err) {
        ip += 4;
        uint32_t has_chk = 0, chkv = 0;
        if (cchk) {
            if (fs - ip < 4) err = ZMT_ST_TRUNCATED;
            else { has_chk = 1; chkv = ldg_le32(p + ip); ip += 4; }
        }
        if (!err && ip != fs) err = ZMT_ST_TRAILING;
        if (!err) { stored_chk[f] = chkv; if (has_chk) status[f] = ZMT_ST_HAS_CHK; }
    }
    if (err) { status[f] = err; for (uint32_t s = 0; s < nslot; s++) T[s].csize = 0; return; }
    if (seq) { needs_seq[f] = 1; for (uint32_t s = 0; s < nslot; s++) T[s].csize = 0; return; }
    if (b > 0) T[b - 1].flags |= LZB_LAST;
    if (bchk) *any_bchk = 1;
}

// ---------------------------------------------------------------- block checksums (FLG.BC), before pass A
// One warp per slot of the two-pass path: XXH32 of the block's stored bytes against the 4 bytes that follow them; a
// mismatch fails the frame with ZMT_ST_BLOCK, so pass A skips it.  Frames of the sequential pass are checked there,
// block by block.  Exits at once when no frame of the batch sets FLG.BC (every frame this library writes).
__global__ void __launch_bounds__(32 * X_WARPS)
lz4_block_checksum_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ frame_off, const uint64_t* __restrict__ first_slot,
                          const LzBlk* __restrict__ tab, uint32_t* __restrict__ status, const uint32_t* __restrict__ any_bchk,
                          uint32_t nframes, uint32_t slot_cap)
{
    __shared__ uint4 tile[X_WARPS][2][32];
    if (*any_bchk == 0) return;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t nslots = first_slot[nframes] < slot_cap ? first_slot[nframes] : slot_cap;
    for (uint64_t t = (uint64_t)blockIdx.x * X_WARPS + wid; t < nslots; t += (uint64_t)gridDim.x * X_WARPS) {
        const LzBlk B = tab[t];
        if (B.csize == 0 || !(B.flags & LZB_BCHK) || (status[B.frame] & 0xFF) != 0) continue;
        const uint8_t* src = in + frame_off[B.frame] + 12 + B.src;
        const uint32_t bs = B.csize & 0x7FFFFFFFu;
        const uint32_t h = warp_xxh32(src, bs, tile[wid], lane);
        if (lane == 0 && h != ldg_le32(src + bs)) d_fail(status, B.frame, ZMT_ST_BLOCK, lane);
    }
}

// ---------------------------------------------------------------- pass A: token parse, literals, match records
struct LzSeq { uint32_t lit, litpos, off, ml, next; uint32_t st; };     // st: 0 ok, 1 last sequence (no match), 2 error

struct LzWin { const uint8_t* w; int32_t pos; const uint8_t* g; };     // window bytes [pos, pos + LZD_WIN) of the block live in w[]
__device__ __forceinline__ uint32_t lzw_byte(const LzWin& W, uint32_t q)
{
    const uint32_t r = q - (uint32_t)W.pos;                 // q >= pos always (positions only move forward from the window base)
    return r < LZD_WIN ? W.w[r] : W.g[q];
}

// Sequence parser for the common extended tokens, all reads out of the staged window without per-byte range tests: taken
// when the whole sequence header (token, up to 2 + 2 extension bytes, offset) provably lies inside the window and in front
// of the block end; anything else goes through lzd_parse_seq.  Returns false if it does not apply.
__device__ __forceinline__ bool lzd_parse_seq_win(const LzWin& W, uint32_t srcSize, uint32_t p, LzSeq& s)
{
    const uint32_t r = p - (uint32_t)W.pos;
    if (r + 24 > LZD_WIN || p + 24 > srcSize) return false;            // room for token + 2 ext + (lit handled below) + offset + 2 ext
    const uint8_t* w = W.w + r;
    const uint32_t tok = w[0];
    uint32_t lit = tok >> 4, q = 1;
    if (lit == 15) { const uint32_t b = w[1]; lit += b; q = 2; if (b == 255) { const uint32_t c = w[2]; if (c == 255) return false; lit += c; q = 3; } }
    if (r + q + lit + 6 > LZD_WIN || p + q + lit + 6 > srcSize) return false;
    s.lit = lit; s.litpos = p + q;
    const uint8_t* o = w + q + lit;
    s.off = o[0] | ((uint32_t)o[1] << 8);
    uint32_t ml = tok & 15, e = 2;
    if (ml == 15) { const uint32_t b = o[2]; ml += b; e = 3; if (b == 255) { const uint32_t c = o[3]; if (c == 255) return false; ml += c; e = 4; } }
    s.ml = ml + 4; s.next = p + q + lit + e; s.st = 0;
    return true;
}

// general sequence parser (any literal / match length, end of block); every read is bounds-checked against srcSize
__device__ __forceinline__ LzSeq lzd_parse_seq(const LzWin& W, uint32_t srcSize, uint32_t p)
{
    LzSeq s; s.lit = s.litpos = s.off = s.ml = 0; s.next = p; s.st = 2;
    if (p >= srcSize) return s;
    const uint32_t tok = lzw_byte(W, p);
    uint32_t lit = tok >> 4, q = p + 1;
    if (lit == 15) {
        uint32_t b;
        do { if (q >= srcSize) return s; b = lzw_byte(W, q++); lit += b; } while (b == 255);
    }
    if (lit > srcSize - q) return s;
    s.lit = lit; s.litpos = q;
    q += lit;
    if (q == srcSize) { s.next = q; s.st = 1; return s; }
    if (srcSize - q < 2) return s;
    s.off = lzw_byte(W, q) | (lzw_byte(W, q + 1) << 8);
    q += 2;
    uint32_t ml = tok & 15;
    if (ml == 15) {
        uint32_t b;
        do { if (q >= srcSize) return s; b = lzw_byte(W, q++); ml += b; } while (b == 255);
    }
    s.ml = ml + 4; s.next = q; s.st = 0;
    return s;
}

// Returns the decoded size or LZD_ERR.  `hist` = bytes of valid history below dst (linked blocks).  rec[] receives
// one record per match: dst (24) | length (24) << 24 | offset (16) << 48.
__device__ uint32_t lzd_parse_block(uint8_t* win, uint8_t* J, const uint8_t* gsrc, const uint8_t* in_end, uint32_t srcSize,
                                    uint8_t* dst, uint32_t dcap, uint32_t hist, unsigned long long* rec, uint32_t* nrec_out, uint32_t lane)
{
    uint32_t ip0 = 0, op = 0, nrec = 0;
    *nrec_out = 0;
    if (srcSize == 0) return LZD_ERR;
    LzWin W; W.w = win; W.g = gsrc;
    for (;;) {
        // ---- stage the window (aligned 16-byte loads; bytes past the end of the input read as zero)
        const uint32_t sh = (uint32_t)((uintptr_t)(gsrc + ip0) & 15);
        W.pos = (int32_t)ip0 - (int32_t)sh;
        __syncwarp();
        {
            const uint8_t* a = gsrc + W.pos + (int32_t)(16 * lane);
            uint4 v = make_uint4(0, 0, 0, 0);
            if (a + 16 <= in_end) v = *reinterpret_cast<const uint4*>(a);
            else { uint8_t* b = reinterpret_cast<uint8_t*>(&v); for (int i = 0; i < 16; i++) if (a + i < in_end) b[i] = a[i]; }
            reinterpret_cast<uint4*>(win)[lane] = v;
        }
        __syncwarp();
        // ---- J[pr] = distance to the next token if a short-literal token starts at ip0 + pr (literal length < 15; match
        //      length plain or extended by ONE byte < 255 — matches of 19..273 bytes are the bulk of the extended tokens on
        //      structured data), and the next token lies in front of the block end; else 0 (the chain follow parses it)
        {
            const uint32_t base = sh + 8 * lane;
            const uint32_t w0 = lds32u(win, base), w1 = lds32u(win, base + 4);
            // the "next token in front of the block end" test only matters in the last stretch of a block
            const bool near_end = ip0 + LZD_NJ + 24 >= srcSize;
            uint32_t j0 = 0, j1 = 0;
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const uint32_t tok = ((j < 4 ? w0 : w1) >> (8 * (j & 3))) & 0xFF;
                const uint32_t lit = tok >> 4;
                const uint32_t m15 = (tok & 15) == 15 ? 1u : 0u;
                const uint32_t ext = win[base + j + 3 + lit];                          // the byte a one-byte match-length extension would be (index < 290)
                const uint32_t d = 3 + lit + m15;
                bool fast = lit != 15 && !(m15 && ext == 255);
                if (near_end) fast = fast && ip0 + 8 * lane + j + d < srcSize;
                const uint32_t v = fast ? d : 0;
                if (j < 4) j0 |= v << (8 * j); else j1 |= v << (8 * (j - 4));
            }
            reinterpret_cast<uint2*>(J)[lane] = make_uint2(j0, j1);
        }
        __syncwarp();
        // ---- follow the chain: lane k keeps the start of the k-th sequence (relative to ip0).  Tokens with length
        //      extensions (J = 0) are parsed right here by all lanes and handed to lane k, so nothing is parsed twice
        uint32_t pr = 0, k = 0, myrel = 0;
        uint32_t fin = 0;                                   // 1: block ends with sequence k-1, 2: malformed
        LzSeq s; s.lit = s.litpos = s.off = s.ml = 0; s.next = 0; s.st = 3;      // st 3: plain token, decoded below
#pragma unroll 4
        for (; k < 32; k++) {
            if (pr >= LZD_NJ) break;
            myrel = lane == k ? pr : myrel;
            uint32_t d = J[pr];
            if (d == 0) {
                LzSeq q;
                if (!lzd_parse_seq_win(W, srcSize, ip0 + pr, q)) q = lzd_parse_seq(W, srcSize, ip0 + pr);
                if (lane == k) s = q;
                if (q.st) { fin = q.st; k++; break; }
                d = q.next - (ip0 + pr);
            }
            pr += d;
        }
        if (fin == 2) return LZD_ERR;
        const uint32_t cnt = k;
        // ---- plain tokens: literal length, match length and offset straight out of the window (the J rule keeps the
        //      whole sequence inside it and in front of the block end)
        if (lane < cnt && s.st == 3) {
            const uint32_t r = myrel + sh;                                  // window index of the token
            const uint32_t tok = win[r];
            s.lit = tok >> 4; s.litpos = ip0 + myrel + 1;
            const uint32_t o = r + 1 + s.lit;
            s.off = win[o] | ((uint32_t)win[o + 1] << 8);
            s.ml = (tok & 15) + 4; s.st = 0;
            if ((tok & 15) == 15) s.ml += win[o + 2];                        // the one extension byte the J rule admitted
        }
        if (lane >= cnt) { s.lit = 0; s.ml = 0; s.st = 0; }
        bool bad = lane < cnt && (s.st == 2 || s.lit > dcap || s.ml > dcap);
        if (bad) { s.lit = 0; s.ml = 0; }
        const uint32_t tot = s.lit + s.ml;
        uint32_t inc = tot;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc += y; }
        const uint32_t my_op = op + inc - tot, my_mp = my_op + s.lit;
        bad = bad || (lane < cnt && ((uint64_t)my_op + tot > dcap || (s.ml && (s.off == 0 || (uint64_t)s.off > (uint64_t)my_mp + hist))));
        if (__any_sync(ZMT_FULL_MASK, bad)) return LZD_ERR;
        // ---- literals: own run per lane, long runs by the whole warp
        if (s.lit && s.lit <= LZD_LONGLIT) {
            uint8_t* d = dst + my_op;
            const uint32_t r = s.litpos - (uint32_t)W.pos;
            const uint8_t* sp = (r + s.lit <= LZD_WIN) ? win + r : gsrc + s.litpos;      // generic pointer: shared or global
            uint32_t i = 0;
            for (; i + 4 <= s.lit; i += 4) { const uint8_t a = sp[i], b = sp[i + 1], c = sp[i + 2], e = sp[i + 3]; d[i] = a; d[i + 1] = b; d[i + 2] = c; d[i + 3] = e; }
            for (; i < s.lit; i++) d[i] = sp[i];
        }
        uint32_t longmask = __ballot_sync(ZMT_FULL_MASK, s.lit > LZD_LONGLIT);
        while (longmask) {
            const int jl = __ffs(longmask) - 1; longmask &= longmask - 1;
            const uint32_t o = __shfl_sync(ZMT_FULL_MASK, my_op, jl), lp = __shfl_sync(ZMT_FULL_MASK, s.litpos, jl), n = __shfl_sync(ZMT_FULL_MASK, s.lit, jl);
            warp_copy_lit(dst + o, gsrc + lp, n, lane);
        }
        // ---- match records
        const uint32_t mmask = __ballot_sync(ZMT_FULL_MASK, s.ml != 0);
        if (s.ml) rec[nrec + __popc(mmask & ((1u << lane) - 1))] = (unsigned long long)my_mp | ((unsigned long long)s.ml << 24) | ((unsigned long long)s.off << 48);
        nrec += __popc(mmask);
        op += __shfl_sync(ZMT_FULL_MASK, inc, 31);
        if (fin == 1) break;
        ip0 += pr;
    }
    *nrec_out = nrec;
    return op;
}

__global__ void __launch_bounds__(32 * LZD_WARPS)
lz4_parse_blocks_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ in_end, const uint64_t* __restrict__ frame_off,
                        uint8_t* __restrict__ out, const uint64_t* __restrict__ out_off, const uint64_t* __restrict__ first_slot,
                        LzBlk* __restrict__ tab, unsigned long long* __restrict__ rec, unsigned long long* __restrict__ out_size,
                        uint32_t* __restrict__ status, uint32_t* __restrict__ needs_seq, uint32_t nframes, uint32_t slot_cap)
{
    __shared__ __align__(16) uint8_t win[LZD_WARPS][LZD_WIN];
    __shared__ __align__(16) uint8_t jt[LZD_WARPS][LZD_NJ];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t t = (uint64_t)blockIdx.x * LZD_WARPS + wid;
    const uint64_t nslots = first_slot[nframes];
    if (t >= nslots || t >= slot_cap) return;
    const LzBlk B = tab[t];
    if (B.csize == 0) return;
    const uint32_t f = B.frame;
    if ((status[f] & 0xFF) != 0) return;
    const uint32_t slot = (uint32_t)(t - first_slot[f]);
    const uint32_t blklog = (B.flags >> 8) & 0xFF, blkmax = 1u << blklog;
    const uint64_t cap = out_off[f + 1] - out_off[f], boff = (uint64_t)slot << blklog;
    uint8_t* dst = out + out_off[f] + boff;
    const uint64_t room = cap - boff;                       // the scan guarantees boff <= cap
    const uint32_t bs = B.csize & 0x7FFFFFFFu;
    const uint64_t abs_src = frame_off[f] + 12 + B.src;
    const uint8_t* src = in + abs_src;
    uint32_t d, nrec = 0;
    if (B.csize & 0x80000000u) {
        if (bs > room) { d_fail(status, f, ZMT_ST_DST_SMALL, lane); return; }
        warp_copy_lit(dst, src, bs, lane);
        d = bs;
    } else {
        const uint32_t dcap = room < blkmax ? (uint32_t)room : blkmax;
        const uint32_t hist = (B.flags & LZB_LINKED) ? (boff < 65536 ? (uint32_t)boff : 65536u) : 0u;
        d = lzd_parse_block(win[wid], jt[wid], src, in_end, bs, dst, dcap, hist, rec + (abs_src + 2) / 3, &nrec, lane);
        if (d == LZD_ERR) { d_fail(status, f, ZMT_ST_BLOCK, lane); return; }
    }
    if (lane == 0) {
        atomicAdd(&out_size[f], (unsigned long long)d);
        tab[t].nrec = nrec;
        // fixed block addressing needs every block but the last to regenerate exactly blockMaxSize bytes
        if (!(B.flags & LZB_LAST) && d != blkmax) needs_seq[f] = 1;
    }
}

// ---------------------------------------------------------------- pass B: match execution
// Ticket order.  Blocks of a linked-block frame form a dependency chain (the first matches of a block usually read the
// tail of the previous one), so tickets must not put the blocks of one frame on neighbouring warps: within a window of
// LZX_WIN frames the order is block-index-major — block 0 of every frame of the window, then block 1 of every frame, ... —
// which keeps as many independent chains in flight as there are frames in the window, and by the time block b+1 of a
// frame comes up its block b has long finished.  (f, b-1) still always holds a lower ticket than (f, b): no deadlock.
// A window whose frames have very different block counts would mostly hand out empty tickets; it falls back to
// frame-major order (flag in the top bit of its base).
#define LZX_WIN 16384u
#define LZX_SPAN 2048u        // bytes of output a step may span: staged in shared memory
__global__ void __launch_bounds__(256)
lz4_ticket_windows_kernel(const uint64_t* __restrict__ first_slot, uint32_t nframes, unsigned long long* __restrict__ wbase)
{
    __shared__ uint32_t red[256];
    const uint32_t nwin = (nframes + LZX_WIN - 1) / LZX_WIN;
    unsigned long long base = 0;
    for (uint32_t w = 0; w < nwin; w++) {
        const uint32_t f0 = w * LZX_WIN, f1 = f0 + LZX_WIN < nframes ? f0 + LZX_WIN : nframes;
        uint32_t mx = 0;
        for (uint32_t f = f0 + threadIdx.x; f < f1; f += 256) { const uint32_t c = (uint32_t)(first_slot[f + 1] - first_slot[f]); mx = c > mx ? c : mx; }
        red[threadIdx.x] = mx;
        __syncthreads();
        for (uint32_t d = 128; d > 0; d >>= 1) { if (threadIdx.x < d && red[threadIdx.x + d] > red[threadIdx.x]) red[threadIdx.x] = red[threadIdx.x + d]; __syncthreads(); }
        mx = red[0];
        __syncthreads();
        const unsigned long long real = first_slot[f1] - first_slot[f0], grid = (unsigned long long)(f1 - f0) * mx;
        const bool frame_major = grid > 8 * real + 65536;
        if (threadIdx.x == 0) wbase[w] = base | (frame_major ? (1ull << 63) : 0ull);
        base += frame_major ? real : grid;
    }
    if (threadIdx.x == 0) wbase[nwin] = base;
}

// STAGED: every step's output window lives in shared memory as well (chains of matches that feed each other run at shared
// memory latency).  zmt_lz4_decompress_device always launches the staged variant; the plain one (all reads from global
// memory) runs only when ZSTDMT_B200_LZ4_STAGED=0 is set, for A/B measurements and tests.
template <bool STAGED>
__global__ void __launch_bounds__(32 * LZD_WARPS)
lz4_exec_blocks_kernel(uint8_t* __restrict__ out, const uint64_t* __restrict__ out_off, const uint64_t* __restrict__ frame_off,
                       const uint64_t* __restrict__ first_slot, const LzBlk* __restrict__ tab, const unsigned long long* __restrict__ rec,
                       uint32_t* __restrict__ prog, const uint32_t* __restrict__ status, const uint32_t* __restrict__ needs_seq,
                       unsigned long long* __restrict__ ticket, const unsigned long long* __restrict__ wbase, uint32_t nframes, uint32_t slot_cap)
{
    __shared__ __align__(16) uint8_t stage[STAGED ? LZD_WARPS : 1][STAGED ? LZX_SPAN + 32 : 16];
    const uint32_t lane = threadIdx.x & 31;
    if (first_slot[nframes] > slot_cap) return;             // the scan reported the undersized table per frame
    const uint32_t nwin = (nframes + LZX_WIN - 1) / LZX_WIN;
    const unsigned long long ntickets = wbase[nwin] & ~(1ull << 63);
    volatile uint32_t* vprog = prog;
    for (;;) {
        unsigned long long tk = 0;
        if (lane == 0) tk = atomicAdd(ticket, 1ull);
        tk = __shfl_sync(ZMT_FULL_MASK, tk, 0);
        if (tk >= ntickets) break;
        // ticket -> window (binary search over the window bases) -> (frame, block) -> slot
        uint32_t lo = 0, hi = nwin;
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if ((wbase[mid] & ~(1ull << 63)) <= tk) lo = mid; else hi = mid; }
        const unsigned long long wb = wbase[lo];
        const unsigned long long tl = tk - (wb & ~(1ull << 63));
        const uint32_t f0 = lo * LZX_WIN, wn = (f0 + LZX_WIN < nframes ? LZX_WIN : nframes - f0);
        uint64_t t;
        if (wb >> 63) t = first_slot[f0] + tl;                          // frame-major window
        else {
            const uint32_t fb = (uint32_t)(tl / wn), ff = f0 + (uint32_t)(tl % wn);
            const uint64_t s0 = first_slot[ff];
            if (fb >= first_slot[ff + 1] - s0) continue;                // this frame has fewer blocks
            t = s0 + fb;
        }
        const LzBlk B = tab[t];
        if (B.csize == 0) continue;                         // empty slot: nobody waits on it
        const uint32_t f = B.frame;
        const bool skip = (B.csize & 0x80000000u) || B.nrec == 0 || (status[f] & 0xFF) != 0 || needs_seq[f] != 0;
        if (!skip) {
            const uint32_t slot = (uint32_t)(t - first_slot[f]);
            const uint32_t blklog = (B.flags >> 8) & 0xFF, blkmax = 1u << blklog;
            uint8_t* dst = out + out_off[f] + ((uint64_t)slot << blklog);
            const unsigned long long* R = rec + (frame_off[f] + 12 + B.src + 2) / 3;
            const bool linked = (B.flags & LZB_LINKED) != 0;
            const bool publish = !(B.flags & LZB_LAST) && (tab[t + 1].flags & LZB_LINKED);     // the next block may read this one
            bool prev_done = !linked;
            uint32_t since_pub = 0;
            uint8_t* const S = stage[STAGED ? (threadIdx.x >> 5) : 0];
            // The records of the NEXT step are loaded while this one executes (one L2 round trip less on the chain of a block).
            unsigned long long rnext = lane < B.nrec ? R[lane] : 0ull;
            for (uint32_t base = 0; base < B.nrec;) {
                const uint32_t cnt = B.nrec - base < 32 ? B.nrec - base : 32;
                uint32_t d = 0, ml = 0, off = 0;
                { const unsigned long long r = lane < cnt ? rnext : 0ull; d = (uint32_t)r & 0xFFFFFFu; ml = (uint32_t)(r >> 24) & 0xFFFFFFu; off = (uint32_t)(r >> 48); }
                const uint32_t d0 = __shfl_sync(ZMT_FULL_MASK, d, 0);
                // ---- the step = the longest prefix of these records whose destinations fit the staging window [d0, d0 + LZX_SPAN)
                const uint32_t nfit = STAGED ? __popc(__ballot_sync(ZMT_FULL_MASK, ml && d + ml - d0 <= LZX_SPAN)) : cnt;       // destinations are sorted: a prefix
                if (nfit == 0) {
                    // one match longer than the window: straight in global memory, by the whole warp
                    const uint32_t qml = __shfl_sync(ZMT_FULL_MASK, ml, 0), qoff = __shfl_sync(ZMT_FULL_MASK, off, 0);
                    if (!prev_done && qoff > d0) {
                        const int64_t e = (int64_t)blkmax + (int64_t)d0 - qoff + qml;
                        const uint32_t need = e > (int64_t)blkmax ? blkmax : (uint32_t)e;
                        uint32_t pv = 0;
                        if (lane == 0) { while ((pv = vprog[t - 1]) < need) __nanosleep(100); }
                        pv = __shfl_sync(ZMT_FULL_MASK, pv, 0);
                        __threadfence();
                        if (pv == LZD_DONE) prev_done = true;
                    }
                    uint8_t* dp = dst + d0;
                    const uint8_t* m = dp - qoff;
                    if (qoff >= qml) warp_copy_lit(dp, m, qml, lane);
                    else if (qoff >= 32) { for (uint32_t i = 0; i < qml; i += 32) { if (i + lane < qml) dp[i + lane] = m[i + lane]; __syncwarp(); } }
                    else { for (uint32_t i = lane; i < qml; i += 32) dp[i] = m[i % qoff]; }
                    __syncwarp();
                    base += 1;
                    rnext = base + lane < B.nrec ? R[base + lane] : 0ull;
                    continue;
                }
                rnext = base + nfit + lane < B.nrec ? R[base + nfit + lane] : 0ull;      // in flight until the next step reads it
                if (lane >= nfit) ml = 0;
                const uint32_t span = __shfl_sync(ZMT_FULL_MASK, d + ml, nfit - 1) - d0;
                const int32_t sp = (int32_t)d - (int32_t)off;           // block-relative source; negative = previous block
                if (!prev_done) {
                    // bytes of the previous block this step needs complete
                    uint32_t need = 0;
                    if (ml && sp < 0) { const int64_t e = (int64_t)blkmax + sp + ml; need = e > (int64_t)blkmax ? blkmax : (uint32_t)e; }
#pragma unroll
                    for (int x = 16; x > 0; x >>= 1) { const uint32_t y = __shfl_xor_sync(ZMT_FULL_MASK, need, x); need = y > need ? y : need; }
                    if (need) {
                        uint32_t pv = 0;
                        if (lane == 0) { while ((pv = vprog[t - 1]) < need) __nanosleep(100); }
                        pv = __shfl_sync(ZMT_FULL_MASK, pv, 0);
                        __threadfence();                                // acquire: the producer's bytes are visible to every lane
                        if (pv == LZD_DONE) prev_done = true;
                    }
                }
                // Which matches must wait for an earlier match of this very step?  Only the destinations [d_j, e_j) of matches
                // j < k matter (sorted, disjoint): a = first j whose destination ends above my source start (binary search over
                // the lanes by shuffle); my source touches a destination of the step iff that j lies before me and starts below
                // my source end.  A match that overlaps its own destination (offset < length) takes the ordered path too.
                const int32_t e_end = ml ? (int32_t)(d + ml) : 0x7FFFFFFF, d_beg = ml ? (int32_t)d : 0x7FFFFFFF;
                uint32_t a = 0;
#pragma unroll
                for (uint32_t stp = 16; stp > 0; stp >>= 1) {
                    const int32_t v = __shfl_sync(ZMT_FULL_MASK, e_end, (a + stp - 1) & 31);
                    if (v <= sp) a += stp;                                  // e_j <= sp: destination j lies entirely below my source
                }
                const int32_t da = __shfl_sync(ZMT_FULL_MASK, d_beg, a & 31);
                const bool indep = ml && off >= ml && !(a < lane && da < sp + (int32_t)ml);
                const bool own = indep && ml <= LZD_LONG;               // copied by its own lane
                // own lane: the part of the source below d0 comes from global memory — its first 8 bytes are requested NOW, before
                // the window load below stalls on its own round trip (one latency per step instead of two)
                const int32_t nlow = !own ? 0 : !STAGED ? (int32_t)ml : sp >= (int32_t)d0 ? 0 : ((int32_t)d0 - sp < (int32_t)ml ? (int32_t)d0 - sp : (int32_t)ml);
                const uint8_t* mp = dst + sp;
                uint8_t x0[8];
#pragma unroll
                for (int j = 0; j < 8; j++) x0[j] = (j < nlow) ? mp[j] : (uint8_t)0;
                // ---- stage the window: output bytes [d0, d0 + span) as they stand (the literals pass A placed; match bytes are
                //      still undefined) with aligned 16-byte loads.  Every match of the step writes its bytes to global memory
                //      AND to the window; a source byte at or above d0 is read from the window.  A chain of matches that feed each
                //      other then runs at shared-memory latency instead of one L2 round trip per link.
                const uint32_t gsh = (uint32_t)((uintptr_t)(dst + d0) & 15);
                if (STAGED) {
                    const uint4* ga = reinterpret_cast<const uint4*>(dst + d0 - gsh);
                    const uint32_t nvec = (gsh + span + 15) >> 4;
                    for (uint32_t i = lane; i < nvec; i += 32) reinterpret_cast<uint4*>(S)[i] = ga[i];
                }
                const int32_t wb = (int32_t)gsh - (int32_t)d0;          // S[wb + p] = window byte of block position p (p >= d0)
                __syncwarp();
                if (own) {
                    uint8_t* dp = dst + d; uint8_t* dw = S + (wb + (int32_t)d);
#pragma unroll
                    for (int j = 0; j < 8; j++) if (j < nlow) { dp[j] = x0[j]; if (STAGED) dw[j] = x0[j]; }
                    int32_t i = 8;
                    for (; i < nlow; i += 8) {                              // loads first, stores after: one L2 latency per 8 bytes, not per byte
                        uint8_t x[8];
#pragma unroll
                        for (int j = 0; j < 8; j++) x[j] = (i + j < nlow) ? mp[i + j] : (uint8_t)0;
#pragma unroll
                        for (int j = 0; j < 8; j++) if (i + j < nlow) { dp[i + j] = x[j]; if (STAGED) dw[i + j] = x[j]; }
                    }
                    i = nlow;
                    for (; i < (int32_t)ml; i++) { const uint8_t x = S[wb + sp + i]; dp[i] = x; dw[i] = x; }        // STAGED only (nlow == ml otherwise)
                }
                uint32_t dm = __ballot_sync(ZMT_FULL_MASK, ml && !own);      // long independent ones too: whole warp
                if (dm) __syncwarp();
                while (dm) {                                            // in order: may read matches of this very step, or themselves
                    const int jq = __ffs(dm) - 1; dm &= dm - 1;
                    const uint32_t qd = __shfl_sync(ZMT_FULL_MASK, d, jq), qml = __shfl_sync(ZMT_FULL_MASK, ml, jq), qoff = __shfl_sync(ZMT_FULL_MASK, off, jq);
                    const int32_t qs = (int32_t)qd - (int32_t)qoff;
                    uint8_t* dp = dst + qd; uint8_t* dw = S + (wb + (int32_t)qd);
                    if (qoff >= qml && !STAGED && qml >= 64) warp_copy_lit(dp, dst + qs, qml, lane);
                    else if (qoff >= qml) {
                        for (uint32_t i = lane; i < qml; i += 32) { const int32_t q = qs + (int32_t)i; const uint8_t x = (STAGED && q >= (int32_t)d0) ? S[wb + q] : dst[q]; dp[i] = x; if (STAGED) dw[i] = x; }
                    } else if (qoff >= 32) {                            // overlapping, period >= warp width: 32-byte waves
                        for (uint32_t i = 0; i < qml; i += 32) {
                            if (i + lane < qml) { const int32_t q = qs + (int32_t)(i + lane); const uint8_t x = (STAGED && q >= (int32_t)d0) ? S[wb + q] : dst[q]; dp[i + lane] = x; if (STAGED) dw[i + lane] = x; }
                            __syncwarp();
                        }
                    } else {                                            // short period: replicate the pattern
                        for (uint32_t i = lane; i < qml; i += 32) { const int32_t q = qs + (int32_t)(i % qoff); const uint8_t x = (STAGED && q >= (int32_t)d0) ? S[wb + q] : dst[q]; dp[i] = x; if (STAGED) dw[i] = x; }
                    }
                    __syncwarp();
                }
                __syncwarp();
                base += nfit;
                if (publish && ++since_pub == 4 && base < B.nrec) {
                    since_pub = 0;
                    // everything below the first match of the next step is final (literals were placed by pass A)
                    const uint32_t upto = (uint32_t)R[base] & 0xFFFFFFu;
                    if (lane == 0) { __threadfence(); vprog[t] = upto; }
                }
            }
        }
        __syncwarp();
        if (lane == 0) { __threadfence(); vprog[t] = LZD_DONE; }
    }
}

// ---------------------------------------------------------------- sequential fallback (one warp per flagged frame)
#define D_WIN   1024u
struct DWin { uint8_t* w; const uint8_t* gsrc; const uint8_t* in_end; int32_t pos; };   // pos: block-relative offset of w[0]

__device__ __forceinline__ void dwin_fill(DWin& W, uint32_t ip, uint32_t lane)
{
    const int32_t np = (int32_t)ip - (int32_t)((uintptr_t)(W.gsrc + ip) & 15);
    __syncwarp();
#pragma unroll
    for (uint32_t k = 0; k < D_WIN / 512; k++) {
        const uint8_t* a = W.gsrc + np + (int32_t)(16 * (lane + 32 * k));
        uint4 v = make_uint4(0, 0, 0, 0);
        if (a + 16 <= W.in_end) v = *reinterpret_cast<const uint4*>(a);
        else { uint8_t* b = reinterpret_cast<uint8_t*>(&v); for (int i = 0; i < 16; i++) if (a + i < W.in_end) b[i] = a[i]; }
        reinterpret_cast<uint4*>(W.w)[lane + 32 * k] = v;
    }
    W.pos = np;
    __syncwarp();
}
// make bytes [ip, ip + k) of the block available in the window (k <= D_WIN - 16)
__device__ __forceinline__ void dwin_need(DWin& W, uint32_t ip, uint32_t k, uint32_t lane)
{
    if ((int32_t)ip < W.pos || (int32_t)(ip + k) > W.pos + (int32_t)D_WIN) dwin_fill(W, ip, lane);
}
__device__ __forceinline__ uint32_t dwin_byte(const DWin& W, uint32_t ip) { return W.w[(int32_t)ip - W.pos]; }

// returns decoded size or 0xFFFFFFFF on error.  `hist` = bytes of valid history before dst.
__device__ uint32_t warp_decode_block(DWin& W, uint32_t srcSize, uint8_t* dst, uint32_t dstCap, uint64_t hist, uint32_t lane)
{
    uint32_t ip = 0, op = 0;
    if (srcSize == 0) return 0xFFFFFFFFu;
    for (;;) {
        if (ip >= srcSize) return 0xFFFFFFFFu;
        dwin_need(W, ip, 20, lane);                         // token + a few length bytes + short literals' head
        const uint32_t token = dwin_byte(W, ip++);
        uint32_t lit = token >> 4;
        if (lit == 15) {
            uint32_t b;
            do { if (ip >= srcSize) return 0xFFFFFFFFu; dwin_need(W, ip, 1, lane); b = dwin_byte(W, ip++); lit += b; } while (b == 255);
        }
        if (lit > srcSize - ip || lit > dstCap - op) return 0xFFFFFFFFu;
        if (lit) {
            if (lit <= 256) {                               // short run: out of the window
                dwin_need(W, ip, lit, lane);
                const uint8_t* s = W.w + ((int32_t)ip - W.pos);
                for (uint32_t i = lane; i < lit; i += 32) dst[op + i] = s[i];
            } else warp_copy_lit(dst + op, W.gsrc + ip, lit, lane);
        }
        ip += lit; op += lit;
        if (ip == srcSize) break;
        if (srcSize - ip < 2) return 0xFFFFFFFFu;
        dwin_need(W, ip, 3, lane);
        const uint32_t off = dwin_byte(W, ip) | (dwin_byte(W, ip + 1) << 8);
        ip += 2;
        if (off == 0 || (uint64_t)off > (uint64_t)op + hist) return 0xFFFFFFFFu;
        uint32_t ml = token & 15;
        if (ml == 15) {
            uint32_t b;
            do { if (ip >= srcSize) return 0xFFFFFFFFu; dwin_need(W, ip, 1, lane); b = dwin_byte(W, ip++); ml += b; } while (b == 255);
        }
        ml += 4;
        if (ml > dstCap - op) return 0xFFFFFFFFu;
        __syncwarp();                                      // literals (and earlier matches) visible to all lanes
        uint8_t* d = dst + op;
        const uint8_t* m = d - off;
        if (off >= ml) { for (uint32_t i = lane; i < ml; i += 32) d[i] = m[i]; }
        else if (off >= 32) {                              // overlapping, period >= warp width: 32-byte waves
            for (uint32_t i = 0; i < ml; i += 32) { if (i + lane < ml) d[i + lane] = m[i + lane]; __syncwarp(); }
        } else {                                           // short period: replicate the pattern
            for (uint32_t i = lane; i < ml; i += 32) d[i] = m[i % off];
        }
        op += ml;
        __syncwarp();
    }
    return op;
}

// Frames flagged by the scan / pass A: blocks in order, output positions from the decoded sizes.  The frame header was
// validated by the scan (a frame whose header failed is never flagged).
__global__ void __launch_bounds__(32 * LZD_WARPS)
lz4_decode_frames_seq_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ in_end, const uint64_t* __restrict__ frame_off,
                             const uint32_t* __restrict__ frame_csize, uint8_t* __restrict__ out, const uint64_t* __restrict__ out_off,
                             unsigned long long* __restrict__ out_size, uint32_t* __restrict__ status, const uint32_t* __restrict__ needs_seq,
                             uint32_t nframes)
{
    __shared__ __align__(16) uint8_t win[LZD_WARPS][D_WIN];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t f = blockIdx.x * LZD_WARPS + wid;
    if (f >= nframes || !needs_seq[f]) return;
    const uint8_t* p = in + frame_off[f] + 12;
    const uint32_t fs = frame_csize[f];
    uint8_t* dst = out + out_off[f];
    const uint64_t cap = out_off[f + 1] - out_off[f];
    const uint32_t flg = p[4], bd = p[5];
    const uint32_t indep = (flg >> 5) & 1, bchk = (flg >> 4) & 1, csz = (flg >> 3) & 1, did = flg & 1;
    const uint32_t blkmax = 1u << (8 + 2 * ((bd >> 4) & 7));
    const uint32_t hl = 2 + (csz ? 8 : 0) + (did ? 4 : 0);
    __syncwarp();
    if (lane == 0) { status[f] &= ~0xFFu; out_size[f] = 0; }           // pass A may have reported an error for a mis-addressed block
    __syncwarp();
    DWin W; W.w = win[wid]; W.in_end = in_end;
    uint32_t ip = 4 + hl + 1;
    uint64_t total = 0;
    for (;;) {
        const uint32_t bh = ldg_le32(p + ip);               // block walk already bounds-checked by the scan
        if (bh == 0) break;
        ip += 4;
        const uint32_t bs = bh & 0x7FFFFFFFu;
        if (total > cap) { d_fail(status, f, ZMT_ST_DST_SMALL, lane); return; }
        uint32_t d;
        if (bh & 0x80000000u) {
            if (bs > cap - total) { d_fail(status, f, ZMT_ST_DST_SMALL, lane); return; }
            warp_copy_lit(dst + total, p + ip, bs, lane);
            d = bs;
        } else {
            const uint64_t room = cap - total;
            const uint32_t dcap = room < blkmax ? (uint32_t)room : blkmax;
            const uint64_t hist = indep ? 0 : (total < 65536 ? total : 65536);
            W.gsrc = p + ip; W.pos = 0x40000000;            // empty window
            d = warp_decode_block(W, bs, dst + total, dcap, hist, lane);
            if (d == 0xFFFFFFFFu) { d_fail(status, f, ZMT_ST_BLOCK, lane); return; }
        }
        if (bchk) {
            __syncwarp();
            const uint32_t h = warp_xxh32(p + ip, bs, reinterpret_cast<uint4(*)[32]>(W.w), lane);      // the window is refilled per block
            if (__shfl_sync(ZMT_FULL_MASK, h != ldg_le32(p + ip + bs), 0)) { d_fail(status, f, ZMT_ST_BLOCK, lane); return; }
        }
        ip += bs + (bchk ? 4 : 0);
        total += d;
        __syncwarp();
    }
    if (lane == 0) out_size[f] = total;
    (void)fs;
}

// content-size check + comparison of the recomputed XXH32 with the stored content checksum
__global__ void lz4_verify_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ frame_off, const uint32_t* __restrict__ frame_csize,
                                  uint32_t* __restrict__ status, const unsigned long long* __restrict__ out_size,
                                  const uint32_t* __restrict__ stored_chk, const uint32_t* __restrict__ computed, uint32_t nframes)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    uint32_t st = status[f];
    if ((st & 0xFF) == ZMT_ST_OK) {
        const uint8_t* p = in + frame_off[f] + 12;
        if (frame_csize[f] >= 15 && (p[4] & 0x08) && ldg_le64(p + 6) != out_size[f]) st = ZMT_ST_CONTENT_SIZE;
        else if ((st & ZMT_ST_HAS_CHK) && stored_chk[f] != computed[f]) st = ZMT_ST_CONTENT_CHECKSUM;
    }
    status[f] = st & 0xFF;
}
