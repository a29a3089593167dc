// lz4_pipe.cuh — the LZ4 block compressor as a two-team software pipeline (included by lz4_kernels.cu).
//
// Same algorithm and same output bytes as lz77_blocks_kernel<0,*> (oracle twin: orc_lz4_block_compress_b200);
// what changes is the schedule.  The per-tile work splits into a front end that carries (e, e_din) from tile to
// tile — candidates, speculative chain walks, path resolution — and a back end that carries the pending
// sequence and the output cursor — marking, piece merge, emission.  Neither needs the other's carry, so a CTA of
// 512 threads runs them as two teams of 256, the front end one tile ahead of the back end, over a
// double-buffered set of tile arrays.  Hand-off is by named barriers (bar.arrive / bar.sync, count 512):
// FULL[b] producer -> consumer, EMPTY[b] consumer -> producer.  With 2 CTAs per SM this gives four independent
// instruction streams per SM instead of two (the kernel is issue/latency bound: DESIGN.md §3).
//
// Shared memory: only what crosses the teams is double-buffered (off, M, V, entry positions, path mask: 9.5 KB per
// buffer).  Piece lengths do not cross: the front end does not store them, the marking walk of the back end
// recomputes them for the true-path pieces only (it has the slack), which keeps the 32-bit hash table and its
// single-pass atomicMax.  (A 16-bit table needs a CAS loop or a two-pass atomicMax per insert, both more instructions.)
#pragma once

#define P_TEAM      256u
#define PB_A        1u             // named barriers: team A, team B, FULL[2], EMPTY[2]   (0 = __syncthreads)
#define PB_B        2u
#define PB_FULL0    3u
#define PB_EMPTY0   5u
#define P_MAXPIECE  1280u         // 4096/4 match pieces + 256 continuation pieces, multiple of 256

// Barrier ids are immediates: ptxas reserves only the ids it sees (a register id makes it reserve all 16,
// and barriers are an occupancy resource).
template <uint32_t ID, uint32_t NTHREADS>
__device__ __forceinline__ void bar_sync()
{
    __syncwarp();                                   // aligned barrier: whole warps only (see CTA_SYNC)
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(NTHREADS) : "memory");
}
template <uint32_t ID, uint32_t NTHREADS>
__device__ __forceinline__ void bar_arrive()
{
    __syncwarp();
    __threadfence_block();
    asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(NTHREADS) : "memory");
}
#define TEAM_A_SYNC()   bar_sync<PB_A, P_TEAM>()
#define TEAM_B_SYNC()   bar_sync<PB_B, P_TEAM>()

struct __align__(16) PipeTile {
    uint16_t off[C_TILE];                 // candidate offset per tile position (0 = none)
    uint32_t M[C_TILE / 32];              // has-candidate bits
    uint32_t V[C_TILE / 32];              // visited-by-own-chain bits
    uint8_t  min_[C_CHAINS];              // entry position of a chain on the true path, relative to its own segment (< 16)
    uint32_t pathmask[C_CHAINS / 32];     // chains on the true path
    uint32_t k0, e_din, do_parse, pad;    // entry chain, offset of the match open at the entry, tile has work
};

struct __align__(16) PipeSmem {
    uint8_t  pad0[16];
    uint8_t  in[LZ4_BLK + 32];
    uint32_t tab[1 << C_HASHLOG];         // hash -> 1 + position
    PipeTile tile[2];
    // ---- front end (team A)
    uint32_t xfree[C_CHAINS];
    uint32_t mpos[C_CHAINS];
    uint16_t xdin[C_CHAINS];
    uint16_t link[C_CHAINS];
    uint8_t  jump[C_CHAINS];
    uint16_t entry[8];
    uint32_t e_next, d_next;
    uint32_t a_any[2];
    // ---- back end (team B)
    uint32_t Sel[C_TILE / 32];
    uint32_t Cont[C_TILE / 32];
    uint8_t  len[C_TILE];                 // piece length per selected piece start (written by the marking walk)
    uint16_t piece[P_MAXPIECE];
    union {                               // segprev is read by head detection, before the heads are written
        uint16_t hidx[C_TILE / 4];        // heads: one per sequence, sequences hold a match of >= 4 bytes
        uint16_t segprev[C_CHAINS];       // per segment: 1 + start of the last non-Cont piece before it (0: none)
    };
    uint32_t longl[2 * (C_TILE / (C_LONGLIT + 1) + 2)];   // jobs: literal runs > C_LONGLIT (start | length << 16, output offset) -- at most
                                                           // 4096/37 + 1 pending per tile -- and 255-runs of match lengths >= 1290 (count, offset | 1<<31)
    __align__(16) uint32_t scanws[16];
    uint32_t nlong;
    uint32_t fin_anchor, fin_out;
    uint64_t mbar;
};
static_assert(sizeof(PipeSmem) + 1024 <= (228 * 1024) / 2, "two CTAs per SM");

// what c_walk / c_emit_seq touch, with the tile arrays of the current buffer
struct PipeView {
    static constexpr bool relen = true;   // the front end does not keep piece lengths: the marking walk recomputes them
    const uint8_t* in; uint16_t* off; uint8_t* len; uint32_t* M; uint32_t* V; uint32_t* Sel; uint32_t* Cont;
    uint32_t* xfree; uint16_t* xdin; uint16_t* link; uint32_t* mpos; uint32_t* longl; uint32_t& nlong;
};

// exclusive scan over one team (8 warps); one team barrier; `ws` = two 8-word halves used alternately
template <uint32_t BARID>
__device__ __forceinline__ uint32_t team_exscan1(uint32_t v, uint32_t* ws, uint32_t parity, uint32_t* total, uint32_t twid, uint32_t lane)
{
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc += y; }
    uint32_t* w = ws + 8 * (parity & 1);
    if (lane == 31) w[twid] = inc;
    bar_sync<BARID, P_TEAM>();
    const uint4 a = *reinterpret_cast<const uint4*>(w), b = *reinterpret_cast<const uint4*>(w + 4);
    const uint32_t x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (uint32_t k = 0; k < 8; k++) { tot += x[k]; if (k < twid) base += x[k]; }
    *total = tot;
    return base + inc - v;
}

// the piece-list scan: team_exscan1 of v plus, with the same barrier, the exclusive max of m (m is 0 or grows with
// the thread index, so that is the last nonzero m below this thread).  `ws`: sums in words 0-7, maxima in words 8-15.
template <uint32_t BARID>
__device__ __forceinline__ uint32_t team_exscan_pieces(uint32_t v, uint32_t m, uint32_t* ws, uint32_t* total, uint32_t* mprev,
                                                      uint32_t twid, uint32_t lane)
{
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc += y; }
    const uint32_t below = __ballot_sync(ZMT_FULL_MASK, m != 0) & ((1u << lane) - 1);
    uint32_t mex = __shfl_sync(ZMT_FULL_MASK, m, below ? 31 - __clz(below) : 0);
    if (!below) mex = 0;
    if (lane == 31) { ws[twid] = inc; ws[8 + twid] = m ? m : mex; }
    bar_sync<BARID, P_TEAM>();
    const uint4 a = *reinterpret_cast<const uint4*>(ws), b = *reinterpret_cast<const uint4*>(ws + 4);
    const uint4 c = *reinterpret_cast<const uint4*>(ws + 8), d = *reinterpret_cast<const uint4*>(ws + 12);
    const uint32_t x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}, y[8] = {c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w};
    uint32_t base = 0, tot = 0, mx = mex;
#pragma unroll
    for (uint32_t k = 0; k < 8; k++) { tot += x[k]; if (k < twid) { base += x[k]; mx = max(mx, y[k]); } }
    *total = tot;
    *mprev = mx;
    return base + inc - v;
}

__global__ void __launch_bounds__(2 * P_TEAM, 2)
lz4_blocks_pipe_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                       uint32_t bpc, uint8_t* __restrict__ tmp, uint32_t* __restrict__ blk_csize, uint32_t nblocks, uint32_t flags)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    PipeSmem& S = *reinterpret_cast<PipeSmem*>(smem_raw);
    constexpr uint32_t NT = 2 * P_TEAM;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint32_t team = tid >> 8, ttid = tid & (P_TEAM - 1), twid = ttid >> 5;

    for (uint32_t blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const uint32_t chunk = blk / bpc, bic = blk % bpc;
        const uint64_t cbase = (uint64_t)chunk * chunk_size;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, chunk, in_bytes, chunk_size);
        const uint64_t boff = (uint64_t)bic * LZ4_BLK;
        uint32_t n = 0;
        if (boff < cbytes) n = (uint32_t)((cbytes - boff) < LZ4_BLK ? (cbytes - boff) : LZ4_BLK);
        if (n == 0) { if (tid == 0) blk_csize[blk] = 0; continue; }
        const uint8_t* src = in + cbase + boff;
        uint8_t* dst = tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE;

        // ---- stage the block into shared memory (TMA bulk copy when 16-byte aligned); all 512 threads
        CTA_SYNC();                                       // previous block fully consumed
        const uint32_t nb16 = ((((uintptr_t)src & 15) == 0) && !(flags & 1)) ? (n & ~15u) : 0;
        if (tid == 0) { if (nb16) mbar_init(&S.mbar, 1); S.nlong = 0; S.a_any[0] = 0; S.a_any[1] = 0; }
        CTA_SYNC();
        if (tid == 0 && nb16) { mbar_expect_tx(&S.mbar, nb16); bulk_g2s(S.in, src, nb16, &S.mbar); }
        for (uint32_t i = nb16 + tid; i < n; i += NT) S.in[i] = src[i];
        for (uint32_t i = n + tid; i < ((n + 3) & ~3u) + 32 && i < LZ4_BLK + 32; i += NT) S.in[i] = 0;
        if (tid < 16) S.pad0[tid] = 0;
        for (uint32_t i = tid; i < (1u << C_HASHLOG); i += NT) S.tab[i] = 0;
        if (tid == 0 && nb16) { mbar_wait(&S.mbar, 0); asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(&S.mbar))); }
        CTA_SYNC();

        const uint32_t limit = n >= 5 ? n - 5 : 0;        // matches end at or before n-5
        const uint32_t ntiles = (n + C_TILE - 1) / C_TILE;

        if (team == 0) {
            // =========================================================== front end: candidates, chains, true path
            uint32_t e = 0, e_din = 0;                    // team-uniform parse state (position, offset of the open match)
            for (uint32_t ti = 0; ti < ntiles; ti++) {
                const uint32_t t0 = ti * C_TILE, t1 = t0 + C_TILE, b = ti & 1;
                PipeTile& T = S.tile[b];
                if (ti >= 2) { if (b) bar_sync<PB_EMPTY0 + 1, 2 * P_TEAM>(); else bar_sync<PB_EMPTY0, 2 * P_TEAM>(); }               // back end released this buffer (tile ti-2)
                if (ttid < C_TILE / 32) T.V[ttid] = 0;
                uint32_t anyM = 0;
#pragma unroll 1
                for (uint32_t r = 0; r < C_TILE / C_ROUND; r++) {
                    // four consecutive positions per thread: three aligned words hold the windows of all four, the four
                    // offsets go out as one 8-byte store, and eight lanes' 4-bit slices make one M word
                    static_assert(C_ROUND == 4 * P_TEAM, "a round is four positions per thread");
                    const uint32_t rel = r * C_ROUND + 4 * ttid, i = t0 + rel;
                    const uint32_t* w = reinterpret_cast<const uint32_t*>(S.in) + (i >> 2);
                    const uint32_t w0 = w[-1], w1 = w[0], w2 = w[1];
                    uint32_t hreg[4], tab[4], o[4], m4 = 0;
                    // the four table reads, then the four window reads, are issued together: no position waits on another
#pragma unroll
                    for (uint32_t k = 0; k < 4; k++) {
                        hreg[k] = (__funnelshift_r(w1, w2, 8 * k) * 2654435761u) >> (32 - C_HASHLOG);
                        tab[k] = S.tab[hreg[k]];
                    }
#pragma unroll
                    for (uint32_t k = 0; k < 4; k++) {
                        const uint32_t ik = i + k;
                        const bool ok = (ik + 12 <= n);
                        const uint32_t v = __funnelshift_r(w1, w2, 8 * k), pv = __funnelshift_r(w0, w1, 8 * k);
                        const uint32_t t = tab[k];
                        const bool hit = t && lds32u(S.in, t ? t - 1 : 0) == v;
                        o[k] = 0;
                        if (ok) {
                            if (ik >= 1 && __funnelshift_r(pv, v, 24) == v) o[k] = 1;
                            else if (ik >= 2 && __funnelshift_r(pv, v, 16) == v) o[k] = 2;
                            else if (ik >= 3 && __funnelshift_r(pv, v, 8) == v) o[k] = 3;
                            else if (ik >= 4 && pv == v) o[k] = 4;
                            else if (hit) o[k] = ik - (t - 1);
                        }
                        if (!ok) hreg[k] = 0xFFFFFFFFu;
                        m4 |= (uint32_t)(o[k] != 0) << k;
                    }
                    *reinterpret_cast<uint2*>(&T.off[rel]) = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
                    uint32_t mw = m4 << (4 * (lane & 7));
                    mw |= __shfl_xor_sync(ZMT_FULL_MASK, mw, 1);
                    mw |= __shfl_xor_sync(ZMT_FULL_MASK, mw, 2);
                    mw |= __shfl_xor_sync(ZMT_FULL_MASK, mw, 4);
                    if ((lane & 7) == 0) T.M[rel >> 5] = mw;
                    anyM |= mw;
                    TEAM_A_SYNC();
                    if (r == 0 && ttid == 0) S.a_any[b ^ 1] = 0;       // every reader of the previous tile's flag is past it
#pragma unroll
                    for (uint32_t k = 0; k < 4; k++) {
                        bool last = hreg[k] != 0xFFFFFFFFu;     // a later position of the quad with the same hash wins anyway
#pragma unroll
                        for (uint32_t k2 = k + 1; k2 < 4; k2++) last &= hreg[k2] != hreg[k];
                        if (last) atomicMax(&S.tab[hreg[k]], i + k + 1);
                    }
                    TEAM_A_SYNC();
                }
                if ((lane & 7) == 0 && anyM) atomicOr(&S.a_any[b], 1u);   // anyM covers the lane's group of eight
                TEAM_A_SYNC();
                const bool tile_has_match = S.a_any[b] != 0;
                const bool do_parse = !((!tile_has_match && !e_din) || e >= t1);
                if (!do_parse) { if (e < t1) e = t1; if (ttid == 0) T.do_parse = 0; }
                else {
                    PipeView W{S.in, T.off, nullptr, T.M, T.V, S.Sel, S.Cont, S.xfree, S.xdin, S.link, S.mpos, S.longl, S.nlong};
                    const uint32_t k0 = (e - t0) / C_SEG;
                    const uint32_t seg0 = t0 + ttid * C_SEG;
                    const bool alive = ttid >= k0;
                    if (alive) c_walk<0>(W, ttid, ttid == k0 ? e : seg0, ttid == k0 ? e_din : 0u, t0, limit);
                    else S.link[ttid] = (uint16_t)ttid;                 // dead: self link, never reached
                    TEAM_A_SYNC();
                    if (alive) c_walk<1>(W, ttid, S.xfree[ttid], S.xdin[ttid], t0, limit);
                    TEAM_A_SYNC();
                    // which chains lie on the true path (see lz77_blocks_kernel phase 3)
                    const uint32_t lk = S.link[ttid];
                    const bool inwarp = (lk != C_END) && (lk != ttid) && ((lk >> 5) == twid);
                    uint32_t jmp = inwarp ? (lk & 31) : lane;
                    uint32_t pm = (1u << lane) | (1u << jmp);
#pragma unroll
                    for (int r = 0; r < 5; r++) { pm |= __shfl_sync(ZMT_FULL_MASK, pm, jmp); jmp = __shfl_sync(ZMT_FULL_MASK, jmp, jmp); }
                    S.jump[ttid] = (uint8_t)(32 * twid + jmp);
                    S.xfree[ttid] = pm;
                    if (ttid < 8) S.entry[ttid] = 0xFFFFu;
                    TEAM_A_SYNC();
                    if (ttid == 0) {
                        uint32_t cur = k0;
                        T.min_[k0] = (uint8_t)((e - t0) & (C_SEG - 1));
                        for (;;) {
                            S.entry[cur >> 5] = (uint16_t)cur;
                            const uint32_t t = S.jump[cur], tl = S.link[t];
                            if (tl == C_END) { S.e_next = S.mpos[t]; S.d_next = S.xdin[t]; break; }
                            T.min_[tl] = (uint8_t)((S.mpos[t] - t0) & (C_SEG - 1));
                            cur = tl;
                        }
                        T.k0 = k0; T.e_din = e_din; T.do_parse = 1;
                    }
                    TEAM_A_SYNC();
                    const uint32_t a = S.entry[twid];
                    const uint32_t pmask = (a != 0xFFFFu) ? S.xfree[a] : 0u;
                    if (lane == 0) T.pathmask[twid] = pmask;
                    if (((pmask >> lane) & 1u) && inwarp) T.min_[lk] = (uint8_t)((S.mpos[ttid] - t0) & (C_SEG - 1));
                    e = S.e_next; e_din = S.d_next;
                }
                if (b) bar_arrive<PB_FULL0 + 1, 2 * P_TEAM>(); else bar_arrive<PB_FULL0, 2 * P_TEAM>();
            }
        } else {
            // =========================================================== back end: mark, merge pieces, emit
            uint32_t out_pos = 0;
            uint32_t pd_valid = 0, pd_lit = 0, pd_start = 0, pd_off = 0, pd_end = 0;    // pending sequence (may still grow)
            for (uint32_t ti = 0; ti < ntiles; ti++) {
                const uint32_t t0 = ti * C_TILE, b = ti & 1;
                PipeTile& T = S.tile[b];
                PipeView W{S.in, T.off, S.len, T.M, T.V, S.Sel, S.Cont, S.xfree, S.xdin, S.link, S.mpos, S.longl, S.nlong};
                if (b) bar_sync<PB_FULL0 + 1, 2 * P_TEAM>(); else bar_sync<PB_FULL0, 2 * P_TEAM>();
                if (T.do_parse) do {
                    const uint32_t k0 = T.k0;
                    if (ttid < C_TILE / 32) { S.Sel[ttid] = 0; S.Cont[ttid] = 0; }
                    TEAM_B_SYNC();
                    if ((T.pathmask[twid] >> lane) & 1u) c_walk<2>(W, ttid, t0 + ttid * C_SEG + T.min_[ttid], ttid == k0 ? T.e_din : 0u, t0, limit);
                    TEAM_B_SYNC();
                    uint32_t np;
                    {
                        // one segment (16 positions) per thread.  segprev[j]: 1 + start of the last non-Cont piece before
                        // segment j (0: none), the piece whose offset a Cont piece at the start of segment j continues
                        const uint32_t sh = 16 * (ttid & 1);
                        uint32_t w = (S.Sel[ttid >> 1] >> sh) & 0xFFFFu;
                        const uint32_t nc = w & ~(S.Cont[ttid >> 1] >> sh);
                        const uint32_t last = nc ? ttid * C_SEG + (31 - __clz(nc)) + 1 : 0u;
                        uint32_t prev;
                        uint32_t base = team_exscan_pieces<PB_B>(__popc(w), last, S.scanws, &np, &prev, twid, lane);
                        S.segprev[ttid] = (uint16_t)prev;
                        while (w) { const uint32_t bit = __ffs(w) - 1; w &= w - 1; S.piece[base++] = (uint16_t)(ttid * C_SEG + bit); }
                    }
                    TEAM_B_SYNC();
                    if (np == 0) break;
                    // pieces and sequences are dealt in runs of ceil(count / 256) per thread, so every warp shares the work
                    uint32_t nh_local = 0, headmask = 0;
                    const uint32_t ppt = (np + P_TEAM - 1) / P_TEAM;
#pragma unroll
                    for (uint32_t k = 0; k < P_MAXPIECE / P_TEAM; k++) {
                        const uint32_t r = ttid * ppt + k;
                        if (k < ppt && r < np) {
                            const uint32_t pr = S.piece[r];
                            bool head = !((S.Cont[pr >> 5] >> (pr & 31)) & 1);
                            if (head) {
                                uint32_t pend, poff;
                                if (r == 0) { pend = pd_valid ? pd_end : 0xFFFFFFFFu; poff = pd_off; }
                                else {
                                    const uint32_t pb = S.piece[r - 1];
                                    pend = t0 + pb + S.len[pb];
                                    if (!((S.Cont[pb >> 5] >> (pb & 31)) & 1)) poff = T.off[pb];
                                    else {                      // Cont pieces start at a segment boundary (c_walk cuts there)
                                        const uint32_t sp = S.segprev[pb / C_SEG];
                                        poff = sp ? T.off[sp - 1] : pd_off;
                                    }
                                }
                                if (pend == t0 + pr && poff == T.off[pr]) head = false;
                            }
                            if (head) { headmask |= 1u << k; nh_local++; }
                        }
                    }
                    uint32_t nh;
                    {
                        uint32_t hb = team_exscan1<PB_B>(nh_local, S.scanws, 1, &nh, twid, lane);
#pragma unroll
                        for (uint32_t k = 0; k < P_MAXPIECE / P_TEAM; k++) if (headmask & (1u << k)) S.hidx[hb++] = (uint16_t)(ttid * ppt + k);
                    }
                    TEAM_B_SYNC();
                    const uint32_t lastp = S.piece[np - 1];
                    const uint32_t tile_end = t0 + lastp + S.len[lastp];
                    if (nh == 0) { pd_end = tile_end; break; }
                    if (pd_valid && S.hidx[0] > 0) { const uint32_t pb = S.piece[S.hidx[0] - 1]; pd_end = t0 + pb + S.len[pb]; }
                    const uint32_t nemit = pd_valid + nh - 1;
                    constexpr uint32_t SPT = 1024 / P_TEAM;
                    const uint32_t spt = (nemit + P_TEAM - 1) / P_TEAM;
                    uint32_t sz = 0, e_lit0[SPT], e_lit[SPT], e_off[SPT], e_len[SPT], cnt = 0;
#pragma unroll
                    for (uint32_t k = 0; k < SPT; k++) {
                        const uint32_t sidx = ttid * spt + k;
                        if (k < spt && sidx < nemit) {
                            uint32_t ls, st, of, en;
                            if (pd_valid && sidx == 0) { ls = pd_lit; st = pd_start; of = pd_off; en = pd_end; }
                            else {
                                const uint32_t h = sidx - pd_valid;
                                const uint32_t pi = S.hidx[h], pr = S.piece[pi];
                                const uint32_t pl = S.piece[S.hidx[h + 1] - 1];
                                st = t0 + pr; of = T.off[pr]; en = t0 + pl + S.len[pl];
                                if (h == 0) ls = pd_valid ? pd_end : pd_lit;
                                else { const uint32_t pp = S.piece[pi - 1]; ls = t0 + pp + S.len[pp]; }
                            }
                            e_lit0[k] = ls; e_lit[k] = st - ls; e_off[k] = of; e_len[k] = en - st;
                            sz += c_seq_size(e_lit[k], e_len[k]); cnt++;
                        }
                    }
                    uint32_t total;
                    uint32_t o = out_pos + team_exscan1<PB_B>(sz, S.scanws, 0, &total, twid, lane);
#pragma unroll
                    for (uint32_t k = 0; k < SPT; k++) {
                        if (k >= cnt) break;
                        o += c_emit_seq(W, dst, o, e_lit0[k], e_lit[k], e_off[k], e_len[k]);
                    }
                    TEAM_B_SYNC();
                    {
                        const uint32_t nl = S.nlong;
                        for (uint32_t s = twid; s < nl; s += P_TEAM / 32) c_long_job(W, dst, s, lane, 32u);
                        out_pos += total;
                        const uint32_t pi = S.hidx[nh - 1], pr = S.piece[pi];
                        uint32_t ls;
                        if (nh >= 2 || pd_valid) { if (pi > 0) { const uint32_t pp = S.piece[pi - 1]; ls = t0 + pp + S.len[pp]; } else ls = pd_end; }
                        else ls = pd_lit;
                        pd_valid = 1; pd_lit = ls; pd_start = t0 + pr; pd_off = T.off[pr]; pd_end = tile_end;
                        TEAM_B_SYNC();
                        if (ttid == 0) S.nlong = 0;
                    }
                } while (0);
                if (ti + 2 < ntiles) { if (b) bar_arrive<PB_EMPTY0 + 1, 2 * P_TEAM>(); else bar_arrive<PB_EMPTY0, 2 * P_TEAM>(); }     // the front end may refill this buffer
            }
            // ---- flush the pending sequence
            uint32_t anchor = 0;
            if (pd_valid) {
                PipeView W{S.in, S.tile[0].off, S.len, S.tile[0].M, S.tile[0].V, S.Sel, S.Cont, S.xfree, S.xdin, S.link, S.mpos, S.longl, S.nlong};
                anchor = pd_end;
                TEAM_B_SYNC();                                 // S.nlong = 0 of the last tile is visible
                if (ttid == 0) (void)c_emit_seq(W, dst, out_pos, pd_lit, pd_start - pd_lit, pd_off, pd_end - pd_start);
                out_pos += c_seq_size(pd_start - pd_lit, pd_end - pd_start);
                TEAM_B_SYNC();
                const uint32_t nl = S.nlong;                            // long literal run and / or long match length of the pending sequence
                for (uint32_t s = 0; s < nl; s++) c_long_job(W, dst, s, ttid, P_TEAM);
            }
            if (ttid == 0) { S.fin_anchor = anchor; S.fin_out = out_pos; }
        }
        CTA_SYNC();                                        // both teams drained
        {   // ---- last literals: all 512 threads
            const uint32_t anchor = S.fin_anchor, out_pos = S.fin_out;
            const uint32_t lit = n - anchor;
            const uint32_t fin = out_pos + 1 + lit + (lit >= 15 ? 1 + (lit - 15) / 255 : 0);
            if (fin >= n) { if (tid == 0) blk_csize[blk] = n | 0x80000000u; }   // stored block (LZ4F rule)
            else {
                uint8_t* op = dst + out_pos;
                uint32_t hl = 1;
                if (lit >= 15) hl += 1 + (lit - 15) / 255;
                const uint32_t nf = lit >= 15 ? (lit - 15) / 255 : 0;
                for (uint32_t i = tid; i < nf; i += NT) op[1 + i] = 255;
                if (tid == 0) {
                    op[0] = (uint8_t)((lit >= 15 ? 15u : lit) << 4);
                    if (lit >= 15) op[1 + nf] = (uint8_t)(lit - 15 - nf * 255);
                    blk_csize[blk] = fin;
                }
                for (uint32_t i = tid; i < lit; i += NT) op[hl + i] = S.in[anchor + i];
            }
        }
    }
}
