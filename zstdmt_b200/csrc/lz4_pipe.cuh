// lz4_pipe.cuh — the LZ77 parse as team functions, and the LZ4 block compressor that runs it as a two-team software
// pipeline (included by lz4_kernels.cu, whose Zstandard encoder runs the same functions with a single team).
//
// Oracle twin of the parse: orc_lz4_block_compress_b200.  The per-tile work splits into a front end that carries
// (e, e_din) from tile to tile — candidates, speculative chain walks, path resolution — and a back end that carries the
// pending sequence and the output cursor — marking, piece merge, emission.  Neither needs the other's carry, so a CTA of
// 512 threads runs them as two teams of 256, the front end one tile ahead of the back end, over a
// double-buffered set of tile arrays.  Hand-off is by named barriers (bar.arrive / bar.sync, count 512):
// FULL[b] producer -> consumer, EMPTY[b] consumer -> producer.  With 2 CTAs per SM this gives four independent
// instruction streams per SM instead of two (the kernel is issue/latency bound: DESIGN.md §3).
//
// Every phase below is run by one team of P_TEAM threads and takes that team's barrier id: PB_A / PB_B here, 0 in the
// Zstandard encoder, whose CTA is one team.
//
// Shared memory: only what crosses the teams is double-buffered (PipeTile: off, M, V, the 4-bit candidate piece lengths
// len4, entry positions, path mask: 11.3 KB per buffer).  The chain walks measure every candidate piece once and the
// marking walk of the back end reads the lengths back, so it compares bytes only for the continuation (Cont) pieces at
// segment starts, whose length depends on the offset carried in (LzBack::clen, one byte per segment).  That keeps the
// 32-bit hash table and its single-pass atomicMax within two CTAs per SM.  (A 16-bit table needs a CAS loop or a
// two-pass atomicMax per insert, both more instructions.)
#pragma once

#define P_TEAM      256u
#define PB_A        1u             // named barriers: team A, team B, FULL[2], EMPTY[2]   (0 = __syncthreads)
#define PB_B        2u
#define PB_FULL0    3u
#define PB_EMPTY0   5u
#define LZ_SPT      (1024u / P_TEAM)   // sequences per thread at most (<= 1024 per tile)

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
template <uint32_t BARID>
__device__ __forceinline__ void team_sync() { bar_sync<BARID, P_TEAM>(); }

// Per-phase cycle probe of lz4_blocks_pipe_kernel, built only with -DZMT_PHASE_PROBE (tools/lz4_phase_probe.py): thread 0
// of each team adds the clock64() cycles since its previous mark to the counter of the phase that mark closes.  The rows
// are those of DESIGN.md §3.4; a phase index means, for team A / team B:
//   0 staging            1 EMPTY wait / FULL wait      2 candidate rounds / marking walk    3 walk 0 / piece list
//   4 walk 1 / head detection    5 path resolution / emission + long jobs    6 FULL arrive / EMPTY arrive
//   7 final sync + last literals (team B: with the flush of the pending sequence)
// Without the define the marks are empty and the kernels compile as if they were not there.
#ifdef ZMT_PHASE_PROBE
#define ZMT_NPHASE 8
__device__ unsigned long long zmt_phase_cycles[2][ZMT_NPHASE];
__device__ __forceinline__ void zmt_phase_mark(uint32_t team, uint32_t ttid, int ph)     // ph < 0: start the clock
{
    __shared__ long long last[2];
    if (ttid == 0) {
        const long long now = clock64();
        if (ph >= 0) atomicAdd(&zmt_phase_cycles[team][ph], (unsigned long long)(now - last[team]));
        last[team] = now;
    }
}
#define ZMT_PHASE(team, ttid, ph) zmt_phase_mark((team), (ttid), (ph))
// inside the team functions: only the LZ4 pipeline's teams (the Zstandard encoder runs them with barrier id 0)
#define ZMT_PHASE_TEAM(BARID, ttid, ph) do { if constexpr ((BARID) != 0) zmt_phase_mark((BARID) == PB_B, (ttid), (ph)); } while (0)
#else
#define ZMT_PHASE(team, ttid, ph) ((void)0)
#define ZMT_PHASE_TEAM(BARID, ttid, ph) ((void)0)
#endif

// exclusive scan over one team (8 warps); one team barrier; `ws` = two 8-word halves used alternately
template <uint32_t BARID>
__device__ __forceinline__ uint32_t team_exscan1(uint32_t v, uint32_t* ws, uint32_t parity, uint32_t* total, uint32_t twid, uint32_t lane)
{
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc += y; }
    uint32_t* w = ws + 8 * (parity & 1);
    if (lane == 31) w[twid] = inc;
    team_sync<BARID>();
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
    team_sync<BARID>();
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

// ---------------------------------------------------------------- block staging (whole CTA, NT threads)
// Stages the n bytes at src into St.in (TMA bulk copy when 16-byte aligned), zeroes the pads and the hash table.  The
// caller has a CTA barrier between the previous block's last reader and this call.
template <uint32_t NT>
__device__ __forceinline__ void lz_stage(LzStage& St, uint32_t* tab, uint64_t* mbar, const uint8_t* src, uint32_t n, uint32_t tid)
{
    const uint32_t nb16 = (((uintptr_t)src & 15) == 0) ? (n & ~15u) : 0;
    if (tid == 0 && nb16) mbar_init(mbar, 1);
    CTA_SYNC();
    if (tid == 0 && nb16) { mbar_expect_tx(mbar, nb16); bulk_g2s(St.in, src, nb16, mbar); }
    for (uint32_t i = nb16 + tid; i < n; i += NT) St.in[i] = src[i];
    for (uint32_t i = n + tid; i < ((n + 3) & ~3u) + 32 && i < LZ4_BLK + 32; i += NT) St.in[i] = 0;
    if (tid < 16) St.pad0[tid] = 0;
    for (uint32_t i = tid; i < (1u << C_HASHLOG); i += NT) tab[i] = 0;
    // one thread observes the TMA completion; the CTA barrier publishes the staged bytes to everyone
    if (tid == 0 && nb16) { mbar_wait(mbar, 0); asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(mbar))); }
    CTA_SYNC();
}

// ---------------------------------------------------------------- front end
// Candidate rounds of the tile at t0 (4 rounds of 1024 positions): fills T.off and T.M.  Returns, uniform
// over the team, whether the tile has a candidate.  any[2] holds that flag per tile parity b; any[b ^ 1] is cleared in
// round 0, once every reader of the previous tile's flag is past the round's first barrier.
template <uint32_t BARID>
__device__ __forceinline__ bool lz_candidates(const uint8_t* in, uint32_t* tab, PipeTile& T, uint32_t* any, uint32_t b,
                                              uint32_t t0, uint32_t n, uint32_t ttid, uint32_t lane)
{
    uint32_t anyM = 0;
#pragma unroll 1
    for (uint32_t r = 0; r < C_TILE / C_ROUND; r++) {
        // four consecutive positions per thread: three aligned words hold the windows of all four, the four
        // offsets go out as one 8-byte store, and eight lanes' 4-bit slices make one M word
        static_assert(C_ROUND == 4 * P_TEAM, "a round is four positions per thread");
        const uint32_t rel = r * C_ROUND + 4 * ttid, i = t0 + rel;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(in) + (i >> 2);
        const uint32_t w0 = w[-1], w1 = w[0], w2 = w[1];
        uint32_t h[4], tv[4], x[4], o[4], m4 = 0;
        // The round is straight-line code from the first table read to the offset store: the four table reads, then
        // the four verifying reads, issued unconditionally so that none waits on another position's compare (an empty
        // slot, t = 0, reads the word below the block, pad0, and is masked out), and the candidate is chosen by selects.
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            h[k] = (__funnelshift_r(w1, w2, 8 * k) * 2654435761u) >> (32 - C_HASHLOG);
            tv[k] = tab[h[k]];
        }
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            const int32_t a = (int32_t)(tv[k] - 1);                     // -1 for an empty slot
            const uint32_t* q = reinterpret_cast<const uint32_t*>(in) + (a >> 2);
            x[k] = __funnelshift_r(q[0], q[1], 8u * (uint32_t)a);      // the shift counts modulo 32
        }
        // i is a multiple of 4, so i + k >= d fails only in the block's first quad, for d > k
        const bool first = (i == 0);
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            const uint32_t ik = i + k;
            const uint32_t v = __funnelshift_r(w1, w2, 8 * k), pv = __funnelshift_r(w0, w1, 8 * k);
            const uint32_t t = tv[k];
            const bool hit = (t != 0) & (x[k] == v);
            // short-period candidates d = 1..4: v(i-d) is a byte-shift of the window; the smallest d wins, then the table
            const bool e1 = (__funnelshift_r(pv, v, 24) == v) & !(first & (k < 1));
            const bool e2 = (__funnelshift_r(pv, v, 16) == v) & !(first & (k < 2));
            const bool e3 = (__funnelshift_r(pv, v, 8) == v) & !(first & (k < 3));
            const bool e4 = (pv == v) & !first;
            uint32_t of = hit ? ik - (t - 1) : 0u;
            of = e4 ? 4u : of;
            of = e3 ? 3u : of;
            of = e2 ? 2u : of;
            of = e1 ? 1u : of;
            o[k] = (ik + 12 <= n) ? of : 0u;                            // LZ4 MFLIMIT: only the block's last quads fail
            m4 |= (uint32_t)(o[k] != 0) << k;
        }
        *reinterpret_cast<uint2*>(&T.off[rel]) = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
        uint32_t mw = m4 << (4 * (lane & 7));
        mw |= __shfl_xor_sync(ZMT_FULL_MASK, mw, 1);
        mw |= __shfl_xor_sync(ZMT_FULL_MASK, mw, 2);
        mw |= __shfl_xor_sync(ZMT_FULL_MASK, mw, 4);
        if ((lane & 7) == 0) T.M[rel >> 5] = mw;
        anyM |= mw;
        team_sync<BARID>();
        if (r == 0 && ttid == 0) any[b ^ 1] = 0;
        // inserts: positions past the MFLIMIT are not inserted, and a later eligible position of the quad with the same
        // hash wins anyway.  A skipped insert is a max with 0, a no-op: ptxas puts a branch region around every
        // predicated shared atomic, even a predicated red.shared.
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            uint32_t val = (i + k + 12 <= n) ? i + k + 1 : 0u;
#pragma unroll
            for (uint32_t k2 = k + 1; k2 < 4; k2++) val = (h[k2] == h[k] && i + k2 + 12 <= n) ? 0u : val;
            atomicMax(&tab[h[k]], val);
        }
        team_sync<BARID>();
    }
    if ((lane & 7) == 0 && anyM) atomicOr(&any[b], 1u);   // anyM covers the lane's group of eight
    team_sync<BARID>();
    return any[b] != 0;
}

// Speculative chains (own segment, then continuation) and the true path through the tile, entered at e inside a match
// of offset e_din (0: free).  Hands the path to the back end (T.k0, T.e_din, T.min_, T.pathmask, T.do_parse) and moves
// (e, e_din) to where it leaves the tile.  A tile without candidates or open match, or one the parse has already passed,
// is skipped.  Returns T.do_parse.
template <uint32_t BARID>
__device__ __forceinline__ bool lz_chains(const uint8_t* in, PipeTile& T, LzFront& F, bool has_match, uint32_t& e, uint32_t& e_din,
                                          uint32_t t0, uint32_t limit, uint32_t ttid, uint32_t lane)
{
    const uint32_t t1 = t0 + C_TILE, twid = ttid >> 5;
    if ((!has_match && !e_din) || e >= t1) {
        if (e < t1) e = t1;
        if (ttid == 0) T.do_parse = 0;
        return false;
    }
    const uint32_t k0 = (e - t0) / C_SEG;
    const uint32_t seg0 = t0 + ttid * C_SEG;
    const bool alive = ttid >= k0;
    if (alive) c_walk0(in, T, F, ttid, ttid == k0 ? e : seg0, ttid == k0 ? e_din : 0u, t0, limit);
    else {                                               // dead: self link, never reached; no V bits, no pieces
        F.link[ttid] = (uint16_t)ttid;
        reinterpret_cast<uint16_t*>(T.V)[ttid] = 0;
        *reinterpret_cast<uint2*>(&T.len4[2 * ttid]) = make_uint2(0u, 0u);
    }
    team_sync<BARID>();
    ZMT_PHASE_TEAM(BARID, ttid, 3);
    if (alive) c_walk<1>(in, T, F, ttid, F.xfree[ttid], F.xdin[ttid], t0, limit);
    team_sync<BARID>();
    ZMT_PHASE_TEAM(BARID, ttid, 4);
    // Which chains lie on the true path (entry k0, follow the links).  Links only go forward.  Each warp resolves its
    // own 32 chains with shuffles (pointer doubling on lane indices: terminal chain + bitmask of the lanes on the way),
    // one thread then hops from warp to warp (<= 8 hops), and each warp reads its path mask back: 2 barriers, not 18.
    const uint32_t lk = F.link[ttid];
    const bool inwarp = (lk != C_END) && (lk != ttid) && ((lk >> 5) == twid);
    uint32_t jmp = inwarp ? (lk & 31) : lane;                 // next lane inside this warp (self = terminal)
    uint32_t pm = (1u << lane) | (1u << jmp);
#pragma unroll
    for (int r = 0; r < 5; r++) { pm |= __shfl_sync(ZMT_FULL_MASK, pm, jmp); jmp = __shfl_sync(ZMT_FULL_MASK, jmp, jmp); }
    F.jump[ttid] = (uint8_t)(32 * twid + jmp);
    F.xfree[ttid] = pm;                                       // xfree is dead after the continuation walk
    if (ttid < 8) F.entry[ttid] = 0xFFFFu;
    team_sync<BARID>();
    if (ttid == 0) {
        uint32_t cur = k0;
        T.min_[k0] = (uint8_t)((e - t0) & (C_SEG - 1));
        for (;;) {
            F.entry[cur >> 5] = (uint16_t)cur;
            const uint32_t t = F.jump[cur], tl = F.link[t];
            if (tl == C_END) { F.e_next = F.mpos[t]; F.d_next = F.xdin[t]; break; }
            T.min_[tl] = (uint8_t)((F.mpos[t] - t0) & (C_SEG - 1));   // entry position of the next warp's first chain on the path
            cur = tl;
        }
        T.k0 = k0; T.e_din = e_din; T.do_parse = 1;
    }
    team_sync<BARID>();
    const uint32_t a = F.entry[twid];
    const uint32_t pmask = (a != 0xFFFFu) ? F.xfree[a] : 0u;
    if (lane == 0) T.pathmask[twid] = pmask;
    // in-warp successor: its entry position is my merge position
    if (((pmask >> lane) & 1u) && inwarp) T.min_[lk] = (uint8_t)((F.mpos[ttid] - t0) & (C_SEG - 1));
    e = F.e_next; e_din = F.d_next;
    return true;
}

// ---------------------------------------------------------------- back end
// pending sequence: the last one found so far; its match may still grow in the next tile, so it is emitted one tile late
struct LzPending { uint32_t valid, lit, start, off, end; };

// length of the selected piece at tile position pr: a Cont piece's from the marking walk, any other from the front end
__device__ __forceinline__ uint32_t lz_piece_len(const PipeTile& T, const LzBack& K, uint32_t pr)
{
    return ((K.Cont[pr >> 5] >> (pr & 31)) & 1u) ? K.clen[pr / C_SEG] : 4u + ((T.len4[pr >> 3] >> (4 * (pr & 7))) & 15u);
}

// Marks the pieces of the true path (c_walk reads their lengths), lists them, and finds the HEADS: piece r starts
// a sequence unless it continues the previous piece's match -- flagged continuation, or contiguous with the same
// offset (the effective offset of a flagged piece is that of the nearest unflagged piece before it).  Returns the
// number of heads nh (0 when nothing is marked); the pending match grows over the pieces before the first head.
template <uint32_t BARID>
__device__ __forceinline__ uint32_t lz_heads(const uint8_t* in, PipeTile& T, LzBack& K, uint32_t* scanws, LzPending& pd, uint32_t& tile_end,
                                             uint32_t t0, uint32_t limit, uint32_t ttid, uint32_t lane)
{
    const uint32_t twid = ttid >> 5, k0 = T.k0;
    if (ttid < C_TILE / 32) { K.Sel[ttid] = 0; K.Cont[ttid] = 0; }
    team_sync<BARID>();
    if ((T.pathmask[twid] >> lane) & 1u) c_walk<2>(in, T, K, ttid, t0 + ttid * C_SEG + T.min_[ttid], ttid == k0 ? T.e_din : 0u, t0, limit);
    team_sync<BARID>();
    ZMT_PHASE_TEAM(BARID, ttid, 2);
    uint32_t np;
    {
        // one segment (16 positions) per thread.  segprev[j]: 1 + start of the last non-Cont piece before
        // segment j (0: none), the piece whose offset a Cont piece at the start of segment j continues
        const uint32_t sh = 16 * (ttid & 1);
        uint32_t w = (K.Sel[ttid >> 1] >> sh) & 0xFFFFu;
        const uint32_t nc = w & ~(K.Cont[ttid >> 1] >> sh);
        const uint32_t last = nc ? ttid * C_SEG + (31 - __clz(nc)) + 1 : 0u;
        uint32_t prev;
        uint32_t base = team_exscan_pieces<BARID>(__popc(w), last, scanws, &np, &prev, twid, lane);
        K.segprev[ttid] = (uint16_t)prev;
        while (w) { const uint32_t bit = __ffs(w) - 1; w &= w - 1; K.piece[base++] = (uint16_t)(ttid * C_SEG + bit); }
    }
    team_sync<BARID>();
    ZMT_PHASE_TEAM(BARID, ttid, 3);
    if (np == 0) return 0;
    // pieces are dealt in runs of ceil(np / 256) per thread, so every warp shares the work
    uint32_t nh_local = 0, headmask = 0;
    const uint32_t ppt = (np + P_TEAM - 1) / P_TEAM;
#pragma unroll
    for (uint32_t k = 0; k < C_MAXPIECE / P_TEAM; k++) {
        const uint32_t r = ttid * ppt + k;
        if (k < ppt && r < np) {
            const uint32_t pr = K.piece[r];
            bool head = !((K.Cont[pr >> 5] >> (pr & 31)) & 1);
            if (head) {
                uint32_t pend, poff;                         // end and effective offset of what precedes piece r
                if (r == 0) { pend = pd.valid ? pd.end : 0xFFFFFFFFu; poff = pd.off; }
                else {
                    const uint32_t pb = K.piece[r - 1];
                    pend = t0 + pb + lz_piece_len(T, K, pb);
                    if (!((K.Cont[pb >> 5] >> (pb & 31)) & 1)) poff = T.off[pb];
                    else {                      // Cont pieces start at a segment boundary (c_walk cuts there)
                        const uint32_t sp = K.segprev[pb / C_SEG];
                        poff = sp ? T.off[sp - 1] : pd.off;
                    }
                }
                if (pend == t0 + pr && poff == T.off[pr]) head = false;
            }
            if (head) { headmask |= 1u << k; nh_local++; }
        }
    }
    uint32_t nh;
    {
        uint32_t hb = team_exscan1<BARID>(nh_local, scanws, 1, &nh, twid, lane);
#pragma unroll
        for (uint32_t k = 0; k < C_MAXPIECE / P_TEAM; k++) if (headmask & (1u << k)) K.hidx[hb++] = (uint16_t)(ttid * ppt + k);
    }
    team_sync<BARID>();
    const uint32_t lastp = K.piece[np - 1];
    tile_end = t0 + lastp + lz_piece_len(T, K, lastp);       // end of the last piece of this tile
    if (nh == 0) pd.end = tile_end;                           // every piece extends the pending sequence
    else if (pd.valid && K.hidx[0] > 0) { const uint32_t pb = K.piece[K.hidx[0] - 1]; pd.end = t0 + pb + lz_piece_len(T, K, pb); }
    return nh;
}

// this thread's run of the sequences the tile closes: [pending] + heads 0 .. nh-2, dealt in runs of ceil(count / 256)
// per thread (head nh-1 becomes the new pending sequence: lz_next_pending).  Per sequence: literals start, literal
// length, offset, match length.
struct LzRun { uint32_t cnt, lit0[LZ_SPT], lit[LZ_SPT], off[LZ_SPT], len[LZ_SPT]; };
__device__ __forceinline__ LzRun lz_seq_run(const PipeTile& T, const LzBack& K, const LzPending& pd, uint32_t nh, uint32_t t0, uint32_t ttid)
{
    LzRun R; R.cnt = 0;
    const uint32_t nemit = pd.valid + nh - 1;
    const uint32_t spt = (nemit + P_TEAM - 1) / P_TEAM;
#pragma unroll
    for (uint32_t k = 0; k < LZ_SPT; k++) {
        const uint32_t sidx = ttid * spt + k;
        if (k < spt && sidx < nemit) {
            uint32_t ls, st, of, en;
            if (pd.valid && sidx == 0) { ls = pd.lit; st = pd.start; of = pd.off; en = pd.end; }
            else {
                const uint32_t h = sidx - pd.valid;          // head index, h <= nh-2
                const uint32_t pi = K.hidx[h], pr = K.piece[pi];
                const uint32_t pl = K.piece[K.hidx[h + 1] - 1];
                st = t0 + pr; of = T.off[pr]; en = t0 + pl + lz_piece_len(T, K, pl);
                if (h == 0) ls = pd.valid ? pd.end : pd.lit;     // pd.lit doubles as "end of everything emitted so far"
                else { const uint32_t pp = K.piece[pi - 1]; ls = t0 + pp + lz_piece_len(T, K, pp); }
            }
            R.lit0[k] = ls; R.lit[k] = st - ls; R.off[k] = of; R.len[k] = en - st; R.cnt++;
        }
    }
    return R;
}

// after emission: the last head of the tile becomes the pending sequence
__device__ __forceinline__ void lz_next_pending(const PipeTile& T, const LzBack& K, LzPending& pd, uint32_t nh, uint32_t tile_end, uint32_t t0)
{
    const uint32_t pi = K.hidx[nh - 1], pr = K.piece[pi];
    uint32_t ls;
    if (nh >= 2 || pd.valid) { if (pi > 0) { const uint32_t pp = K.piece[pi - 1]; ls = t0 + pp + lz_piece_len(T, K, pp); } else ls = pd.end; }
    else ls = pd.lit;                          // first sequence of the block: literals start where emission stands (0)
    pd.valid = 1; pd.lit = ls; pd.start = t0 + pr; pd.off = T.off[pr]; pd.end = tile_end;
}

// ---------------------------------------------------------------- the LZ4 pipeline
struct __align__(16) PipeSmem {
    LzStage  stage;
    uint32_t tab[1 << C_HASHLOG];         // hash -> 1 + position
    PipeTile tile[2];
    LzFront  fe;                          // team A
    uint32_t a_any[2];
    LzBack   be;                          // team B
    __align__(16) uint32_t scanws[16];
    uint32_t nlong;
    uint32_t fin_anchor, fin_out;
    uint64_t mbar;
};
static_assert(sizeof(PipeSmem) + 1024 <= (228 * 1024) / 2, "two CTAs per SM");

__global__ void __launch_bounds__(2 * P_TEAM, 2)
lz4_blocks_pipe_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* __restrict__ chunk_bytes,
                       uint32_t bpc, uint8_t* __restrict__ tmp, uint32_t* __restrict__ blk_csize, uint32_t nblocks)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    PipeSmem& S = *reinterpret_cast<PipeSmem*>(smem_raw);
    constexpr uint32_t NT = 2 * P_TEAM;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint32_t team = tid >> 8, ttid = tid & (P_TEAM - 1), twid = ttid >> 5;
    ZMT_PHASE(team, ttid, -1);

    for (uint32_t blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const uint32_t chunk = blk / bpc, bic = blk % bpc;
        const uint64_t cbase = (uint64_t)chunk * chunk_size;
        const uint64_t cbytes = zmt_chunk_len(chunk_bytes, chunk, in_bytes, chunk_size);
        const uint64_t boff = (uint64_t)bic * LZ4_BLK;
        uint32_t n = 0;
        if (boff < cbytes) n = (uint32_t)((cbytes - boff) < LZ4_BLK ? (cbytes - boff) : LZ4_BLK);
        if (n == 0) { if (tid == 0) blk_csize[blk] = 0; continue; }
        uint8_t* dst = tmp + (uint64_t)blk * ZMT_LZ4_TMP_STRIDE;

        CTA_SYNC();                                       // previous block fully consumed
        if (tid == 0) { S.nlong = 0; S.a_any[0] = 0; S.a_any[1] = 0; }
        lz_stage<NT>(S.stage, S.tab, &S.mbar, in + cbase + boff, n, tid);
        ZMT_PHASE(team, ttid, 0);

        const uint32_t limit = n >= 5 ? n - 5 : 0;        // matches end at or before n-5
        const uint32_t ntiles = (n + C_TILE - 1) / C_TILE;

        if (team == 0) {
            // =========================================================== front end: candidates, chains, true path
            uint32_t e = 0, e_din = 0;                    // team-uniform parse state (position, offset of the open match)
            for (uint32_t ti = 0; ti < ntiles; ti++) {
                const uint32_t t0 = ti * C_TILE, b = ti & 1;
                PipeTile& T = S.tile[b];
                if (ti >= 2) { if (b) bar_sync<PB_EMPTY0 + 1, 2 * P_TEAM>(); else bar_sync<PB_EMPTY0, 2 * P_TEAM>(); }               // back end released this buffer (tile ti-2)
                ZMT_PHASE(0, ttid, 1);
                const bool has_match = lz_candidates<PB_A>(S.stage.in, S.tab, T, S.a_any, b, t0, n, ttid, lane);
                ZMT_PHASE(0, ttid, 2);
                lz_chains<PB_A>(S.stage.in, T, S.fe, has_match, e, e_din, t0, limit, ttid, lane);
                ZMT_PHASE(0, ttid, 5);
                if (b) bar_arrive<PB_FULL0 + 1, 2 * P_TEAM>(); else bar_arrive<PB_FULL0, 2 * P_TEAM>();
                ZMT_PHASE(0, ttid, 6);
            }
        } else {
            // =========================================================== back end: mark, merge pieces, emit
            uint32_t out_pos = 0;
            LzPending pd = {0, 0, 0, 0, 0};
            for (uint32_t ti = 0; ti < ntiles; ti++) {
                const uint32_t t0 = ti * C_TILE, b = ti & 1;
                PipeTile& T = S.tile[b];
                if (b) bar_sync<PB_FULL0 + 1, 2 * P_TEAM>(); else bar_sync<PB_FULL0, 2 * P_TEAM>();
                ZMT_PHASE(1, ttid, 1);
                if (T.do_parse) {
                    uint32_t tile_end;
                    const uint32_t nh = lz_heads<PB_B>(S.stage.in, T, S.be, S.scanws, pd, tile_end, t0, limit, ttid, lane);
                    ZMT_PHASE(1, ttid, 4);
                    if (nh) {
                        const LzRun R = lz_seq_run(T, S.be, pd, nh, t0, ttid);
                        uint32_t sz = 0;
#pragma unroll
                        for (uint32_t k = 0; k < LZ_SPT; k++) if (k < R.cnt) sz += c_seq_size(R.lit[k], R.len[k]);
                        uint32_t total;
                        uint32_t o = out_pos + team_exscan1<PB_B>(sz, S.scanws, 0, &total, twid, lane);
#pragma unroll
                        for (uint32_t k = 0; k < LZ_SPT; k++) {
                            if (k >= R.cnt) break;
                            o += c_emit_seq(S.stage.in, S.be, S.nlong, dst, o, R.lit0[k], R.lit[k], R.off[k], R.len[k]);
                        }
                        team_sync<PB_B>();
                        const uint32_t nl = S.nlong;
                        for (uint32_t s = twid; s < nl; s += P_TEAM / 32) c_long_job(S.stage.in, S.be, dst, s, lane, 32u);
                        out_pos += total;
                        lz_next_pending(T, S.be, pd, nh, tile_end, t0);
                        team_sync<PB_B>();
                        if (ttid == 0) S.nlong = 0;
                    }
                }
                ZMT_PHASE(1, ttid, 5);
                if (ti + 2 < ntiles) { if (b) bar_arrive<PB_EMPTY0 + 1, 2 * P_TEAM>(); else bar_arrive<PB_EMPTY0, 2 * P_TEAM>(); }     // the front end may refill this buffer
                ZMT_PHASE(1, ttid, 6);
            }
            // ---- flush the pending sequence
            uint32_t anchor = 0;
            if (pd.valid) {
                anchor = pd.end;
                team_sync<PB_B>();                             // S.nlong = 0 of the last tile is visible
                if (ttid == 0) (void)c_emit_seq(S.stage.in, S.be, S.nlong, dst, out_pos, pd.lit, pd.start - pd.lit, pd.off, pd.end - pd.start);
                out_pos += c_seq_size(pd.start - pd.lit, pd.end - pd.start);
                team_sync<PB_B>();
                const uint32_t nl = S.nlong;                   // long literal run and / or long match length of the pending sequence
                for (uint32_t s = 0; s < nl; s++) c_long_job(S.stage.in, S.be, dst, s, ttid, P_TEAM);
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
                for (uint32_t i = tid; i < lit; i += NT) op[hl + i] = S.stage.in[anchor + i];
            }
        }
        ZMT_PHASE(team, ttid, 7);
    }
}
