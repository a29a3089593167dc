// zstd_entropy.cuh — CTA-wide entropy stage of the Zstandard encoder (RFC 8878 bitstreams).
//
// Replaces, for one ~16 KiB "sub-block" of sequences + literals produced by the shared LZ77 front end
// (lz4_kernels.cu), what ZSTD_compress does after match finding at the reference call site
// lib/zstd-mt_compress.c:284-286:
//   literals  : raw / RLE / Huffman (4 streams, tree described by direct 4-bit weights)
//   sequences : LL / OF / ML codes + extra bits on the PREDEFINED FSE tables (mode 0,0,0), the three state
//               chains run chunk-parallel on the 32 lanes of one warp (speculative entry states, verified),
//               every bit field is then placed in parallel from a scan of bit counts
//   block     : 3-byte header, raw fallback when nothing is gained
// Every block is self-contained (own Huffman tree, predefined sequence tables, explicit offsets: no repeat
// codes), so the decoder can give each block its own CTA.
#pragma once
#include "common.cuh"

#define Z_MAXSEQ     4352u           // sequences per sub-block (4 tiles x 1024 + pending + slack)
#define Z_MAXLIT     (64u * 1024u + 256u)   // literal bytes per block: a pending match can hold back the sub-block flushes of a whole
                                           // 64 KiB window (match, then incompressible data to the end), so the bound is the window
#define Z_BITWORDS   3072u           // shared bit buffer: 12 KiB
#define Z_HUF_MAXBITS 11
#define Z_WARM        16u             // warm-up symbols of a speculative FSE chain chunk

// litlen: literal length in bits 0-23, offset bits 16-23 in bits 24-31 (the level 6-12 class reaches 4 MiB back);
// off: offset bits 0-15.  Eight bytes, as the level-3 encoder writes them (its offsets stay below 2^16).
struct __align__(8) ZSeq { uint32_t litlen; uint16_t off; uint16_t mlen; };
__device__ __forceinline__ uint32_t zseq_ll(const ZSeq& q) { return q.litlen & 0xFFFFFFu; }
__device__ __forceinline__ uint32_t zseq_off(const ZSeq& q) { return (uint32_t)q.off | ((q.litlen >> 24) << 16); }

// per-CTA scratch in global memory (L2 resident): sequence records, literal bytes, FSE (nbBits,value) pairs
struct ZScratch {
    ZSeq     seq[Z_MAXSEQ];
    uint8_t  lit[Z_MAXLIT];
    uint32_t fse[3][Z_MAXSEQ];       // (nbBits << 16) | value, per stream LL / OF / ML
};

// entropy-stage shared memory; a union with the LZ77 tile arrays (dead between tiles: ZstdSmem)
struct ZEnt {
    uint32_t hist[256];
    uint8_t  hlen[256];
    uint16_t hcode[256];
    uint16_t order[256];
    uint32_t ncnt[512];
    uint16_t npar[512];
    uint32_t bits[Z_BITWORDS];
    uint32_t sbits[5];               // literal stream bit totals (4) + scratch
    uint32_t wcnt[16];               // symbols per weight
    uint32_t wbase[16];
    uint32_t nused, maxsym, maxcnt, maxbits, mode;
    uint32_t seqbits, fin[3];        // final FSE states
    uint8_t  wdesc[136];             // Huffman tree description when coded with FSE (header byte + <= 127 bytes)
    uint32_t wdesc_len;
    uint8_t  codes[Z_MAXSEQ];        // symbol codes of the stream the chain warp is working on, in encoding order
};

// ---- predefined-distribution FSE encoding tables (filled by the host once per device: zstd_tables_init)
struct ZFseCTable { uint16_t state[64]; int32_t dnb[64]; int32_t dfs[64]; uint32_t log; };
// shared-memory copy used by the chain lanes (lane-divergent lookups would serialise in the constant cache)
struct ZFseShared { uint16_t state[3][64]; int2 tt[3][64]; };      // tt = (deltaNbBits, deltaFindState); order LL, OF, ML
__constant__ ZFseCTable c_fse_ll, c_fse_of, c_fse_ml;
__constant__ uint8_t  c_ll_code[64], c_ml_code[128];
__constant__ uint32_t c_ll_base[36], c_ml_base[53];
__constant__ uint8_t  c_ll_bits[36], c_ml_bits[53];

__device__ __forceinline__ uint32_t z_highbit(uint32_t v) { return 31 - __clz(v); }
__device__ __forceinline__ uint32_t z_ll_code(uint32_t ll) { return ll < 64 ? c_ll_code[ll] : z_highbit(ll) + 19; }
__device__ __forceinline__ uint32_t z_ml_code(uint32_t mlb) { return mlb < 128 ? c_ml_code[mlb] : z_highbit(mlb) + 36; }

// append `nb` bits of `v` at absolute bit position `pos` of a zero-initialised shared word array
__device__ __forceinline__ void z_put_bits(uint32_t* buf, uint32_t pos, uint32_t v, uint32_t nb)
{
    if (!nb) return;
    const uint64_t x = (uint64_t)(v & (nb >= 32 ? 0xFFFFFFFFu : ((1u << nb) - 1))) << (pos & 31);
    atomicOr(&buf[pos >> 5], (uint32_t)x);
    if ((uint32_t)(x >> 32)) atomicOr(&buf[(pos >> 5) + 1], (uint32_t)(x >> 32));
}

// sequential bit appender for one thread's contiguous bit range (first/last words shared with neighbours)
struct ZBitRun {
    uint32_t* buf; uint64_t acc; uint32_t nacc, word;
    __device__ __forceinline__ void start(uint32_t* b, uint32_t pos) { buf = b; word = pos >> 5; nacc = pos & 31; acc = 0; }
    __device__ __forceinline__ void add(uint32_t v, uint32_t nb)
    {
        acc |= (uint64_t)v << nacc; nacc += nb;
        if (nacc >= 32) { atomicOr(&buf[word++], (uint32_t)acc); acc >>= 32; nacc -= 32; }
    }
    __device__ __forceinline__ void finish() { if (nacc) atomicOr(&buf[word], (uint32_t)acc); }
};

// copy `n` bytes out of a shared word buffer (byte offset 0) to global memory
__device__ __forceinline__ void z_copy_out(uint8_t* dst, const uint32_t* buf, uint32_t n, uint32_t t, uint32_t nt)
{
    const uint8_t* b = reinterpret_cast<const uint8_t*>(buf);
    for (uint32_t i = t; i < n; i += nt) dst[i] = b[i];
}

// Encode one block.  All 256 threads call it.  Returns (CTA-uniform) the bytes written at dst.
//   seqs/nseq, lits/nlit : from the scratch;  raw/regen : the block's content in shared memory (raw fallback)
__device__ __forceinline__ void z_load_fse_shared(ZFseShared& F, uint32_t tid, uint32_t nt)
{
    for (uint32_t i = tid; i < 3 * 64; i += nt) {
        const uint32_t k = i >> 6, j = i & 63;
        const ZFseCTable& T = k == 0 ? c_fse_ll : k == 1 ? c_fse_of : c_fse_ml;
        F.state[k][j] = T.state[j]; F.tt[k][j] = make_int2(T.dnb[j], T.dfs[j]);
    }
}

// FSE-compress the Huffman weights (RFC 8878 §4.2.1.2; HUF_compressWeights + FSE_writeNCount + FSE_compress_usingCTable
// [ext]) — one thread, at most 255 weights over an alphabet of <= 12 values, table log 6.  Writes header byte (= size)
// + payload into Z.wdesc, returns the total length or 0 when the weights are not compressible this way.
__device__ uint32_t z_fse_weights(ZEnt& Z, uint32_t nw /* weights listed = maxsym */, uint32_t maxbits)
{
    uint8_t* wt = reinterpret_cast<uint8_t*>(Z.ncnt);              // scratch: weights (256 B) | state table | symbol tt
    uint16_t* stab = reinterpret_cast<uint16_t*>(Z.ncnt + 64);     // 64 entries
    int32_t* dnb = reinterpret_cast<int32_t*>(Z.ncnt + 96);        // 16
    int32_t* dfs = reinterpret_cast<int32_t*>(Z.ncnt + 112);       // 16
    if (nw < 2) return 0;
    uint32_t count[13]; int norm[13];
    for (int i = 0; i < 13; i++) count[i] = 0;
    uint32_t maxw = 0;
    for (uint32_t s = 0; s < nw; s++) { const uint32_t w = Z.hlen[s] ? maxbits + 1 - Z.hlen[s] : 0; wt[s] = (uint8_t)w; count[w]++; if (w > maxw) maxw = w; }
    uint32_t maxc = 0; for (uint32_t i = 0; i <= maxw; i++) maxc = count[i] > maxc ? count[i] : maxc;
    if (maxc == nw || maxc <= 1) return 0;                          // one symbol only / nothing repeats
    // ---- normalise to 64 (every present value >= 1)
    const int LOG = 6, SIZE = 64;
    int sum = 0, big = 0;
    for (uint32_t i = 0; i <= maxw; i++) { norm[i] = count[i] ? (int)((count[i] * (uint32_t)SIZE) / nw) : 0; if (count[i] && norm[i] == 0) norm[i] = 1; sum += norm[i]; if (count[i] > count[big]) big = (int)i; }
    while (sum != SIZE) {
        if (sum < SIZE) { norm[big] += SIZE - sum; sum = SIZE; }
        else {                                                       // take from the largest entries, never below 1
            int b2 = -1; for (uint32_t i = 0; i <= maxw; i++) if (norm[i] > 1 && (b2 < 0 || norm[i] > norm[b2])) b2 = (int)i;
            if (b2 < 0) return 0;
            const int take = (norm[b2] - 1) < (sum - SIZE) ? (norm[b2] - 1) : (sum - SIZE);
            norm[b2] -= take; sum -= take;
        }
    }
    // ---- NCount header (forward bit order)
    // bits are gathered in a register and leave as whole bytes (a bit-at-a-time read-modify-write of shared memory made
    // this single-thread step the longest wait of the literal pipeline)
    uint8_t* out = Z.wdesc + 1; uint32_t bitpos = 0;
    uint64_t acc = 0; uint32_t nacc = 0; uint8_t* wp = out;
    auto put = [&](uint32_t v, uint32_t nb) { acc |= (uint64_t)(v & ((1u << nb) - 1)) << nacc; nacc += nb; bitpos += nb; while (nacc >= 8) { *wp++ = (uint8_t)acc; acc >>= 8; nacc -= 8; } };
    put((uint32_t)(LOG - 5), 4);
    {
        int remaining = SIZE + 1, threshold = SIZE, nbBits = LOG + 1; uint32_t sym = 0; bool prev0 = false;
        const uint32_t alpha = maxw + 1;
        while (sym < alpha && remaining > 1) {
            if (prev0) {
                uint32_t start = sym;
                while (sym < alpha && norm[sym] == 0) sym++;
                if (sym == alpha) break;
                while (sym >= start + 3) { start += 3; put(3, 2); }
                put(sym - start, 2);
            }
            int cnt = norm[sym++];
            const int mx = (2 * threshold - 1) - remaining;
            remaining -= cnt;
            cnt++;
            if (cnt >= threshold) cnt += mx;
            put((uint32_t)cnt, (uint32_t)nbBits - ((cnt < mx) ? 1u : 0u));
            prev0 = (cnt == 1);
            while (remaining < threshold) { nbBits--; threshold >>= 1; }
        }
        if (remaining != 1) return 0;
    }
    if (nacc) { *wp++ = (uint8_t)acc; }
    const uint32_t hdr_bytes = (bitpos + 7) >> 3;
    // ---- encoding table (FSE_buildCTable)
    {
        int cumul[14]; uint8_t tsym[64]; int pos = 0; const int step = (SIZE >> 1) + (SIZE >> 3) + 3;
        cumul[0] = 0; for (uint32_t u = 1; u <= maxw + 1; u++) cumul[u] = cumul[u - 1] + norm[u - 1];
        for (uint32_t sy = 0; sy <= maxw; sy++) for (int i = 0; i < norm[sy]; i++) { tsym[pos] = (uint8_t)sy; pos = (pos + step) & (SIZE - 1); }
        for (int u = 0; u < SIZE; u++) { const int sy = tsym[u]; stab[cumul[sy]++] = (uint16_t)(SIZE + u); }
        int total = 0;
        for (uint32_t sy = 0; sy <= maxw; sy++) {
            const int n = norm[sy];
            if (n == 0) { dnb[sy] = ((LOG + 1) << 16) - SIZE; dfs[sy] = 0; }
            else if (n == 1) { dnb[sy] = (LOG << 16) - SIZE; dfs[sy] = total - 1; total++; }
            else { const int hb = 31 - __clz((uint32_t)(n - 1)); const int mbo = LOG - hb; dnb[sy] = (mbo << 16) - (n << mbo); dfs[sy] = total - n; total += n; }
        }
    }
    // ---- two interleaved states, last weight first (FSE_compress_usingCTable_generic)
    if (hdr_bytes >= 100) return 0;
    uint8_t* bs = out + hdr_bytes; uint32_t bpos = 0;
    const uint32_t bcap = (127 - hdr_bytes) * 8;                     // the FSE form must fit 127 bytes (header byte < 128)
    bool over = false;
    acc = 0; nacc = 0; wp = bs;
    auto putb = [&](uint32_t v, uint32_t nb) {
        if (bpos + nb > bcap) { over = true; return; }
        acc |= (uint64_t)(v & ((1u << nb) - 1)) << nacc; nacc += nb; bpos += nb;
        while (nacc >= 8) { *wp++ = (uint8_t)acc; acc >>= 8; nacc -= 8; }
    };
    auto init = [&](uint32_t sy) -> uint32_t { const uint32_t nbo = (uint32_t)(dnb[sy] + (1 << 15)) >> 16; return stab[(((nbo << 16) - (uint32_t)dnb[sy]) >> nbo) + dfs[sy]]; };
    auto enc = [&](uint32_t& st, uint32_t sy) { const uint32_t nbo = (st + (uint32_t)dnb[sy]) >> 16; putb(st & ((1u << nbo) - 1), nbo); st = stab[(st >> nbo) + dfs[sy]]; };
    int ip = (int)nw; uint32_t s1, s2;
    if (nw & 1) { s1 = init(wt[--ip]); s2 = init(wt[--ip]); enc(s1, wt[--ip]); }
    else { s2 = init(wt[--ip]); s1 = init(wt[--ip]); }
    while (ip > 0) { enc(s2, wt[--ip]); enc(s1, wt[--ip]); }
    putb(s2, (uint32_t)LOG); putb(s1, (uint32_t)LOG);
    putb(1, 1);
    if (nacc) *wp++ = (uint8_t)acc;
    const uint32_t total_bytes = hdr_bytes + ((bpos + 7) >> 3);
    if (over || total_bytes >= 128) return 0;
    Z.wdesc[0] = (uint8_t)total_bytes;
    return 1 + total_bytes;
}

// named barrier for the 7 literal warps (224 threads); barrier 0 stays the CTA-wide one
__device__ __forceinline__ void z_lit_sync() { __syncwarp(); asm volatile("bar.sync 1, 224;" ::: "memory"); }

// exclusive scan over the 224 literal threads (7 warps); `ws` >= 9 words, double use protected by the leading barrier
__device__ __forceinline__ uint32_t z_lit_exscan(uint32_t v, uint32_t* ws, uint32_t* total)
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(ZMT_FULL_MASK, inc, d); if (lane >= (uint32_t)d) inc += y; }
    z_lit_sync();
    if (lane == 31) ws[wid] = inc;
    z_lit_sync();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (uint32_t w = 0; w < 7; w++) { const uint32_t x = ws[w]; if (w < wid) base += x; tot += x; }
    *total = tot;
    return base + inc - v;
}

// Encode one block.  All 256 threads call it.  Returns (CTA-uniform) the bytes written at dst.
//   seqs/nseq, lits/nlit : from the scratch;  raw/regen : the block's content in shared memory (raw fallback)
// Warp 7 runs the three serial FSE state chains while warps 0..6 do the whole literal pipeline (histogram, Huffman
// tree, canonical codes, 4 bit streams, literal section written to dst) behind their own named barrier.
template <class SYNC>
__device__ uint32_t z_encode_block(ZEnt& Z, const ZFseShared& F, ZScratch* zs, uint32_t nseq, uint32_t nlit, const uint8_t* raw, uint32_t regen,
                                   bool last, uint8_t* dst, uint32_t* scanws, SYNC cta_sync)
{
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, NT = blockDim.x;
    const uint8_t* lits = zs->lit;
    uint8_t* const p = dst + 3;                              // literals section starts right after the block header

    Z.hist[tid] = 0;
    if (tid < 16) { Z.wcnt[tid] = 0; }
    if (tid == 0) { Z.nused = 0; Z.maxsym = 0; Z.maxcnt = 0; Z.maxbits = 0; Z.mode = 0; Z.seqbits = 0; }
    for (uint32_t i = tid; i < Z_BITWORDS; i += NT) Z.bits[i] = 0;
    cta_sync();

    if (wid == 7) {
        // ------------------------------------------------------------ FSE state chains
        // Encoding order is last sequence first (RFC 8878 §3.1.1.3.2.1.1: the decoder reads backwards); step t encodes
        // sequence nseq-1-t.  A chain is serial in its state, but FSE states re-synchronise quickly: the state after a
        // symbol lies in that symbol's sub-range of the table (one value for the many symbols of probability 1/64),
        // whatever the state before.  So the 32 lanes each take a contiguous chunk of steps: a lane warms up over
        // the Z_WARM steps before its chunk from an arbitrary valid state (exact when the warm-up reaches step 0),
        // runs its chunk, and the warp then checks every chunk's entry state against its predecessor's exit state and
        // re-runs the (rare) chunks that guessed wrong until nothing changes.  Same bits as the serial chain,
        // ~nseq/32 + Z_WARM serial steps per stream instead of nseq.  One stream at a time: the symbol codes of the
        // current stream sit in shared memory (Z.codes), the (nbBits, value) pairs go to the scratch as before.
        if (nseq) {
            const uint32_t c = (nseq + 31) / 32;
            const uint32_t t_begin = lane * c, t_end = t_begin + c < nseq ? t_begin + c : nseq;
            const bool have = t_begin < nseq;
            const uint32_t w0 = t_begin > Z_WARM ? t_begin - Z_WARM : 0;
            for (uint32_t kk = 0; kk < 3; kk++) {
                __syncwarp();
                for (uint32_t idx = lane; idx < nseq; idx += 32) {
                    const ZSeq q = zs->seq[idx];
                    const uint32_t code = kk == 0 ? z_ll_code(zseq_ll(q)) : kk == 1 ? z_highbit(zseq_off(q) + 3u) : z_ml_code((uint32_t)q.mlen - 3u);
                    Z.codes[nseq - 1 - idx] = (uint8_t)code;
                }
                __syncwarp();
                const int2* const TT = F.tt[kk];
                const uint16_t* const ST = F.state[kk];
                // FSE_initCState2: the state "after" a first symbol, no bits
                auto init_state = [&](int2 tt) -> uint32_t { const uint32_t nbo = (uint32_t)(tt.x + (1 << 15)) >> 16; return ST[(((nbo << 16) - (uint32_t)tt.x) >> nbo) + tt.y]; };
                uint32_t sin = 0;
                if (have) {
                    sin = init_state(TT[Z.codes[w0]]);
                    for (uint32_t t = w0 + 1; t < t_begin; t++) { const int2 tt = TT[Z.codes[t]]; const uint32_t nbo = (sin + (uint32_t)tt.x) >> 16; sin = ST[(sin >> nbo) + tt.y]; }
                }
                auto run_chunk = [&](uint32_t st) -> uint32_t {
#pragma unroll 4
                    for (uint32_t t = t_begin; t < t_end; t++) {
                        const int2 tt = TT[Z.codes[t]];
                        uint32_t outv = 0;
                        if (t == 0) st = init_state(tt);
                        else { const uint32_t nbo = (st + (uint32_t)tt.x) >> 16; outv = (nbo << 16) | (st & ((1u << nbo) - 1)); st = ST[(st >> nbo) + tt.y]; }
                        zs->fse[kk][nseq - 1 - t] = outv;
                    }
                    return st;
                };
                uint32_t sout = have ? run_chunk(sin) : 0;
                for (;;) {                                   // repair chunks whose speculative entry state was wrong
                    const uint32_t prev = __shfl_up_sync(ZMT_FULL_MASK, sout, 1);
                    const bool bad = have && lane > 0 && prev != sin;
                    if (!__any_sync(ZMT_FULL_MASK, bad)) break;
                    if (bad) { sin = prev; sout = run_chunk(sin); }
                    __syncwarp();
                }
                const uint32_t fin = __shfl_sync(ZMT_FULL_MASK, sout, (nseq - 1) / c);
                if (lane == 0) Z.fin[kk] = fin;
            }
        }
    } else {
        // ------------------------------------------------------------ literal pipeline (224 threads)
        const uint32_t LT = 224;
        for (uint32_t i = tid; i < nlit; i += LT) atomicAdd(&Z.hist[lits[i]], 1u);
        z_lit_sync();
        for (uint32_t s = tid; s < 256; s += LT) {
            const uint32_t c = Z.hist[s];
            Z.hlen[s] = 0;
            if (c) { atomicAdd(&Z.nused, 1u); atomicMax(&Z.maxsym, s); atomicMax(&Z.maxcnt, c); }
        }
        z_lit_sync();
        const uint32_t nused = Z.nused, maxsym = Z.maxsym;
        uint32_t lmode = 0;                                  // 0 raw, 1 RLE, 2 Huffman (direct-weight trees only: symbols 0..128)
        if (nlit && Z.maxcnt == nlit) lmode = 1;
        else if (nlit >= 64 && nused >= 2) lmode = 2;
        uint32_t tree_bytes = 0, lit_payload = 0, sbytes[4] = {0, 0, 0, 0}, swords[4] = {0, 0, 0, 0};
        if (lmode == 2) {
            // order[]: present symbols by ascending (count, symbol)
            for (uint32_t s = tid; s < 256; s += LT) {
                const uint32_t c = Z.hist[s];
                if (c) {
                    uint32_t r = 0;
                    for (uint32_t t = 0; t < 256; t++) { const uint32_t ct = Z.hist[t]; r += (ct && (ct < c || (ct == c && t < s))) ? 1u : 0u; }
                    Z.order[r] = (uint16_t)s;
                }
            }
            z_lit_sync();
            if (tid == 0) {
                // two-queue Huffman: leaves 0..nused-1 (ascending), internal nodes nused..2*nused-2
                for (uint32_t i = 0; i < nused; i++) Z.ncnt[i] = Z.hist[Z.order[i]];
                uint32_t li = 0, ii = nused, ni = nused;
                for (uint32_t k = 0; k + 1 < nused; k++) {
                    uint32_t a, b;
                    if (li < nused && (ii >= ni || Z.ncnt[li] <= Z.ncnt[ii])) a = li++; else a = ii++;
                    if (li < nused && (ii >= ni || Z.ncnt[li] <= Z.ncnt[ii])) b = li++; else b = ii++;
                    Z.ncnt[ni] = Z.ncnt[a] + Z.ncnt[b]; Z.npar[a] = (uint16_t)ni; Z.npar[b] = (uint16_t)ni; ni++;
                }
                const uint32_t root = ni - 1;
                Z.ncnt[root] = 0;                            // reuse ncnt[] as depth (parents have larger indices)
                for (int v = (int)root - 1; v >= 0; v--) Z.ncnt[v] = Z.ncnt[Z.npar[v]] + 1;
                uint32_t maxl = 0;
                for (uint32_t i = 0; i < nused; i++) maxl = maxl > Z.ncnt[i] ? maxl : Z.ncnt[i];
                if (maxl > Z_HUF_MAXBITS) {
                    // length-limit: clamp to 11, repay the Kraft excess by lengthening the longest shorter codes
                    // (leaf 0 = rarest = longest code), then hand back any overshoot by shortening 11-bit codes
                    int32_t excess = 0;                      // in units of 2^-11
                    for (uint32_t i = 0; i < nused; i++) { if (Z.ncnt[i] > Z_HUF_MAXBITS) Z.ncnt[i] = Z_HUF_MAXBITS; excess += 1 << (Z_HUF_MAXBITS - Z.ncnt[i]); }
                    excess -= 1 << Z_HUF_MAXBITS;
                    while (excess > 0) {
                        int best = -1;
                        for (uint32_t i = 0; i < nused; i++)
                            if (Z.ncnt[i] < Z_HUF_MAXBITS) { if (best < 0) best = (int)i; if ((1 << (Z_HUF_MAXBITS - 1 - Z.ncnt[i])) <= excess) { best = (int)i; break; } }
                        if (best < 0) break;
                        excess -= 1 << (Z_HUF_MAXBITS - 1 - Z.ncnt[best]);
                        Z.ncnt[best]++;
                    }
                    for (uint32_t i = 0; i < nused && excess < 0; i++)
                        if (Z.ncnt[i] == Z_HUF_MAXBITS) { Z.ncnt[i]--; excess++; }
                    maxl = Z_HUF_MAXBITS;
                }
                Z.maxbits = maxl;
                for (uint32_t i = 0; i < nused; i++) Z.hlen[Z.order[i]] = (uint8_t)Z.ncnt[i];
            }
            z_lit_sync();
            const uint32_t maxbits = Z.maxbits;
            // canonical codes in the decoder's table order: ascending weight, then symbol
            for (uint32_t s = tid; s < 256; s += LT) { const uint32_t l = Z.hlen[s]; if (l) atomicAdd(&Z.wcnt[maxbits + 1 - l], 1u); }
            z_lit_sync();
            if (tid == 0) { uint32_t acc = 0; for (uint32_t w = 1; w <= maxbits; w++) { Z.wbase[w] = acc; acc += Z.wcnt[w] << (w - 1); } }
            z_lit_sync();
            uint32_t mybitsum = 0;
            for (uint32_t s = tid; s < 256; s += LT) {
                const uint32_t l = Z.hlen[s];
                if (l) {
                    const uint32_t w = maxbits + 1 - l;
                    uint32_t r = 0;
                    for (uint32_t t = 0; t < s; t++) r += (Z.hlen[t] == l) ? 1u : 0u;
                    Z.hcode[s] = (uint16_t)((Z.wbase[w] + (r << (w - 1))) >> (w - 1));
                    mybitsum += Z.hist[s] * l;
                }
            }
            uint32_t totbits;
            (void)z_lit_exscan(mybitsum, scanws, &totbits);
            // tree description: FSE-coded weights when smaller (or when direct 4-bit weights cannot express symbols > 128)
            if (tid == 0) {
                const uint32_t direct = maxsym <= 128 ? 1 + (maxsym + 1) / 2 : 0xFFFFu;
                // The FSE form is built only where it is mandatory (a symbol above 128).  Where the direct form exists it costs
                // <= 65 bytes per block, the FSE form would save ~30 of them (0.4 % of the output on text) — and this single-thread
                // step is a serial wait for the whole CTA.
                const uint32_t fl = direct == 0xFFFFu ? z_fse_weights(Z, maxsym, maxbits) : 0u;
                Z.wdesc_len = (fl && fl < direct) ? fl : (direct != 0xFFFFu ? 0u : 0xFFFFu);       // 0: direct form, 0xFFFF: no valid form
            }
            z_lit_sync();
            const uint32_t wl = Z.wdesc_len;
            tree_bytes = wl == 0 ? 1 + (maxsym + 1) / 2 : wl;
            const uint32_t est = (totbits + 7) / 8 + 4 + tree_bytes + 6;
            if (wl == 0xFFFFu || est >= nlit || est + 64 > Z_BITWORDS * 4) lmode = 0;       // Huffman does not pay (or would not fit the bit buffer)
        }
        uint32_t lit_hdr, lit_body;
        if (lmode == 2) {
            // 4 streams x 56 threads, contiguous runs, reverse bit order
            const uint32_t per = (nlit + 3) / 4;
            const uint32_t k = tid / 56, u = tid % 56;
            const uint32_t s0 = k * per, s1 = (s0 + per < nlit) ? s0 + per : nlit;
            const uint32_t cnt = s1 > s0 ? s1 - s0 : 0, g = (cnt + 55) / 56;
            const uint32_t a = s0 + u * g < s1 ? s0 + u * g : s1, b = a + g < s1 ? a + g : s1;
            uint32_t mybits = 0;
            for (uint32_t i = a; i < b; i++) mybits += Z.hlen[lits[i]];
            uint32_t tot;
            const uint32_t pre = z_lit_exscan(mybits, scanws, &tot);
            if (u == 0) Z.sbits[k] = pre;
            if (tid == 0) Z.sbits[4] = tot;
            z_lit_sync();
            const uint32_t base_k = Z.sbits[k], end_k = k == 3 ? Z.sbits[4] : Z.sbits[k + 1];
            uint32_t woff = 0;
            for (uint32_t q = 0; q < 4; q++) {
                const uint32_t tq = (q == 3 ? Z.sbits[4] : Z.sbits[q + 1]) - Z.sbits[q];
                sbytes[q] = tq / 8 + 1; swords[q] = (tq + 32) / 32;
                if (q < k) woff += swords[q];
            }
            const uint32_t pos_lo = end_k - (pre + mybits);      // my run sits after everything that FOLLOWS it in the stream
            ZBitRun R; R.start(Z.bits + woff, pos_lo);
            for (uint32_t i = b; i > a; i--) { const uint32_t sy = lits[i - 1]; R.add(Z.hcode[sy], Z.hlen[sy]); }
            R.finish();
            if (u == 0) z_put_bits(Z.bits + woff, end_k - base_k, 1, 1);     // end marker above the last symbol's code
            lit_payload = sbytes[0] + sbytes[1] + sbytes[2] + sbytes[3];
            lit_body = tree_bytes + 6 + lit_payload;
            lit_hdr = (nlit < 1024 && lit_body < 1024) ? 3 : (nlit < 16384 && lit_body < 16384) ? 4 : 5;
            z_lit_sync();
            if (tid == 0) {
                const uint32_t fmt = lit_hdr == 3 ? 1u : lit_hdr == 4 ? 2u : 3u;
                const uint32_t nb = lit_hdr == 3 ? 10u : lit_hdr == 4 ? 14u : 18u;
                const uint64_t v = 2ull | ((uint64_t)fmt << 2) | ((uint64_t)nlit << 4) | ((uint64_t)lit_body << (4 + nb));
                for (uint32_t i = 0; i < lit_hdr; i++) p[i] = (uint8_t)(v >> (8 * i));
                uint8_t* q = p + lit_hdr;
                if (Z.wdesc_len) { for (uint32_t i = 0; i < Z.wdesc_len; i++) *q++ = Z.wdesc[i]; }       // FSE-coded weights
                else {
                    *q++ = (uint8_t)(127 + maxsym);         // direct weights for symbols 0 .. maxsym-1 (the last one is implied)
                    for (uint32_t s = 0; s < maxsym; s += 2) {
                        const uint32_t w0 = Z.hlen[s] ? Z.maxbits + 1 - Z.hlen[s] : 0;
                        const uint32_t w1 = (s + 1 < maxsym && Z.hlen[s + 1]) ? Z.maxbits + 1 - Z.hlen[s + 1] : 0;
                        *q++ = (uint8_t)((w0 << 4) | w1);
                    }
                }
                q[0] = (uint8_t)sbytes[0]; q[1] = (uint8_t)(sbytes[0] >> 8); q[2] = (uint8_t)sbytes[1]; q[3] = (uint8_t)(sbytes[1] >> 8);
                q[4] = (uint8_t)sbytes[2]; q[5] = (uint8_t)(sbytes[2] >> 8);
            }
            uint8_t* q = p + lit_hdr + tree_bytes + 6;
            uint32_t wo = 0;
            for (uint32_t kq = 0; kq < 4; kq++) { z_copy_out(q, Z.bits + wo, sbytes[kq], tid, LT); q += sbytes[kq]; wo += swords[kq]; }
        } else {
            lit_body = lmode == 1 ? 1 : nlit;
            lit_hdr = nlit < 32 ? 1 : nlit < 4096 ? 2 : 3;
            if (tid == 0) {
                const uint32_t type = lmode;                  // 0 raw, 1 RLE
                if (lit_hdr == 1) p[0] = (uint8_t)(type | (nlit << 3));
                else if (lit_hdr == 2) { const uint32_t v = type | (1u << 2) | (nlit << 4); p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
                else { const uint32_t v = type | (3u << 2) | (nlit << 4); p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); }
                if (lmode == 1) p[lit_hdr] = lits[0];
            }
            if (lmode == 0) for (uint32_t i = tid; i < nlit; i += LT) p[lit_hdr + i] = lits[i];
        }
        if (tid == 0) Z.seqbits = lit_hdr + lit_body;            // literals section size, for everyone after the join
    }
    cta_sync();
    const uint32_t lit_total = Z.seqbits;

    // ------------------------------------------------------------ sequences: bit counts in encoding order (index j = nseq-1-i)
    for (uint32_t i = tid; i < Z_BITWORDS; i += NT) Z.bits[i] = 0;
    uint32_t seq_bits = 0, seq_pre = 0, my_cnt = 0, my_first = 0;
    if (nseq) {
        const uint32_t g = (nseq + NT - 1) / NT;
        my_first = tid * g < nseq ? tid * g : nseq;
        const uint32_t my_end = my_first + g < nseq ? my_first + g : nseq;
        my_cnt = my_end - my_first;
        uint32_t b = 0;
        for (uint32_t j = my_first; j < my_end; j++) {
            const uint32_t i = nseq - 1 - j;
            const ZSeq q = zs->seq[i];
            const uint32_t llc = z_ll_code(zseq_ll(q)), mlc = z_ml_code((uint32_t)q.mlen - 3u), ofc = z_highbit(zseq_off(q) + 3u);
            b += c_ll_bits[llc] + c_ml_bits[mlc] + ofc;
            b += (zs->fse[0][i] >> 16) + (zs->fse[1][i] >> 16) + (zs->fse[2][i] >> 16);
        }
        seq_pre = block_exscan(b, scanws, &seq_bits);
        seq_bits += c_fse_ml.log + c_fse_of.log + c_fse_ll.log;          // final state flush
    }
    const uint32_t seq_hdr = nseq == 0 ? 1 : (nseq < 128 ? 2 : 3);        // nbSeq bytes (+ modes byte when nseq > 0)
    const uint32_t seq_body = nseq ? seq_bits / 8 + 1 : 0;
    const uint32_t bsize = lit_total + seq_hdr + seq_body;
    const bool use_raw = bsize >= regen || (seq_body + 8 > Z_BITWORDS * 4) || nseq >= 0x7F00;
    cta_sync();

    // ------------------------------------------------------------ write
    if (use_raw) {
        if (tid == 0) { const uint32_t h = (regen << 3) | (last ? 1u : 0u); dst[0] = (uint8_t)h; dst[1] = (uint8_t)(h >> 8); dst[2] = (uint8_t)(h >> 16); }
        for (uint32_t i = tid; i < regen; i += NT) dst[3 + i] = raw[i];
        cta_sync();
        return 3 + regen;
    }
    if (tid == 0) {
        const uint32_t h = (bsize << 3) | (2u << 1) | (last ? 1u : 0u);
        dst[0] = (uint8_t)h; dst[1] = (uint8_t)(h >> 8); dst[2] = (uint8_t)(h >> 16);
        uint8_t* s = p + lit_total;                            // sequences section header
        if (nseq == 0) s[0] = 0;
        else if (nseq < 128) { s[0] = (uint8_t)nseq; s[1] = 0; }
        else { s[0] = (uint8_t)((nseq >> 8) + 128); s[1] = (uint8_t)nseq; s[2] = 0; }
    }
    if (nseq) {
        ZBitRun R; R.start(Z.bits, seq_pre);
        for (uint32_t j = my_first; j < my_first + my_cnt; j++) {
            const uint32_t i = nseq - 1 - j;
            const ZSeq q = zs->seq[i];
            const uint32_t ll = zseq_ll(q), llc = z_ll_code(ll), mlc = z_ml_code((uint32_t)q.mlen - 3u), ofv = zseq_off(q) + 3u, ofc = z_highbit(ofv);
            const uint32_t fl = zs->fse[0][i], fo = zs->fse[1][i], fm = zs->fse[2][i];
            // per sequence (zstd_compress_sequences.c order): FSE OF, ML, LL state bits, then extra bits LL, ML, OF
            R.add(fo & 0xFFFF, fo >> 16); R.add(fm & 0xFFFF, fm >> 16); R.add(fl & 0xFFFF, fl >> 16);
            R.add(ll - c_ll_base[llc], c_ll_bits[llc]);
            R.add((uint32_t)q.mlen - c_ml_base[mlc], c_ml_bits[mlc]);
            R.add(ofv - (1u << ofc), ofc);
        }
        R.finish();
        if (tid == 0) {
            uint32_t pos = seq_bits - (c_fse_ml.log + c_fse_of.log + c_fse_ll.log);
            z_put_bits(Z.bits, pos, Z.fin[2], c_fse_ml.log); pos += c_fse_ml.log;      // flush ML, OF, LL (decoder reads LL, OF, ML)
            z_put_bits(Z.bits, pos, Z.fin[1], c_fse_of.log); pos += c_fse_of.log;
            z_put_bits(Z.bits, pos, Z.fin[0], c_fse_ll.log); pos += c_fse_ll.log;
            z_put_bits(Z.bits, pos, 1, 1);
        }
        cta_sync();
        z_copy_out(p + lit_total + seq_hdr, Z.bits, seq_body, tid, NT);
    }
    cta_sync();
    return 3 + bsize;
}
