"""The GPU schedule of the LZ4 level-1 block compressor (lz4_blocks_pipe_kernel) restated in plain Python and numpy.

The zstd level-3 encoder (zstd_blocks_kernel) runs the same phase functions of lz4_pipe.cuh with one team, so its
parse is this one too.  Per 64 KiB block:
  candidate rounds  lz_candidates: rounds of 1024 positions, four per thread (a quad), the 12-bit table as it stood
                    before the round, short periods d = 1..4 before the table, the MFLIMIT mask, and the inserts
                    (atomicMax; an insert is skipped when a later eligible position of its quad has the same hash);
  front end / tile  c_walk MODE 0 (own segment: V bits, len4, exit state) and MODE 1 (continuation: link, mpos,
                    len4 ORs), the in-warp pointer doubling (5 rounds), the warp-to-warp hops, min_, pathmask, k0 and
                    do_parse, from the entry (e, e_din) carried between tiles (lz_chains);
  back end / tile   c_walk MODE 2 (Sel, Cont, clen, the one-step shortcut over the own segment's V bits), the piece
                    list and segprev, head detection, lz_seq_run / lz_next_pending with c_seq_size and c_emit_seq (the
                    long jobs per tile), the flush of the pending sequence and the last literals (lz_heads & co.).

`lz4_block` returns the block's LZ4 bytes as the kernel writes them (None when the block is stored raw), its
sequences (literal length, offset, match length) and named events (a dict name -> list of details), and asserts on
every tile the invariants the kernel relies on (see `Invariant`).  `mutant` swaps in a wrong rule, so that a test can
show the corpus notices it (MUTANTS)."""
from collections import defaultdict

import numpy as np

BLK = 65536
C_TILE, C_SEG, C_ROUND, C_HASHLOG = 4096, 16, 1024, 12
C_CHAINS = C_TILE // C_SEG
C_MAXPIECE, C_LONGLIT = 1280, 32
P_TEAM = 256
LZ_SPT = 1024 // P_TEAM
LONGL_WORDS = 2 * (C_TILE // (C_LONGLIT + 1) + 2)   # LzBack::longl: two words per job
LONG_ML_RUNS = 4                                     # c_emit_seq: a match length with more 255 bytes than this is a job
END = 0xFFFF
MUTANTS = ("own_from_segment_start",   # MODE 2 takes the own segment's V bits from the segment start, not the entry
           "head_prev_piece_offset")   # head detection takes a Cont piece's own T.off instead of the segprev lookup


class Invariant(AssertionError):
    """A property the kernel relies on does not hold on this tile."""


def need(cond, what, *detail):
    if not cond:
        raise Invariant(what, *detail)


def _words(s, n):
    """v(i): the little-endian 32-bit window at every position i in [-4, n) (zeros below the block and past it), as an
    int64 array indexed by i + 4."""
    b = np.zeros(n + 12, np.int64)
    b[4: 4 + n] = np.frombuffer(bytes(s[:n]), np.uint8)
    return b[0: n + 4] | (b[1: n + 5] << 8) | (b[2: n + 6] << 16) | (b[3: n + 7] << 24)


def _hash(v):
    return ((v * 2654435761) & 0xFFFFFFFF) >> (32 - C_HASHLOG)


# ------------------------------------------------------------------------------------------------- candidate rounds
def candidates(s, n, ev=None, base=0):
    """off[i] for every position of the block (0 = no candidate), round by round as lz_candidates computes it."""
    ev = defaultdict(list) if ev is None else ev
    w = _words(s, n)
    v = w[4:]
    h = _hash(v)
    tab = np.zeros(1 << C_HASHLOG, np.int64)
    off = np.zeros(n, np.int64)
    for r0 in range(0, n, C_ROUND):
        r1 = min(r0 + C_ROUND, n)
        i = np.arange(r0, r1)
        vi, hi = v[r0:r1], h[r0:r1]
        elig = i + 12 <= n
        t = tab[hi]
        hit = (t != 0) & (v[np.maximum(t - 1, 0)] == vi)
        of = np.where(hit, i - (t - 1), 0)
        loc = np.zeros(i.size, np.int64)
        for d in (4, 3, 2, 1):                                   # the smallest d wins
            loc = np.where((i >= d) & (w[i + 4 - d] == vi), d, loc)
        of = np.where(loc != 0, loc, of)
        off[r0:r1] = np.where(elig, of, 0)
        # events of the round
        for q in np.flatnonzero(elig & (loc != 0) & hit & (i - (t - 1) != loc)).tolist():
            ev["period_beats_table"].append(base + r0 + q)
        ev["collision_verify_fails"] += (base + r0 + np.flatnonzero(elig & (t != 0) & ~hit & (loc == 0))).tolist()
        if r0 == 0:
            for k in range(min(4, n)):
                if k + 12 <= n and any(w[k + 4 - d] == v[k] for d in range(k + 1, 5)):
                    ev["first_quad_d_gt_k"].append((k, int(off[k])))
        order = np.argsort(vi, kind="stable")
        sv = vi[order]
        seen = np.zeros(i.size, bool)
        seen[order[1:]] = sv[1:] == sv[:-1]                      # an earlier position of this round has the same window
        rep = np.flatnonzero(elig & seen & (off[r0:r1] == 0))
        ev["repeat_in_round_no_candidate"] += (base + r0 + rep).tolist()
        # inserts, quad by quad
        val = np.where(elig, i + 1, 0)
        nq = -(-i.size // 4)
        hq = np.full(4 * nq, -1, np.int64); hq[: i.size] = hi
        eq = np.zeros(4 * nq, bool); eq[: i.size] = elig
        hq, eq = hq.reshape(nq, 4), eq.reshape(nq, 4)
        keep = eq.copy()
        for k in range(4):
            for k2 in range(k + 1, 4):
                same = hq[:, k] == hq[:, k2]
                skip = same & eq[:, k] & eq[:, k2]
                keep[:, k] &= ~skip
                for q in np.flatnonzero(skip).tolist():
                    ev["insert_skipped_same_hash"].append((base + r0 + 4 * q + k, k2 - k))
                for q in np.flatnonzero(same & eq[:, k] & ~eq[:, k2]).tolist():
                    ev["insert_stands_later_past_mflimit"].append(base + r0 + 4 * q + k)
        keep = keep.reshape(-1)[: i.size]
        ref = tab.copy()
        np.maximum.at(tab, hi[keep], val[keep])
        np.maximum.at(ref, hi[elig], val[elig])
        need(np.array_equal(tab, ref), "a skipped insert changed the table", r0)
    return off


# ------------------------------------------------------------------------------------------------- one tile
class Tile:
    """What the front end hands the back end (PipeTile) plus the front end's own per-chain state (LzFront)."""

    def __init__(self, s, off, t0, limit):
        self.s, self.t0, self.t1, self.limit = s, t0, t0 + C_TILE, limit
        self.off = [int(x) for x in off[t0: t0 + C_TILE]] + [0] * max(0, C_TILE - (len(off) - t0))
        self.M = [x != 0 for x in self.off]
        self.V = [0] * C_CHAINS
        self.len4 = [0] * C_TILE
        self.len4_src = {}                       # position -> (first writer mode, value), for the one-value invariant
        self.w1_writers = defaultdict(int)       # position -> MODE 1 writers
        self.xfree = [0] * C_CHAINS
        self.xdin = [0] * C_CHAINS
        self.link = [0] * C_CHAINS
        self.mpos = [0] * C_CHAINS
        self.min_ = [0] * C_CHAINS
        self.pathmask = [0] * 8
        self.w0 = {}                             # chain -> (start p, start din, pieces, exit p, exit din) of walk 0
        self.why = {}                            # chain -> how its continuation ended (walk 1)

    def extend(self, p, d, cap):
        """c_extend: bytes (<= cap) for which s[p + i] == s[p + i - d]."""
        s, L = self.s, 0
        while L < cap and s[p + L] == s[p + L - d]:
            L += 1
        return L

    def nib(self, qr, L, mode):
        v = L - 4
        need(0 <= v <= 15, "candidate piece longer than 19", qr, L)
        if qr in self.len4_src:
            need(self.len4_src[qr][1] == v, "two writers of one len4 nibble disagree", qr, self.len4_src[qr], (mode, v))
        else:
            self.len4_src[qr] = (mode, v)
        if mode == 1:
            self.w1_writers[qr] += 1
            self.len4[qr] |= v
        else:
            self.len4[qr] = v


def c_walk(T, mode, k, p, din, ev, back=None, mutant=None, dry=False):
    """One chain walk.  MODE 0 / 1 write the tile's state (V, len4, xfree / xdin, link / mpos); MODE 2 marks into
    `back` (Sel, Cont, clen).  dry: a MODE 0 walk that writes nothing (the entry invariant re-walks from the entry).
    Returns (link, mpos, din, pieces) with pieces [(tile position, length, Cont)]."""
    t0, t1, limit = T.t0, T.t1, T.limit
    lk, mp, pieces, why = None, 0, [], None
    while True:
        if p >= t1:
            lk, mp, why = END, p, "leave_in_match" if din else "leave_free"
            break
        rel = p - t0
        j = rel // C_SEG
        if mode == 0 and j != k:
            mp = p
            break
        if din:
            if mode != 0 and j != k and T.M[rel] and T.off[rel] == din:
                lk, mp, why = j, p, "merge_same_match"           # chain j's own first step is this very match
                break
            if mode == 1 and j != k and T.M[rel]:
                ev["w1_boundary_other_offset"].append(t0 + rel)
            cap = min(limit - p if p < limit else 0, C_SEG)
            E = T.extend(p, din, cap)
            if mode == 2:
                if E:
                    back.mark(rel, True, E)
                    pieces.append((rel, E, True))
                else:
                    ev["match_ends_on_boundary"].append(t0 + rel)
            p += E
            if E != C_SEG:
                din = 0
            continue
        if mode == 2 and j == k:
            s0 = rel & ~(C_SEG - 1)
            own = T.V[k] & ((0xFFFF << (rel & 15)) & 0xFFFF)
            if mutant == "own_from_segment_start":
                own = T.V[k]
            p = t0 + s0 + C_SEG
            if own:
                for b in range(16):
                    if own >> b & 1:
                        back.mark(s0 + b, False)
                        pieces.append((s0 + b, 4 + T.len4[s0 + b], False))
                qr = s0 + own.bit_length() - 1
                q = t0 + qr
                B = t0 + s0 + C_SEG
                if B - q < 4:
                    B += C_SEG
                e = q + 4 + T.len4[qr]
                if e == B:
                    din = T.off[qr]
                if e > p:
                    p = e
            continue
        if mode != 0 and j != k and (rel & (C_SEG - 1)) == 0:
            lk, mp, why = j, p, "merge_free_start"               # free at a segment start
            break
        s0 = rel & ~15
        q_rel = next((x for x in range(rel, s0 + 16) if T.M[x]), None)
        if q_rel is None:                                        # segment exhausted: free at its end
            nx = t0 + (j + 1) * C_SEG
            if mode == 0:
                mp = nx
            elif j + 1 == C_CHAINS:
                lk, mp, why = END, t1, "last_segment_exhausted"
            else:
                lk, mp, why = j + 1, nx, "segment_exhausted"
            break
        qr = q_rel
        q = t0 + qr
        if mode != 0 and j != k and (T.V[j] >> (qr & 15)) & 1:
            lk, mp, why = j, q, "merge_v_bit"
            break
        d = T.off[qr]
        B = (q & ~(C_SEG - 1)) + C_SEG
        if B - q < 4:
            B += C_SEG
        if mode == 2:
            need(qr in T.len4_src, "the marking walk reads a len4 nibble no walk wrote", t0 + qr)
            L = 4 + T.len4[qr]
            back.mark(qr, False)
        else:
            end = min(B, limit)
            need(q + 4 <= limit, "a candidate starts past limit - 4", q)
            L = 4 + T.extend(q + 4, d, end - (q + 4))
            if mode == 1:
                T.nib(qr, L, mode)
        pieces.append((qr, L, False))
        p = q + L
        if p == B:
            din = d
    if mode == 1:
        T.why[k] = why
        ev["w1_" + why].append(mp)
    return lk, mp, din, pieces


def front_tile(T, e, e_din, has_match, ev):
    """lz_chains: returns (do_parse, k0, e_next, d_next)."""
    t0, t1 = T.t0, T.t1
    if (not has_match and not e_din) or e >= t1:
        if e >= t1:
            ev["parse_passed_tile"].append(t0)
        return False, None, max(e, t1), e_din
    k0 = (e - t0) // C_SEG
    ev["k0"].append(k0)
    for k in range(C_CHAINS):
        if k < k0:
            T.link[k] = k                                        # dead: self link, never reached
            continue
        p, din = (e, e_din) if k == k0 else (t0 + k * C_SEG, 0)
        _, mp, dout, pieces = c_walk(T, 0, k, p, din, ev)
        vb = 0
        for qr, L, _ in pieces:
            vb |= 1 << (qr & 15)
            T.nib(qr, L, 0)
        T.V[k] = vb                                              # (walk 0 stores its segment's len4 words whole)
        T.xfree[k], T.xdin[k] = mp, dout
        T.w0[k] = (p, din, pieces, mp, dout)
    for k in range(k0, C_CHAINS):
        lk, mp, dout, _ = c_walk(T, 1, k, T.xfree[k], T.xdin[k], ev)
        need(lk == END or lk > k, "a link goes backwards", k, lk)
        T.link[k], T.mpos[k] = lk, mp
        if lk == END:
            T.xdin[k] = dout
    for qr, c in T.w1_writers.items():
        if c >= 2 and T.len4[qr] == 15:
            ev["nibble15_shared_by_walk1"].append((t0 + qr, c))
    # in-warp pointer doubling: 5 rounds of shuffles
    jmp, pm = [0] * C_CHAINS, [0] * C_CHAINS
    for t in range(C_CHAINS):
        lk = T.link[t]
        inwarp = lk != END and lk != t and (lk >> 5) == (t >> 5)
        jmp[t] = lk & 31 if inwarp else t & 31
        pm[t] = (1 << (t & 31)) | (1 << jmp[t])
    for _ in range(5):
        npm, nj = pm[:], jmp[:]
        for t in range(C_CHAINS):
            src = (t & ~31) | jmp[t]
            npm[t] = pm[t] | pm[src]
            nj[t] = jmp[src]
        pm, jmp = npm, nj
    for t in range(k0, C_CHAINS):
        src = (t & ~31) | jmp[t]
        need(jmp[src] == jmp[t], "pointer doubling has not converged after 5 rounds", t)
        way, x = 1 << (t & 31), t
        while T.link[x] != END and (T.link[x] >> 5) == (t >> 5):
            x = T.link[x]
            way |= 1 << (x & 31)
        need(pm[t] == way and (x & 31) == jmp[t], "pointer doubling found another way through the warp", t)
    jump = [(t & ~31) | jmp[t] for t in range(C_CHAINS)]
    # the warp hops of thread 0
    entry = [None] * 8
    cur, hops = k0, 0
    T.min_[k0] = (e - t0) & (C_SEG - 1)
    while True:
        entry[cur >> 5] = cur
        t = jump[cur]
        tl = T.link[t]
        hops += 1
        need(hops <= 8, "more than 8 warp hops", t0)
        if tl == END:
            e_next, d_next = T.mpos[t], T.xdin[t]
            break
        need(tl != t and (tl >> 5) > (t >> 5), "a warp hop does not leave its warp", t, tl)
        if (tl >> 5) - (t >> 5) >= 2:
            ev["link_skips_warp"].append(t0 + t * C_SEG)
        T.min_[tl] = (T.mpos[t] - t0) & (C_SEG - 1)
        cur = tl
    ev["warp_hops"].append(hops)
    for w in range(8):
        a = entry[w]
        T.pathmask[w] = pm[a] if a is not None else 0
        if a is not None:
            steps, x = 0, a
            while True:                                          # chain length inside the warp: rounds it needed
                lk = T.link[x]
                if lk == END or (lk >> 5) != w:
                    break
                x, steps = lk, steps + 1
            ev["inwarp_path_steps"].append(steps)
        elif w > (k0 >> 5) and any(entry[x] is not None for x in range(w + 1, 8)):
            ev["warp_without_path_chain"].append((t0, w))
        for lane in range(32):
            t = 32 * w + lane
            lk = T.link[t]
            if (T.pathmask[w] >> lane) & 1 and lk != END and lk != t and (lk >> 5) == w:
                T.min_[lk] = (T.mpos[t] - t0) & (C_SEG - 1)
    ev["path_warps"].append(sum(x is not None for x in entry))
    need(e_next <= t1 + C_SEG, "the parse leaves the tile more than a segment past its end", t0, e_next)
    if k0 == 0 and e_din:
        ev["entry_in_match_seg0"].append(t0)
    if k0 == 1 and e_din:
        ev["entry_in_match_seg1"].append(t0)
    ev["entry_min"].append((e - t0) & (C_SEG - 1))
    return True, k0, e_next, d_next


class Back:
    """LzBack for one tile: Sel, Cont, clen."""

    def __init__(self):
        self.sel, self.cont, self.clen = set(), set(), {}

    def mark(self, rel, cont, E=None):
        self.sel.add(rel)
        if cont:
            need(rel % C_SEG == 0 and 1 <= E <= C_SEG, "Cont piece off a segment start or of a bad length", rel, E)
            self.cont.add(rel)
            self.clen[rel // C_SEG] = E


class Pending:
    def __init__(self):
        self.valid, self.lit, self.start, self.off, self.end = 0, 0, 0, 0, 0


def check_entry(T, k, m, ev):
    """The true path enters chain k (at tile position m, free) on its walk-0 trajectory: walk 0 re-run from m takes
    exactly the V bits at or past m and leaves the segment in the same state."""
    p0, din0, pieces, mp, dout = T.w0[k]
    _, mp2, dout2, pieces2 = c_walk(T, 0, k, T.t0 + m, 0, ev, dry=True)
    want = [(qr, L) for qr, L, _ in pieces if qr >= m]
    need([(qr, L) for qr, L, _ in pieces2] == want and (mp2, dout2) == (mp, dout),
         "the true path enters a chain off its walk-0 trajectory", T.t0 + m, k)
    rel = m & 15
    if T.t0 + m == p0:
        ev["entry_form"].append("walk0_start")
    elif (T.V[k] >> rel) & 1:
        ev["entry_form"].append("v_bit")
    else:
        ev["entry_form"].append("free_inside")


def lz_piece_len(T, K, pr):
    return K.clen[pr // C_SEG] if pr in K.cont else 4 + T.len4[pr]


def back_tile(T, k0, e_din, pd, ev, mutant=None):
    """lz_heads + lz_seq_run + lz_next_pending: returns the sequences the tile closes, as (literal start, literal
    length, offset, match length)."""
    t0 = T.t0
    K = Back()
    for w in range(8):
        for lane in range(32):
            k = 32 * w + lane
            if (T.pathmask[w] >> lane) & 1:
                ev["path_" + T.why[k]].append(t0 + k * C_SEG)
                if k != k0 or not e_din:
                    check_entry(T, k, k * C_SEG + T.min_[k], ev)
                c_walk(T, 2, k, t0 + k * C_SEG + T.min_[k], e_din if k == k0 else 0, ev, back=K, mutant=mutant)
    for j, E in K.clen.items():
        ev["cont_len"].append(E)
    piece = sorted(K.sel)
    np_ = len(piece)
    need(np_ <= C_MAXPIECE, "more pieces than C_MAXPIECE", t0, np_)
    need(np_ <= 4 * C_CHAINS + 1, "more pieces than 4 per segment and one at the entry", t0, np_)
    last = [0] * C_CHAINS
    for pr in piece:
        if pr not in K.cont:
            last[pr // C_SEG] = pr + 1
    segprev, m = [0] * C_CHAINS, 0
    for j in range(C_CHAINS):
        segprev[j] = m
        m = max(m, last[j])
    if np_ == 0:
        return [], None
    ppt = -(-np_ // P_TEAM)
    need(ppt <= C_MAXPIECE // P_TEAM, "ppt past the unrolled loop", t0, ppt)
    ev["ppt"].append(ppt)
    ev["pieces"].append(np_)
    hidx = []
    for r, pr in enumerate(piece):
        head = pr not in K.cont
        if head:
            if r == 0:
                pend, poff = (pd.end if pd.valid else None), pd.off
            else:
                pb = piece[r - 1]
                pend = t0 + pb + lz_piece_len(T, K, pb)
                if pb not in K.cont or mutant == "head_prev_piece_offset":
                    poff = T.off[pb]
                else:
                    sp = segprev[pb // C_SEG]
                    poff = T.off[sp - 1] if sp else pd.off
                    if not sp:
                        ev["cont_offset_from_pending"].append(t0 + pb)
                    elif (sp - 1) // (32 * C_SEG) < pb // (32 * C_SEG):
                        ev["segprev_from_earlier_warp"].append(t0 + pb)
            if pend == t0 + pr and poff == T.off[pr]:
                head = False
                ev["fold_after_cont" if r and piece[r - 1] in K.cont else "fold_same_offset"].append(t0 + pr)
        if r == 0 and not head:
            ev["first_piece_extends_pending"].append(t0)
        if head:
            hidx.append(r)
    nh = len(hidx)
    need(nh <= C_TILE // 4, "more heads than hidx holds", t0, nh)
    lastp = piece[-1]
    tile_end = t0 + lastp + lz_piece_len(T, K, lastp)
    if nh == 0:
        need(pd.valid, "a tile without heads and nothing pending", t0)
        ev["tile_without_head"].append(t0)
        pd.end = tile_end
        return [], tile_end
    if pd.valid and hidx[0] > 0:
        pb = piece[hidx[0] - 1]
        pd.end = t0 + pb + lz_piece_len(T, K, pb)
    # lz_seq_run
    nemit = pd.valid + nh - 1
    need(nemit <= LZ_SPT * P_TEAM, "more sequences than LZ_SPT per thread", t0, nemit)
    ev["spt"].append(-(-nemit // P_TEAM))
    out = []
    for sidx in range(nemit):
        if pd.valid and sidx == 0:
            ls, st, of, en = pd.lit, pd.start, pd.off, pd.end
        else:
            h = sidx - pd.valid
            pi = hidx[h]
            pr = piece[pi]
            pl = piece[hidx[h + 1] - 1]
            st, of, en = t0 + pr, T.off[pr], t0 + pl + lz_piece_len(T, K, pl)
            if h == 0:
                ls = pd.end if pd.valid else pd.lit
            else:
                pp = piece[pi - 1]
                ls = t0 + pp + lz_piece_len(T, K, pp)
        out.append((ls, st - ls, of, en - st))
    # lz_next_pending
    pi = hidx[nh - 1]
    pr = piece[pi]
    if nh >= 2 or pd.valid:
        ls = t0 + piece[pi - 1] + lz_piece_len(T, K, piece[pi - 1]) if pi > 0 else pd.end
    else:
        ls = pd.lit
    pd.valid, pd.lit, pd.start, pd.off, pd.end = 1, ls, t0 + pr, T.off[pr], tile_end
    if ls < t0 and t0 + pr - ls > C_LONGLIT:
        ev["pending_long_literals_from_earlier_tile"].append(t0)
    return out, tile_end


# ------------------------------------------------------------------------------------------------- emission
def c_seq_size(lit, L):
    s = 1 + lit + 2
    if lit >= 15:
        s += 1 + (lit - 15) // 255
    if L - 4 >= 15:
        s += 1 + (L - 19) // 255
    return s


def _len_bytes(x):
    return bytes([255] * (x // 255) + [x % 255])


def c_emit_seq(s, lit0, lit, off, mlen):
    """The bytes of one sequence and the long jobs it queues."""
    need(lit >= 0 and mlen >= 4 and 1 <= off <= lit0 + lit, "a malformed sequence", lit0, lit, off, mlen)
    ml = mlen - 4
    b = bytearray([((15 if lit >= 15 else lit) << 4) | (15 if ml >= 15 else ml)])
    if lit >= 15:
        b += _len_bytes(lit - 15)
    b += bytes(s[lit0: lit0 + lit])
    b += bytes([off & 255, off >> 8])
    jobs = int(lit > C_LONGLIT)
    if ml >= 15:
        b += _len_bytes(ml - 15)
        jobs += (ml - 15) // 255 > LONG_ML_RUNS
    need(len(b) == c_seq_size(lit, mlen), "c_seq_size disagrees with the sequence written", lit, mlen)
    return bytes(b), jobs


def lz4_block(src, ev=None, base=0, mutant=None):
    """The kernel's encoding of one block (<= 64 KiB): (LZ4 block bytes or None when stored raw, [(ll, off, ml)],
    offsets, events)."""
    ev = defaultdict(list) if ev is None else ev
    n = len(src)
    assert 0 < n <= BLK
    s = bytes(np.asarray(src, np.uint8).tobytes()) + bytes(40)
    off = candidates(s, n, ev, base)
    limit = n - 5 if n >= 5 else 0
    if n < 16:
        ev["block_shorter_than_16"].append(n)
    e = e_din = 0
    pd = Pending()
    body, seqs = bytearray(), []

    def emit(rows):
        nonlocal body
        jobs = 0
        for ls, lit, of, ml in rows:
            b, j = c_emit_seq(s, ls, lit, of, ml)
            body += b
            jobs += j
            seqs.append((lit, of, ml))
        return jobs

    for t0 in range(0, n, C_TILE):
        T = Tile(s, off, t0, limit)
        has_match = any(T.M)
        do, k0, e, e_din2 = front_tile(T, e, e_din, has_match, ev)
        if not do:
            if pd.valid:
                ev["tile_skipped_while_pending"].append(base + t0)
            continue
        din_in = e_din
        e_din = e_din2
        rows, _ = back_tile(T, k0, din_in, pd, ev, mutant)
        if rows:
            nl = emit(rows)
            need(nl <= LONGL_WORDS // 2, "more long jobs than LzBack::longl holds", t0, nl)
            ev["nlong"].append(nl)
    anchor = 0
    if pd.valid:
        anchor = pd.end
        nl = emit([(pd.lit, pd.start - pd.lit, pd.off, pd.end - pd.start)])
        ml = pd.end - pd.start - 4
        if pd.start - pd.lit > C_LONGLIT and ml >= 15 and (ml - 15) // 255 > LONG_ML_RUNS:
            ev["flush_long_literals_and_long_match"].append(base)
        ev["flush_jobs"].append(nl)
    lit = n - anchor
    fin = len(body) + 1 + lit + (1 + (lit - 15) // 255 if lit >= 15 else 0)
    ev["csize_minus_n"].append(fin - n)
    if fin >= n:
        return None, seqs, off, ev
    body += bytes([(15 if lit >= 15 else lit) << 4])
    if lit >= 15:
        body += _len_bytes(lit - 15)
    body += s[anchor: n]
    assert len(body) == fin
    return bytes(body), seqs, off, ev


def lz4_chunk(part, ev=None, mutant=None):
    """Every block of one chunk: ([(bytes or None, seqs, off)], events)."""
    ev = defaultdict(list) if ev is None else ev
    out = []
    for b0 in range(0, len(part), BLK):
        blk, seqs, off, _ = lz4_block(part[b0: b0 + BLK], ev, b0, mutant)
        out.append((blk, seqs, off))
    return out, ev


def parse_block(b):
    """(ll, off, ml) rows of an LZ4 block (the literals-only last sequence left out)."""
    rows, i = [], 0
    while i < len(b):
        tok = b[i]; i += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                x = b[i]; i += 1; ll += x
                if x != 255:
                    break
        i += ll
        if i >= len(b):
            break
        of = b[i] | (b[i + 1] << 8); i += 2
        ml = tok & 15
        if ml == 15:
            while True:
                x = b[i]; i += 1; ml += x
                if x != 255:
                    break
        rows.append((ll, of, ml + 4))
    return rows
