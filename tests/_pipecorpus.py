"""Inputs that drive the LZ4 level-1 compressor (and the zstd level-3 encoder on the same front end) to the edges of
their GPU schedule, as tests/_pipesched.py models it.  Every input is random bytes with a fixed seed plus placed
copies; each case carries a predicate over the model's events (and the twin's sequences) that names the edges it is
built for, and its builder takes knock_out=True to leave those constructions out, so that the test can show the
predicate depends on them.

A builder(knock_out) returns (src, chunk size or None for explicit sizes, marks, check) with check(ev, seqs, marks):
ev the model's events over the whole input, seqs[c][b] the twin's (ll, off, ml) rows of block b of chunk c, and marks
what the builder records about its layout."""
import numpy as np

import _pipesched as ps
import zstdmt_b200 as z

T, S, LB = ps.C_TILE, ps.C_SEG, ps.BLK


def rnd(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8)


def place(buf, pos, off, n):
    """buf[pos: pos + n] = the bytes `off` before them (an LZ copy), and the byte after them differs from the one `off`
    before it, so that the match is exactly n long."""
    assert off >= 1 and pos - off >= 0
    for i in range(0, n, off):
        k = min(off, n - i)
        buf[pos + i: pos + i + k] = buf[pos + i - off: pos + i - off + k]
    e = pos + n
    if e < buf.size and buf[e] == buf[e - off]:
        buf[e] ^= 0x55


def run(rng, buf, pos, n, d):
    """A match of exactly n bytes at pos with offset d <= 4 (the short-period candidate, which the candidate rounds
    always find): d random bytes before pos repeat to pos + n, and the byte after differs."""
    buf[pos - d: pos + n] = np.resize(rnd(rng, d), n + d)
    if pos + n < buf.size and buf[pos + n] == buf[pos + n - d]:
        buf[pos + n] ^= 0x55
    if buf[pos - d - 1] == buf[pos - 1]:
        buf[pos - d - 1] ^= 0x5A                                 # no candidate one position early


def _has(ev, name, want):
    got = set(ev.get(name, []))
    missing = [w for w in want if w not in got]
    assert not missing, (name, missing[:8])


def _h(v):
    return ((v * 2654435761) & 0xFFFFFFFF) >> 20


# ------------------------------------------------------------------------------------------------- candidate rounds
def cand_rounds(knock_out=False):
    """One block.  At 2000 (quad-aligned) a 6-byte run: three eligible positions of one quad with one window, so the
    first two inserts are skipped.  The block ends with a run over n - 13 .. n - 1, so that in the last quad with an
    eligible position, n - 12, a later position has the same hash but is past MFLIMIT (the earlier insert stands).
    A window v1 at 100 and a different one v2 with the same 12-bit hash at 1500 (the verify read fails), a window at
    2100 repeated at 2400 (same round: no candidate yet) and at 3300 (next round: a candidate), a period-2 run at 6000
    whose bytes also occurred in an earlier round (period and table hit together: d = 2 wins), and a block that starts
    with 8 zero bytes (d > k in the first quad, where the bytes below the block read as zeros)."""
    rng = np.random.default_rng(9001)
    n = 3 * T + 1000
    buf = rnd(rng, n)
    buf[:8] = 1 if knock_out else 0
    if not knock_out:
        buf[2000: 2006] = 0xA7
        buf[n - 13:] = 0xB3
        v1 = int.from_bytes(buf[100:104].tobytes(), "little")
        for c in range(1, 1 << 24):
            v2 = (v1 + (c << 8) * 0x1001) & 0xFFFFFFFF
            if v2 != v1 and _h(v2) == _h(v1):
                break
        buf[1500: 1504] = np.frombuffer(v2.to_bytes(4, "little"), np.uint8)
        buf[2400: 2408] = buf[2100: 2108]
        buf[3300: 3308] = buf[2100: 2108]
        buf[5000: 5040] = np.resize(buf[5000: 5002], 40)
        buf[6000: 6040] = buf[5000: 5040]

    def check(ev, seqs, m):
        _has(ev, "insert_skipped_same_hash", [(2000, 2), (2001, 1)])
        assert any(p >= n - 15 for p in ev.get("insert_stands_later_past_mflimit", []))
        _has(ev, "collision_verify_fails", [1500])
        _has(ev, "repeat_in_round_no_candidate", [2400])
        assert any(6000 <= p < 6040 for p in ev.get("period_beats_table", []))
        assert any(k > 0 for k, _ in ev.get("first_quad_d_gt_k", []))
    return buf, LB, {}, check


# ------------------------------------------------------------------------------------------------- tile entries
def tile_entries(knock_out=False):
    """Block 0: before tile boundary b (1..15) a match of x + 3 bytes from t1 - 3 (the piece is cut at t1 + 16, B - q
    < 4), so the parse enters tile b free at min_ = x = b; a copy in the middle of every tile gives it work.  Block 1:
    a long copy across boundary 1 (entry inside a match at segment 0), a match from t1 - 2 that runs past t1 + 16
    (the piece ends exactly at B = t1 + 16: entry inside a match at segment 1), and a tile whose last segment has no
    candidate (free entry at 0)."""
    rng = np.random.default_rng(9002)
    buf = rnd(rng, 2 * LB)
    for t in range(16):
        place(buf, t * T + 2000, 1500 + 7 * t, 40)
    for t in range(16, 32):
        place(buf, t * T + 2000, 1500 + 7 * t, 40)
    if not knock_out:
        for b in range(1, 16):
            run(rng, buf, b * T - 3, b + 3, 4)
        run(rng, buf, LB + T - 300, 600, 3)                     # across boundary 1 of block 1
        run(rng, buf, LB + 2 * T - 2, 80, 2)                    # piece [t1 - 2, t1 + 16) reaches B: segment 1

    def check(ev, seqs, m):
        assert set(range(16)) <= set(ev.get("entry_min", [])), sorted(set(ev.get("entry_min", [])))
        assert ev.get("entry_in_match_seg0") and ev.get("entry_in_match_seg1")
    return buf, 1 << 20, {}, check


# ------------------------------------------------------------------------------------------------- walk 1 and the path
def walks(knock_out=False):
    """Two blocks of random bytes with copies of 4 to 40 bytes at offsets up to 3000 every 5 to 30 bytes (many
    speculative chains whose continuations meet: by V bit, at a free segment start, and at a boundary candidate with
    the carried offset or another one; 19-byte pieces several continuations take), a 1100-byte copy from the start
    of a round whose source starts 8 bytes before it (only its first window is in the table, so one continuation runs
    through the round's two warps to the next round's first boundary: a link that skips a whole warp, and a warp
    without a chain on the path), one tile with a single short copy at its start (the
    path runs segment by segment through every warp: in-warp chains of 31 links, all five doubling rounds), and copies
    that leave the tile free and inside a match.  Block 2 is the generator's mixed content, where candidates at almost
    every position make many continuations meet (there several take one 19-byte piece)."""
    rng = np.random.default_rng(9003)
    buf = rnd(rng, 3 * LB)
    if not knock_out:
        buf[2 * LB:] = z.gen_stream(z.GEN_MIX, LB, 1 << 20, first=2)
        p = 4000
        while p < LB - 200:
            ln = int(rng.integers(4, 41))
            place(buf, p, int(rng.integers(100, 3000)), ln)
            p += ln + int(rng.integers(0, 26))
        place(buf, LB + 5 * 1024 + 40, 48, 1100)               # only its first window is in the table
        place(buf, LB + 2 * T, 1000, 6)
        place(buf, LB + 3 * T - 40, 1700, 200)
        place(buf, LB + 4 * T - 5, 900, 5)

    def check(ev, seqs, m):
        for name in ("w1_merge_v_bit", "w1_merge_free_start", "w1_merge_same_match", "w1_boundary_other_offset",
                     "w1_leave_free", "w1_leave_in_match", "w1_last_segment_exhausted", "w1_segment_exhausted",
                     "nibble15_shared_by_walk1", "link_skips_warp", "warp_without_path_chain",
                     "path_merge_v_bit", "path_merge_free_start", "path_merge_same_match"):
            assert ev.get(name), name
        assert max(ev.get("inwarp_path_steps", [0])) >= 17 and max(ev.get("path_warps", [0])) == 8
        assert {"walk0_start", "v_bit"} <= set(ev.get("entry_form", []))
    return buf, 1 << 20, {}, check


# ------------------------------------------------------------------------------------------------- marking and heads
def marking(knock_out=False):
    """Copies that cross a segment boundary and end x = 1..16 bytes past it (Cont pieces of every length) or exactly
    on it (E = 0), each inside one round with its source starting 6 bytes before the round (no candidate at the
    boundary, so the match goes on as a Cont piece), a copy at offset 600 across a round boundary (no candidate in its own round:
    Cont pieces, then the boundary candidate of the next round with the same offset, folded by head detection after a
    Cont piece), a 700-byte copy (segprev found in an earlier warp), a copy across a tile boundary (a Cont at the
    tile's start continues the pending offset; the tile's first piece extends the pending sequence), a 5000-byte copy
    (a tile without heads), and a tile of random bytes after a sequence (skipped while a sequence is pending)."""
    rng = np.random.default_rng(9004)
    buf = rnd(rng, 2 * LB)
    if not knock_out:
        for x in range(0, 17):                                   # block 1, round 2x + 2: Cont of x bytes
            r0 = LB + (2 * x + 2) * 1024
            place(buf, r0 + 39, 45, 9 + x)                       # B = r0 + 48; source windows past r0 - 1 unseen
        place(buf, 2 * 1024 - 300, 600, 700)                     # rounds 1 | 2 of tile 0
        place(buf, T + 2000, 2500, 700)
        place(buf, 2 * T - 100, 1800, 300)                       # tile 1 | 2
        place(buf, 4 * T - 500, 3000, 5000)                      # tile 4 without heads
        place(buf, 7 * T + 100, 900, 30)                         # tile 8: nothing; tile 7's sequence pending

    def check(ev, seqs, m):
        assert set(range(1, 17)) <= set(ev.get("cont_len", []))
        for name in ("match_ends_on_boundary", "fold_after_cont", "fold_same_offset", "segprev_from_earlier_warp",
                     "cont_offset_from_pending", "first_piece_extends_pending", "tile_without_head",
                     "tile_skipped_while_pending"):
            assert ev.get(name), name
    return buf, 1 << 20, {}, check


# ------------------------------------------------------------------------------------------------- density
WORDS = np.array([[j, 64 + j, 128 + j, 192 + j] for j in range(64)], np.uint8)


def de_bruijn(k):
    """B(k, 2): a cyclic sequence of k * k symbols in which every ordered pair occurs once."""
    a, seq = [0] * (2 * k), []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1: p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq


def dense(knock_out=False):
    """Tile 0 defines 64 four-byte words w_j = (j, 64 + j, 128 + j, 192 + j), each followed by a separator.  Tiles 1-3:
    the words in the order of a de Bruijn sequence B(64, 2): every word is a 4-byte match and two neighbours never
    share an offset, so a tile holds close to 1024 pieces and sequences (ppt = spt = 4; some words lose their table
    slot to another window).  Tiles 4-5: runs of 33 literals, each followed by a 4-byte match at offset 4 (a
    long-literal job per sequence: > 100 per tile).  The block ends with 100 literals and a 2000-byte copy that stays pending to the flush (a long literal job and a long match-length job)."""
    rng = np.random.default_rng(9005)
    buf = rnd(rng, LB)
    pre = np.concatenate([np.append(w, 64 + (j * 7 + 1) % 64) for j, w in enumerate(WORDS)])
    buf[100: 100 + pre.size] = pre
    if not knock_out:
        seq = de_bruijn(64)
        buf[T: 4 * T] = WORDS[seq[: 3 * T // 4]].reshape(-1)
        for p in range(4 * T, 6 * T - 36, 37):
            buf[p: p + 33] = rnd(rng, 33)
            run(rng, buf, p + 33, 4, 4)                          # the run's first 4 bytes are the literals' last 4
        buf[LB - 2300: LB - 2200] = rnd(rng, 100)
        run(rng, buf, LB - 2200, 2000, 3)

    def check(ev, seqs, m):
        assert max(ev.get("ppt", [0])) >= 3 and max(ev.get("spt", [0])) >= 3
        assert max(ev.get("nlong", [0])) >= 100
        assert ev.get("flush_long_literals_and_long_match")
    return buf, 1 << 20, {}, check


def _hash_slots_clean(buf, words, lo, hi):
    """Every window in buf[lo: hi] whose 12-bit hash is a word's hash is that word (no other window takes its slot)."""
    key = lambda a: int.from_bytes(a.tobytes(), "little")
    wh = {_h(key(w)): key(w) for w in words}
    return len(wh) == len(words) and all(wh.get(_h(key(buf[i: i + 4])), key(buf[i: i + 4])) == key(buf[i: i + 4])
                                         for i in range(lo, hi))


def densest_tile(knock_out=False):
    """A tile with the most pieces the rule admits, 4 * 256 + 1 = 1025 (ppt 5).  A segment holds at most 4 piece
    starts plus a Cont piece, and only when the match is still open at its start; a segment that closes a match on its
    end boundary has at most 3 starts unless it began free at offset 0, which only the tile's entry can.  So a tile gains
    one piece over 4 per segment at most once: here, by an entry inside a match.
    16 words of four byte classes ((c0, c1, c2, c3) with c_k in [64 k, 64 k + 64)) chosen so that no other window of
    the region takes a word's hash slot.  Tile 2, round 2: the words in random order (their first occurrences); round 3:
    words at offsets 0, 4, 8, 12 of every segment, each a 4-byte match whose piece ends on its cut.  At t1 = 3 * 4096 one
    byte x continues the match of the word at t1 - 4 (a 1-byte Cont at the tile's start), and from t1 + 1 on the words
    run at offsets 1, 5, 9, 13 of every segment of tile 3 (the last spills 1 byte into the next segment): 1 + 1024
    pieces.  A word is never followed by the word that followed its source, so every match is exactly 4 bytes and two
    neighbours never share an offset.  knock_out: x does not continue the match (no Cont, 1024 pieces)."""
    K, t1 = 16, 3 * T
    rng = np.random.default_rng(29)
    buf = rnd(rng, LB)
    words = np.stack([rng.choice(64, K, replace=False) + 64 * c for c in range(4)], axis=1).astype(np.uint8)
    occ = list(range(t1 - 2048, t1, 4)) + list(range(t1 + 1, 4 * T + 64, 4))
    ws, hist = [], {w: [] for w in range(K)}             # hist: (position, follower) of each word's occurrences
    xw = None
    for i, q in enumerate(occ):
        if q == t1 + 1:                                  # the word at t1 - 4: its source's follower gives x
            wl = ws[-1]
            xw = [f for pp, f in hist[wl] if pp < t1 - 1024][-1]
            hist[wl].append((t1 - 4, xw))
        prev = ws[-1] if i and occ[i - 1] + 4 == q else None
        bad = set()
        if prev is not None:
            bad.add(prev)
            r0 = occ[i - 1] - occ[i - 1] % 1024
            src = [f for pp, f in hist[prev] if pp < r0]
            if src:
                bad.add(src[-1])                         # the follower at the source: the match would grow
        w = int(rng.choice([b for b in range(K) if b not in bad]))
        if prev is not None:
            hist[prev].append((occ[i - 1], w))
        ws.append(w)
    for q, w in zip(occ, ws):
        buf[q: q + 4] = words[w]
    buf[t1] = words[xw][0] if not knock_out else words[xw][0] ^ 0x20
    buf[4 * T + 64] ^= 0x5A
    assert _hash_slots_clean(buf, words, t1 - 2048, 4 * T + 80)

    def check(ev, seqs, m):
        assert max(ev.get("pieces", [0])) == 4 * 256 + 1 and max(ev.get("ppt", [0])) == 5
    return buf, 1 << 20, {}, check


def pending_literals(knock_out=False):
    """Random bytes across a tile boundary, then one match 10 bytes into the next tile: the tile's only sequence is
    left pending with a literal run of more than 32 bytes that began in the tile before."""
    rng = np.random.default_rng(9006)
    buf = rnd(rng, 3 * T)
    place(buf, 500, 300, 20)
    if not knock_out:
        place(buf, T + 10, 2000, 30)

    def check(ev, seqs, m):
        assert ev.get("pending_long_literals_from_earlier_tile")
    return buf, 1 << 20, {}, check


# ------------------------------------------------------------------------------------------------- block end
def _size_of(buf):
    _, _, _, ev = ps.lz4_block(buf)
    return ev["csize_minus_n"][-1]


def block_sizes(knock_out=False):
    """Three 4096-byte chunks of random bytes, each with one copy whose length is tuned so that the block encodes to
    exactly n - 1 (written compressed), n and n + 1 bytes (stored raw)."""
    rng = np.random.default_rng(9007)
    chunk = 4096
    buf = rnd(rng, 3 * chunk)
    if not knock_out:
        for c, want in enumerate((-1, 0, 1)):
            base = buf[c * chunk: (c + 1) * chunk].copy()
            for ln in range(4, 40):
                part = base.copy()
                place(part, 2000, 1000, ln)
                if _size_of(part) == want:
                    break
            assert _size_of(part) == want, (c, want)
            buf[c * chunk: (c + 1) * chunk] = part

    def check(ev, seqs, m):
        assert {-1, 0, 1} <= set(ev["csize_minus_n"])
    return buf, chunk, {}, check


def tiny_blocks(knock_out=False):
    """Chunks of 1..15 bytes (and 16..31): blocks shorter than a staging word."""
    rng = np.random.default_rng(9008)
    lo = 16 if knock_out else 1
    sizes = list(range(lo, lo + 15))
    buf = np.concatenate([np.zeros(s, np.uint8) if s % 3 == 0 else rnd(rng, s) for s in sizes])

    def check(ev, seqs, m):
        assert set(range(1, 16)) <= set(ev.get("block_shorter_than_16", []))
    return buf, None, {"sizes": sizes}, check


BUILDERS = [cand_rounds, tile_entries, walks, marking, dense, densest_tile, pending_literals, block_sizes, tiny_blocks]


def parts(src, chunk, marks):
    """The chunk contents of a case (tiny_blocks: one chunk per listed size)."""
    if chunk is None:
        out, a = [], 0
        for s in marks["sizes"]:
            out.append(src[a: a + s]); a += s
        return out
    return [src[i: i + chunk] for i in range(0, max(src.size, 1), chunk)]
