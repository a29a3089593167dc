"""Inputs that drive the chain-search encoders (zstd levels 6-12, LZ4 levels 10-12) to the edges of their GPU
schedule (tests/_searchsched.py models it).  Every input is built with a fixed seed from random bytes and placed
copies; each case names its levels and a predicate that asserts, from the model's events and the twin's sequences,
that the edge was reached.

Case: name, codec ("zstd" or "lz4"), levels, src, chunk size, explicit chunk sizes (or None), check(level, ev, seqs,
best) where ev are the model's events over every chunk, seqs[c][b] the twin's (ll, off, ml) rows of block b of chunk c
and best[c] the twin's best[] of chunk c, and optionally gpu_check(level, rep) on what the GPU test's check() returns."""
from collections import namedtuple

import numpy as np

import _lz4hc as hc
import _zlazy as zl

Case = namedtuple("Case", "name codec levels src chunk chunk_bytes check gpu_check", defaults=(None,))
ZB, LB, Q, R = 16384, 65536, 16384, 64


def rnd(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8)


def place(buf, pos, off, n):
    """buf[pos: pos + n] = the bytes `off` before them (overlapping like an LZ copy), and the byte after them differs
    from the one `off` before it, so that the match is exactly n long."""
    assert off >= 1 and pos - off >= 0
    for i in range(0, n, off):
        k = min(off, n - i)
        buf[pos + i: pos + i + k] = buf[pos + i - off: pos + i - off + k]
    e = pos + n
    if e < buf.size and buf[e] == buf[e - off]:
        buf[e] ^= 0x55


def starts(rows):
    """(match start, offset, length) of one block's (ll, off, ml) rows, block-relative."""
    rows = np.asarray(rows, np.int64).reshape(-1, 3)
    st = np.cumsum(rows[:, 0] + rows[:, 2]) - rows[:, 2]
    return np.stack([st, rows[:, 1], rows[:, 2]], axis=1)


def _details(ev, name):
    return ev.get(name, [])


def abs_starts(blocks, block):
    """(absolute match start, offset, length) of every match of one chunk's per-block rows."""
    out = [starts(rows) + [b * block, 0, 0] for b, rows in enumerate(blocks)]
    return np.concatenate(out) if out else np.zeros((0, 3), np.int64)


def unpack(m):
    return int(m) & 511, int(m) >> 9


# ------------------------------------------------------------------------------------------------- zstd
def zstd_phases():
    """Block 0: random source.  Blocks 1-2: a 300-byte copy starting at every phase 0..63 of a 64-position range, so
    that its second best[] piece (at start + 256) is a range entry folding into it at that phase.  Block 4: a copy of
    block 3, one merged match of the whole block made of 64 pieces of 256 whose folds carry from 63 ranges into one
    sequence; every fourth range has no entry, so each fold's previous range opens no sequence.  (Block 4 copies
    block 3, which nothing else copies: no nearer candidate ties with it.)"""
    rng = np.random.default_rng(601)
    buf = rnd(rng, 5 * ZB + 1000)
    cur = ZB + 40
    for ph in range(R):
        p = cur + (ph - cur) % R
        if p // ZB != (p + 300) // ZB:
            p = (p // ZB + 1) * ZB + 40
            p += (ph - p) % R
        place(buf, p, p - (100 + 211 * ph), 300)
        cur = p + 320
    place(buf, 4 * ZB, ZB, ZB)

    def check(level, ev, seqs, best):
        assert set(_details(ev, "fold_at_entry")) == set(range(R))
        assert max(_details(ev, "carry_from_k_ranges")) == 63
        assert _details(ev, "fold_after_range_without_sequence")
        assert [tuple(r) for r in seqs[0][4].tolist()] == [(0, ZB, ZB)]
    return Case("zstd_phases", "zstd", (6, 8, 12), buf, 1 << 20, None, check)


def zstd_range_ends():
    """Copies that end exactly at a range end and one byte either side, copies that skip a whole range, and random
    bytes between them, so that ranges have literal entries."""
    rng = np.random.default_rng(602)
    buf = rnd(rng, 3 * ZB)
    p, k = ZB + 100, 0
    for d in (0, -1, 1) * 8:
        end = (p // R + 2) * R + d
        ln = 40 + 7 * (k % 5)
        place(buf, end - ln, end - ln - (200 + 97 * k), ln)
        p, k = end + 30, k + 1
    for j in range(8):
        s = 2 * ZB + 200 + j * 600
        place(buf, s, s - (300 + 131 * j), 140 + 3 * j)

    def check(level, ev, seqs, best):
        for name in ("match_ends_at_range_end", "match_ends_one_before_range_end", "match_ends_one_past_range_end",
                     "match_skips_range", "range_no_entry", "entry_is_literal"):
            assert len(_details(ev, name)) >= 6, name
    return Case("zstd_range_ends", "zstd", (6, 8, 12), buf, 1 << 20, None, check)


def defer_pairs(rng, buf, at, minmatch, depth2):
    """At `at` a short match (minmatch bytes) and one (depth 1) or two (depth 2) positions later a 64-byte one; the
    sources lie at the start of buf.  Returns the next free source position."""
    Rr = rnd(rng, 64)
    pre = rnd(rng, 2 if depth2 else 1)
    src = at - 5000
    buf[src: src + 64] = Rr
    s2 = src + 100
    short = np.concatenate([pre, Rr[: minmatch - pre.size]])
    buf[s2: s2 + short.size] = short
    buf[s2 + short.size] = Rr[minmatch - pre.size] ^ 0x5A                       # the short match stops there
    buf[at: at + pre.size] = pre
    buf[at + pre.size: at + pre.size + 64] = Rr
    buf[at + pre.size + 64] ^= 0x33


def tie_pair(rng, buf, at, k, ls, o0, ll, o1):
    """At `at` a match of exactly ls bytes at offset o0; k (1 or 2) positions later one of exactly ll bytes at offset o1
    (the k bytes at `at` come first, then 64 bytes R whose first ll bytes the longer match copies)."""
    Rr, pre = rnd(rng, 64), rnd(rng, k)
    a, b = at - o0, at + k - o1
    assert a + ls < b or b + ll < a
    buf[at: at + k] = pre
    buf[at + k: at + k + 64] = Rr
    buf[at + k + 64] ^= 0x33
    buf[b: b + ll] = Rr[:ll]
    buf[b + ll] = Rr[ll] ^ 0x5A
    short = np.concatenate([pre, Rr[: ls - k]])
    buf[a: a + ls] = short
    buf[a + ls] = Rr[ls - k] ^ 0x5A


# zstd ties: gain = 4 len - highbit(off + 3); offsets 5000 and 6000 share highbit 12, 3000 has 11 and 9000 has 13
ZSTD_TIES = [(1, 6, 5000, 7, 6000, False), (1, 6, 5000, 7, 3000, True),       # gain(m1) = g + 4 / g + 5
             (2, 6, 5000, 8, 9000, False), (2, 6, 5000, 8, 6000, True)]       # gain(m2) = g + 7 / g + 8
LZ4_TIES = [(1, 5, 5000, 6, 6000, False), (1, 5, 5000, 7, 6000, True),         # l1 = l0 + 1 / l0 + 2
            (2, 5, 5000, 7, 6000, False), (2, 5, 5000, 8, 6000, True)]         # l2 = l0 + 2 / l0 + 3


def place_ties(rng, buf, first, ties):
    """Every threshold tie at its own position from `first` on, followed by 2000 zeros so that its block is written
    compressed rather than raw (a raw block would hide the parse); returns [(position, k, deferred at lazy depth 2)]."""
    out = []
    for i, (k, ls, o0, ll, o1, defer) in enumerate(ties):
        at = first + 12000 * i
        tie_pair(rng, buf, at, k, ls, o0, ll, o1)
        buf[at + 200: at + 2200] = 0                                        # the block shrinks: its parse is written
        out.append((at, k, defer))
    return out


def check_ties(ties, rows, lazy):
    """A tie does not defer, one past it does (the look two ahead only at lazy depth 2)."""
    st = set(rows[:, 0].tolist())
    for at, k, defer in ties:
        d = defer and (k == 1 or lazy >= 2)
        assert (at in st, at + k in st) == (not d, d), (at, k, defer, lazy)


def zstd_defer():
    """Lazy deferrals at r1 - 1 (the longer match at p + 1 lies in the next range) and at r1 - 2 with depth 2 (p + 2),
    and matches exactly on each lazy threshold and one past it (ZSTD_TIES)."""
    rng = np.random.default_rng(603)
    buf = rnd(rng, 4 * ZB + 60000)
    for j in range(6):
        defer_pairs(rng, buf, ZB + 600 + j * 900 + (63 - (ZB + 600 + j * 900) % R), 5, False)
        a = 2 * ZB + 600 + j * 900
        defer_pairs(rng, buf, a + (62 - a % R), 5, True)
    ties = place_ties(rng, buf, 4 * ZB + 10000, ZSTD_TIES)

    def check(level, ev, seqs, best):
        d = _details(ev, "defer_looks_into_next_range")
        assert any(p % R == 63 and k == 1 for p, k in d)
        assert any(p % R == 62 and k == 2 for p, k in d) == (level >= 8)
        check_ties(ties, abs_starts(seqs[0], ZB), zl.params(level)[2])
    return Case("zstd_defer", "zstd", (6, 8, 12), buf, 1 << 20, None, check)


def lz4_defer_ties():
    """Matches exactly on each lazy threshold of the LZ4 class and one past it (LZ4_TIES)."""
    rng = np.random.default_rng(607)
    buf = rnd(rng, 2 * LB)
    ties = place_ties(rng, buf, 10000, LZ4_TIES)

    def check(level, ev, seqs, best):
        check_ties(ties, abs_starts(seqs[0], LB), hc.PARAMS[level][1])
    return Case("lz4_defer_ties", "lz4", (10, 12), buf, 1 << 20, None, check)


def zstd_ends():
    """Matches that run to the block end, with the remaining length at every residue mod 4 and the source at every
    alignment mod 4 (the kernel's 4-byte compare, its tail loop and its funnel-shift load)."""
    rng = np.random.default_rng(604)
    buf = rnd(rng, 17 * ZB)
    combos = []
    for r in range(4):
        for s in range(4):
            b = 1 + 4 * r + s
            p = (b + 1) * ZB - (200 + r)
            src = 1000 + 64 * (4 * r + s)
            src += (s - src) % 4
            place(buf, p, p - src, 200 + r)
            combos.append((b, 200 + r, s))

    def check(level, ev, seqs, best):
        for b, ln, s in combos:
            st = starts(seqs[0][b])
            hit = st[(st[:, 0] + st[:, 2] == ZB)]
            assert len(hit) and hit[-1, 2] >= ln and (b * ZB + hit[-1, 0] - hit[-1, 1]) % 4 == s, (b, ln, s)
    return Case("zstd_ends", "zstd", (6, 12), buf, 1 << 20, None, check)


def zstd_offsets(level):
    """Offset_Value 2^k - 1 and 2^k (offset + 3) for k = 16 .. log2 of the level's window."""
    rng = np.random.default_rng(605 + level)
    kmax = 22 if level >= 10 else 21
    buf = rnd(rng, (1 << kmax) + 64 * ZB)
    want = []
    p = (1 << kmax) + 1000
    for k in range(16, kmax + 1):
        for ov in ((1 << k) - 1, 1 << k):
            place(buf, p, ov - 3, 48)
            want.append(ov)
            p += 300

    def check(lv, ev, seqs, best):
        got = {int(r[1]) + 3 for blk in seqs[0] for r in blk.tolist()}
        assert set(want) <= got
    return Case("zstd_offsets_l%d" % level, "zstd", (level,), buf, 8 << 20, None, check)


def zeros_chunks(minmatch, codec, levels):
    """Chunks of zeros with short explicit sizes side by side in one group: zeros hash to key 0, the key of every
    position without a hash too (a chunk's last minMatch - 1 bytes and the gap up to the chunk size), so a chain of key
    0 runs through every chunk and must stop at its own chunk's start."""
    chunk = 4096
    sizes = [0, 1, minmatch, minmatch + 1, 12, 13, 14, 64, 300, 17, 4096, 5, 4095, 100, 2000, 4096]
    buf = np.zeros(chunk * len(sizes), np.uint8)

    def check(level, ev, seqs, best):
        for c, n in enumerate(sizes):
            for blk in seqs[c]:
                st = starts(blk)
                assert (st[:, 1] <= st[:, 0]).all()
        assert sum(len(b) for s in seqs for b in s) >= 8
    return Case(codec + "_zeros_chunks", codec, levels, buf, chunk, sizes, check)


# ------------------------------------------------------------------------------------------------- LZ4
CARRIES = sorted({1, 2, 3, 4, 5, 6, 7, 31, 32, 33, 63, 64, 65, 127, 128, 129, 191, 192, 193, 250, 251, 252, 253, 254, 255}
                 | set(range(9, 256, 24)))


def lz4_quarters():
    """Every block carries three quarter boundaries; at each, a match crosses it and ends c = 1..255 positions into the
    next quarter, in one of three ways: its next best[] piece continues it (the entry folds into the open sequence), a
    match of another offset follows at once (no fold), or one literal comes between.  The last block has a merged
    match longer than a quarter (a quarter that opens no sequence) and a lazy deferral at q0 - 1, the block after it
    one at q0 - 2.  4000 zeros in each block make it shrink, so that it is written compressed rather than raw."""
    rng = np.random.default_rng(701)
    plan = [(c, v) for c in CARRIES for v in ("fold", "other", "literal")]
    nblk = -(-len(plan) // 3) + 2
    buf = rnd(rng, nblk * LB)
    it = iter(plan)
    for b in range(nblk - 2):
        buf[b * LB + 6000: b * LB + 10000] = 0                              # the block shrinks: its parse is written
        for qi in (1, 2, 3):
            c, v = next(it, (None, None))
            if c is None:
                break
            q0 = b * LB + qi * Q
            s1 = b * LB + 200 + qi * 1500 + c
            if v == "fold":
                st = q0 + c - 256
                place(buf, st, st - s1, 256 + 60)
            else:
                ln = min(256, c + 40)
                st = q0 + c - ln
                place(buf, st, st - s1, ln)
                if v == "other":
                    s2 = s1 + 700
                    while buf[s2] == buf[q0 + c - (st - s1)]:
                        s2 += 1
                    place(buf, q0 + c, q0 + c - s2, 50)
                else:
                    buf[q0 + c + 1: q0 + c + 51] = buf[q0 + c + 1 - (st - s1): q0 + c + 51 - (st - s1)]
                    buf[q0 + c + 51] ^= 0x21
    b0 = (nblk - 2) * LB
    place(buf, b0 + Q - 10, Q, Q + 100)                                   # quarter 1 opens no sequence
    defer_pairs(rng, buf, b0 + 3 * Q - 1, 4, False)
    defer_pairs(rng, buf, b0 + LB + 3 * Q - 2, 4, True)

    def check(level, ev, seqs, best):
        assert set(CARRIES) <= set(_details(ev, "quarter_carry_pos"))
        assert len(_details(ev, "quarter_entry_fold")) >= len(CARRIES)
        assert len(_details(ev, "quarter_entry_no_fold")) >= len(CARRIES)
        assert len(_details(ev, "quarter_entry_literal")) >= len(CARRIES)
        assert _details(ev, "open_across_whole_quarter")
        d = _details(ev, "defer_looks_into_next_quarter")
        assert any(k == 1 for _, k in d) and any(k == 2 for _, k in d)
    return Case("lz4_quarters", "lz4", (10, 12), buf, 16 << 20, None, check)


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


def kernel_constant(name, _files=("lz4_hc.cuh", "lz4_hc_rule.h", "lz4_kernels.cu")):
    """The value of an integer #define of the LZ4 class's sources (unsigned literals, integer division)."""
    import os
    import re
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zstdmt_b200", "csrc")
    defs = {}
    for f in _files:
        for m in re.finditer(r"^#define\s+(\w+)\s+(.+)$", open(os.path.join(csrc, f)).read(), re.M):
            defs[m.group(1)] = re.sub(r"//.*|/\*.*?\*/", "", m.group(2)).strip()

    def ev(n):
        expr = re.sub(r"\b(\d+)u\b", r"\1", defs[n]).replace("/", "//")
        return eval(re.sub(r"\b([A-Z_][A-Z0-9_]*)\b", lambda m: str(ev(m.group(1))), expr))
    return ev(name)


MAXSEQ, MAXLONG = kernel_constant("L4H_MAXSEQ"), kernel_constant("L4H_MAXLONG")


def lz4_dense():
    """The densest quarters of one 64 KiB block.
      quarter 0: 64 four-byte words w_j = (j, 64 + j, 128 + j, 192 + j), each followed by a separator, then random bytes
                 and a copy that ends exactly at the quarter's end (the sequence left open);
      quarter 1: the words in the order of a de Bruijn sequence B(64, 2): every pair of neighbours occurs once, so every
                 word is a 4-byte match (no 4-byte window straddling two words has occurred before, and the byte
                 classes keep matches from growing) and two neighbours never share an offset: 4096 sequences;
      quarter 2: literal runs of 33 bytes, each followed by one of the words (a 4-byte match); a run's first byte
                 differs from every earlier follower of the word before it and its last byte from every earlier byte
                 before the word after it, so that no word's match grows into the run;
      quarter 3: runs of 33 literals, each followed by a 1300-byte copy of quarter 0."""
    rng = np.random.default_rng(702)
    buf = rnd(rng, 2 * LB)
    words = np.array([[j, 64 + j, 128 + j, 192 + j] for j in range(64)], np.uint8)
    pre = np.concatenate([np.append(w, 64 + (j * 7 + 1) % 64) for j, w in enumerate(words)])
    buf[100: 100 + pre.size] = pre
    place(buf, Q - 120, Q - 120 - 2000, 120)
    seq = de_bruijn(64)
    buf[Q: 2 * Q] = words[seq].reshape(-1)
    followers = {j: set() for j in range(64)}                                 # class-c bytes seen right after word j
    leaders = {j: set() for j in range(64)}                                   # ... and right before it
    p, j, prev = 2 * Q, 0, seq[-1]
    while p + 37 <= 3 * Q:
        lit = rnd(rng, 33)                                                  # inside: 4-byte windows all but unique
        lit[[0, 32]] = rng.integers(128, 192, 2)                            # ends in class c: no window (lit, w) occurred
        while int(lit[0]) in followers[prev]:                               # else the word's match would grow
            lit[0] = rng.integers(128, 192)
        followers[prev].add(int(lit[0]))
        prev = (j * 29) % 64
        while int(lit[32]) in leaders[prev]:                                # else a match would start a byte early
            lit[32] = rng.integers(128, 192)
        leaders[prev].add(int(lit[32]))
        buf[p: p + 33] = lit
        buf[p + 33: p + 37] = words[prev]
        p += 37; j += 1
    for k in range(9):                                                      # sources: quarter 0, copied once each
        s = 3 * Q + 33 + 1334 * k
        place(buf, s, s - (2000 + 1310 * k), 1300)
    # derivation of the bounds: a quarter holds its own sequences, which start at distinct positions at least 4 apart
    # inside it (<= Q / 4), and the one left open before it: <= Q / 4 + 1 <= L4H_MAXSEQ.  It queues a long job per
    # literal run > 32 bytes of an emitted sequence (each followed by a match of >= 4 bytes: <= Q / 37 inside the
    # quarter, + 2 for the runs that begin before it: the open sequence's and the first new one's) and per match of
    # >= 1294 bytes (<= (Q + 255) / 1294 that end in it, + the open one): <= 442 + 2 + 12 + 1 = 457 <= L4H_MAXLONG.
    bound_seq, bound_long = Q // 4 + 1, Q // 37 + 2 + (Q + 255) // 1294 + 1
    assert bound_seq <= MAXSEQ and bound_long <= MAXLONG

    def check(level, ev, seqs, best):
        held, jobs = _details(ev, "held_sequences"), _details(ev, "long_jobs")
        assert max(held) == Q // 4 + 1 <= bound_seq
        assert max(jobs) == Q // 37 - 1 <= bound_long         # every run but the one of the sequence left open
        assert (starts(seqs[0][0])[:, 2] >= 1294).sum() == 9
    return Case("lz4_dense", "lz4", (10, 12), buf, 1 << 20, None, check)


def lz4_block_ends():
    """Chunks whose last block has n mod 65536 in {1..13, 16384 + 1..13, 3 * 16384 + 1..13} (the last of these with a
    tiny last quarter).  In each last block of 13 bytes or more, a copy runs into the block's end: the match that
    stops at blockEnd - 5 has a length of every residue mod 4; in others a match starts at exactly blockEnd - 12, or
    an 11-byte copy starts at blockEnd - 11, after random bytes, where no match may start.  Long last blocks are zeros
    but for their last 4000 bytes, so that they shrink and are not stored raw."""
    rng = np.random.default_rng(703)
    chunk = 2 * LB
    tails = [t for base in (0, Q, 3 * Q) for t in range(base + 1, base + 14)]
    sizes = [LB + t for t in tails]
    buf = rnd(rng, chunk * len(sizes))
    for c, (n, t) in enumerate(zip(sizes, tails)):
        a = c * chunk + LB
        if t > 8000:
            buf[a: a + t - 4000] = 0                 # the block shrinks: it is written compressed, not raw
        if t < 13:
            continue
        if c % 2:
            ln = 12 + (c // 2) % 4                   # a copy of ln bytes into the block end: the match stops 5 before
        else:
            ln = 12 if c % 4 == 0 else 11            # a match may start at t - 12; a copy starting at t - 11 is too late
        place(buf, a + t - ln, 3000, ln)

    def check(level, ev, seqs, best):
        at12, at11, ends = [], 0, set()
        for c, t in enumerate(tails):
            rows = starts(seqs[c][1]) if len(seqs[c]) > 1 else np.zeros((0, 3), np.int64)
            if t < 13:
                assert not len(rows)
                continue
            rows = rows[rows[:, 0] >= t - 4000]
            at12 += [int(r[0]) for r in rows if r[0] == t - 12]
            if c % 4 == 2:
                a = c * chunk + LB + t - 11
                assert np.array_equal(buf[a: a + 11], buf[a - 3000: a - 3000 + 11]) and (rows[:, 0] < t - 12).all()
                at11 += 1
            assert all(r[0] + 12 <= t and r[0] + r[2] <= t - 5 for r in rows)
            ends |= {int(r[2]) % 4 for r in rows if r[0] + r[2] == t - 5}
        assert at12 and at11 and ends == {0, 1, 2, 3}
    return Case("lz4_block_ends", "lz4", (10, 12), buf, chunk, sizes, check)


# ------------------------------------------------------------------------------------------------- chain depth
def chain_depth(codec, level):
    """The chain walk of the search kernel, at the level's depth d.  Three targets, each with its own key K (minMatch
    random bytes) that occurs only at the target and at the candidates before it (nearest first):
      take : c1 = K, c2 = K + 1 equal byte, c3 .. c(d-1) = K, c(d) = K + 30 equal bytes: the candidate exactly d
             steps back is the longest and is taken; c3 .. c(d-1) differ at qs[bl] and are passed over unmeasured;
      miss : c1 .. c(d) = K, c(d+1) = K + 30 equal bytes: one step too far, so best is the nearest of d equal ones;
      tie  : c1, c2 = K, c3 = K + 15 equal bytes, c4 = K, c5 = K + 15 equal bytes: the nearer of two equal wins.
    Every K candidate is followed by a byte that differs from the target's, and preceded by one that differs from the
    byte before the target.  4000 zeros after each target make its block shrink, so that it is not stored raw."""
    if codec == "zstd":
        mm, depth, _ = zl.params(level)
        block = ZB
    else:
        mm, depth, block = 4, hc.PARAMS[level][0], LB
    rng = np.random.default_rng(800 + level)
    buf = rnd(rng, 4 * block)
    plans = {"take": {1: 0, 2: 1, depth: 30}, "miss": {depth + 1: 30}, "tie": {3: 15, 5: 15}}
    ncand = {"take": depth, "miss": depth + 1, "tie": 5}
    targets = {}
    for t, name in enumerate(("take", "miss", "tie")):
        K, T = rnd(rng, mm), rnd(rng, 64)
        pos = (t + 1) * block + 200
        cand = {}
        for i in range(ncand[name], 0, -1):                   # farthest first
            eq = plans[name].get(i, 0)
            body = np.concatenate([K, T[:eq], [T[eq] ^ 0x80], rnd(rng, 6)]).astype(np.uint8)
            buf[pos] = 0
            buf[pos + 1: pos + 1 + body.size] = body
            cand[i] = pos + 1
            pos += 1 + body.size
        P = pos + 50
        buf[P - 1] = 1                                          # differs from the 0 before every candidate
        buf[P: P + mm] = K
        buf[P + mm: P + mm + 64] = T
        buf[P + mm + 64] ^= 0x11
        buf[P + mm + 200: P + mm + 4200] = 0                    # the block shrinks: its parse is written
        targets[name] = (P, cand)
    want = {"take": (mm + 30, depth), "miss": (mm, 1), "tie": (mm + 15, 3)}

    def check(lv, ev, seqs, best):
        for name, (P, cand) in targets.items():
            ln, c = want[name]
            assert unpack(best[0][P]) == (ln, P - cand[c]), (name, unpack(best[0][P]), (ln, P - cand[c]))
        rows = abs_starts(seqs[0], block)
        for name in ("take", "tie"):
            P, cand = targets[name]
            ln, c = want[name]
            assert [tuple(r) for r in rows[rows[:, 0] == P].tolist()] == [(P, P - cand[c], ln)], name
    return Case("%s_chain_depth_l%d" % (codec, level), codec, (level,), buf, 1 << 20, None, check)


# ------------------------------------------------------------------------------------------------- bit buffer
Z_BITBUF = 3072 * 4                      # the zstd entropy stage's bit buffer (Z_BITWORDS words)


def far_copies(rng, buf, b0, lengths):
    """Back-to-back copies of the given lengths from [40000, 2^20) into buf[b0:]: no literals, every offset in
    (2^20, 2^21) (offset code 20), and each copy exactly its length (the next copy's first byte differs from the byte
    after the source)."""
    p, nxt = b0, None
    for ln in lengths:
        while True:
            s = int(rng.integers(40000, (1 << 20) - 1000))
            if nxt is None or buf[s] != nxt:
                break
        buf[p: p + ln] = buf[s: s + ln]
        nxt = buf[s + ln]
        p += ln
    if p < buf.size and buf[p] == nxt:
        buf[p] ^= 0x55


def zstd_bitbuf():
    """Two 16 KiB blocks of level 6 made of back-to-back far copies (offset code 20, no literals) on both sides of the
    entropy stage's 12 KiB bit buffer: block 128 of 5-byte copies, whose sequence bits overflow it while the compressed
    block would still be smaller than its content (so the twin stores it raw for the overflow alone), and block 129 of
    6- and 7-byte copies whose sequence bits fit, with less than 2 KiB to spare."""
    import _zenc as ze
    rng = np.random.default_rng(900)
    buf = rnd(rng, (1 << 21) + 3 * ZB)
    over = [5] * (ZB // 5 - 1) + [5 + ZB % 5]
    n7 = 1000
    n6 = (ZB - 7 * n7) // 6
    under = [7] * n7 + [6] * n6
    under[-1] += ZB - sum(under)
    rng.shuffle(under)
    far_copies(rng, buf, 1 << 21, over)
    far_copies(rng, buf, (1 << 21) + ZB, under)
    A, B = (1 << 21) // ZB, (1 << 21) // ZB + 1

    def check(level, ev, seqs, best):
        ra, rb = seqs[0][A].astype(np.int64), seqs[0][B].astype(np.int64)
        for rows, plan in ((ra, over), (rb, under)):           # a copy whose source overlaps another's may match nearer
            assert abs(len(rows) - len(plan)) <= 4 and rows[:, 0].sum() <= 4
            assert (rows[:, 1] > (1 << 20)).sum() >= len(plan) - 8
        ta, tb = (ze.block_b200(r, ze.literals_of(buf[k * ZB: (k + 1) * ZB], r), buf[k * ZB: (k + 1) * ZB], False)[1]
                  for k, r in ((A, ra), (B, rb)))
        assert ta.raw_reason == ze.RAW_BITBUF and ta.bsize < ZB
        assert tb.raw_reason == 0 and Z_BITBUF - 2048 < tb.seq_body + 8 <= Z_BITBUF

    def gpu_check(level, rep):
        assert rep.types[A] == 0 and rep.types[B] == 2 and rep.raw_bitbuf == 1
    return Case("zstd_bitbuf", "zstd", (6,), buf, 4 << 20, None, check, gpu_check)


# ------------------------------------------------------------------------------------------------- n - 1 and n
def lz4_exact_sizes():
    """Two chunks of three 64 KiB blocks: block 0 random, block 1 random but for one copy from block 0 whose length is
    tuned so that block 1 encodes to exactly 65535 bytes (chunk 0, written compressed) or exactly 65536 (chunk 1,
    stored raw: the encoding does not shrink it), block 2 copies from block 1 (a raw block is history for the next)."""
    rng = np.random.default_rng(1000)
    chunk = 3 * LB
    buf = rnd(rng, 2 * chunk)
    for c in range(2):
        c0 = c * chunk
        for j in range(20):                                     # block 2: 20 copies of 1000 bytes from block 1
            d = c0 + 2 * LB + 500 + j * 3000
            place(buf, d, d - (c0 + LB + 1000 + j * 3000), 1000)
    tuned = []
    for c, target in enumerate((LB - 1, LB)):
        c0 = c * chunk
        base = buf[c0: c0 + chunk].copy()
        ln, size = 260, None
        for _ in range(40):
            part = base.copy()
            place(part, LB + 100, LB + 100 - 200, ln)
            size = len(hc.encode_block(part[LB: 2 * LB].tobytes(), [tuple(r) for r in hc.twin_sequences(part, 10)[1].tolist()]))
            if size == target:
                break
            ln += size - target
        assert size == target, (c, size, target)
        buf[c0: c0 + chunk] = part
        tuned.append(ln)

    def check(level, ev, seqs, best):
        for c, target in enumerate((LB - 1, LB)):
            blk = buf[c * chunk + LB: c * chunk + 2 * LB].tobytes()
            assert len(hc.encode_block(blk, [tuple(r) for r in seqs[c][1].tolist()])) == target
            rows = abs_starts(seqs[c], LB)
            back = rows[(rows[:, 0] >= 2 * LB)]
            assert len(back) and ((back[:, 0] - back[:, 1] >= LB) & (back[:, 0] - back[:, 1] < 2 * LB)).all()

    def gpu_check(level, rep):
        framed, frames, _ = rep
        assert [[(r, n) for r, n, _ in blocks] for _, _, blocks in frames] == [[(True, LB), (False, LB), (False, LB)],
                                                                               [(True, LB), (True, LB), (False, LB)]]
    return Case("lz4_exact_sizes", "lz4", (10, 12), buf, chunk, None, check, gpu_check)


def cases():
    return [zstd_phases(), zstd_range_ends(), zstd_defer(), zstd_ends(), zstd_offsets(6), zstd_offsets(12),
            zeros_chunks(5, "zstd", (6, 12)), zstd_bitbuf()] + [chain_depth("zstd", lv) for lv in (6, 8, 9, 12)] + \
           [lz4_quarters(), lz4_dense(), lz4_block_ends(), zeros_chunks(4, "lz4", (10, 12)), lz4_defer_ties(),
            lz4_exact_sizes()] + [chain_depth("lz4", lv) for lv in (10, 12)]


def parts(case):
    """The chunk contents of a case."""
    src, chunk = case.src, case.chunk
    if case.chunk_bytes is None:
        return [src[i: i + chunk] for i in range(0, max(src.size, 1), chunk)]
    return [src[c * chunk: c * chunk + int(b)] for c, b in enumerate(case.chunk_bytes)]
