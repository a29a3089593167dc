"""Inputs that drive the zstd encoder's entropy stage (z_encode_block) to its edges, tuned on the CPU with its twin
(_zenc.block_b200) and named by the schedule model (_zentsched.events).

Each Case builds one input from a knob k: make(k) -> (src, chunk, chunk_bytes).  The case's k is found by a search over
a fixed range, with fixed seeds, for the first k whose blocks at the case's level satisfy the predicate; `knock` is the
knob value that removes the edge (a neighbour, or the construction without its key ingredient), where the predicate
must fail (knock None: the first knob value of the range that misses the edge).  Levels: 3 (the level-3 class: 64 KiB
windows cut into sub-blocks) or 9 (the search class: 16 KiB blocks).  Every case's input also goes through level 3 on the GPU; the cases built at level 9 go through level 9 as well."""
import numpy as np

import _zenc as ze
import _zentsched as zs

ZB = 16384


class Case:
    def __init__(self, name, level, make, ks, pred, knock, doc):
        self.name, self.level, self.make, self.ks, self.pred, self.knock_of, self.doc = name, level, make, ks, pred, knock, doc
        self._k = None

    def events(self, k):
        src, chunk, cb = self.make(k)
        out = []
        for c, content in enumerate(ze.chunks(src, chunk, cb)):
            out += [(c, b, ev) for b, ev in zs.chunk_events(content, self.level)]
        return out

    def reaches(self, k):
        return bool(self.pred([ev for _, _, ev in self.events(k)]))

    @property
    def k(self):
        if self._k is None:
            for k in (self.ks() if callable(self.ks) else self.ks):
                if self.reaches(k):
                    self._k = k
                    break
            else:
                raise AssertionError("no knob value reaches %s" % self.name)
        return self._k

    def built(self):
        return self.make(self.k)

    def knock(self):
        if self.knock_of is not None:
            return self.knock_of(self.k)
        for k in (self.ks() if callable(self.ks) else self.ks):
            if not self.reaches(k):
                return k
        raise AssertionError("every knob value reaches %s" % self.name)

    def knocked(self):
        return self.make(self.knock())


def rnd(rng, n, hi=256):
    return rng.integers(0, hi, n, dtype=np.uint8)


def one(evs, **want):
    """Some block has every field of `want` (a value, or a predicate)."""
    return any(all((v(ev.get(f)) if callable(v) else ev.get(f) == v) for f, v in want.items()) for ev in evs)


# ------------------------------------------------------------------------------------------------- block size
def copy_block(seed, L):
    """3000 random bytes with one copy of L bytes (source 1900 bytes back): raw literals and one sequence, so the
    compressed size falls by one byte per byte of L."""
    rng = np.random.default_rng(seed)
    x = rnd(rng, 3000)
    x[2000: 2000 + L] = x[100: 100 + L]
    x[2000 + L] = x[100 + L] ^ 0x5A
    x[1999] = x[99] ^ 0xA5
    return x, 1 << 20, None


def size_cases(level):
    mk = lambda L: copy_block(40 + level, L)
    return [
        Case("bsize_regen_minus1_L%d" % level, level, mk, range(4, 40),
             lambda e: any(ev["bsize"] == ev["regen"] - 1 and not ev["raw_reason"] for ev in e),
             lambda k: k - 1, "bsize == regen - 1: compressed"),
        Case("bsize_regen_L%d" % level, level, mk, range(4, 40),
             lambda e: any(ev["bsize"] == ev["regen"] and ev["raw_reason"] == ze.RAW_SIZE for ev in e),
             lambda k: k + 1, "bsize == regen: raw"),
    ]


# ------------------------------------------------------------------------------------------------- literal estimate
def alpha_block(seed, n, A, tail=2000):
    """n random literals over 0..A-1, then `tail` zeros (one long match): one compressed block whose literal section
    is about n bytes at log2(A) bits each."""
    rng = np.random.default_rng(seed)
    return np.concatenate([rnd(rng, n, A), np.zeros(tail, np.uint8)]), 1 << 20, None


def est_cases(level):
    mk = lambda n: alpha_block(50 + level, n, 128)
    huf = lambda e: any(ev["est"] == ev["nlit"] - 1 and ev["lit_mode"] == 2 and not ev["raw_reason"] for ev in e)
    raw = lambda e: any(ev["est"] == ev["nlit"] and ev["lit_reason"] == ze.LIT_EST and not ev["raw_reason"] for ev in e)
    return [
        Case("est_nlit_minus1_L%d" % level, level, mk, range(500, 900), huf, lambda k: k - 40, "est == nlit - 1: Huffman"),
        Case("est_nlit_L%d" % level, level, mk, range(500, 900), raw, lambda k: k + 40, "est == nlit: raw literals"),
    ]


def huf_bitbuf_block(seed, L):
    """One 16 KiB block of random literals over 0..63 (6 bits each) with one copy of L bytes: the Huffman estimate lands
    on the 12 KiB bit buffer as L varies."""
    rng = np.random.default_rng(seed)
    x = rnd(rng, ZB, 64)
    x[ZB - 200 - L: ZB - 200] = x[1000: 1000 + L]
    x[ZB - 200] = (x[1000 + L] + 1) % 64
    x[ZB - 201 - L] = (x[999] + 1) % 64
    return x, 1 << 20, None


def huf_bitbuf_cases():
    mk = lambda L: huf_bitbuf_block(60, L)
    return [
        Case("huf_bitbuf_12288", 9, mk, range(20, 400),
             lambda e: any(ev["est"] + 64 == 12288 and ev["lit_mode"] == 2 and not ev["raw_reason"] for ev in e),
             lambda k: k - 1, "est + 64 == 12288: Huffman"),
        Case("huf_bitbuf_12289", 9, mk, range(20, 400),
             lambda e: any(ev["est"] + 64 == 12289 and ev["lit_reason"] == ze.LIT_BITBUF and not ev["raw_reason"] for ev in e),
             lambda k: k + 1, "est + 64 == 12289: raw literals"),
    ]


# ------------------------------------------------------------------------------------------------- sequence bit buffer
def far_block(seed, near):
    """Level 9: 2 MiB of random history, then one 16 KiB block of back-to-back far copies (5- and 6-byte, sources
    2^20 .. 2^21 back: offset code 20); the first `near` copies take their sources 2^19 .. 2^20 back (offset code 19,
    one bit less each), which moves the sequence bits across the bit buffer one bit at a time.
    Level 3 was tried first and does not get there: a level-3 sequence carries at most 28 bits (literal length 0,
    match length 4, offset below 64 KiB), so the buffer needs about 3,500 far matches in one 16 KiB sub-block, each
    still in its slot of the 4096-entry hash table, which every position of the window overwrites.  32 KiB of
    back-to-back 4-, 5- and 6-byte copies from random sources in the window's first half gave at most 439 sequences
    and a 1530-byte seq_body per sub-block (DESIGN §4)."""
    rng = np.random.default_rng(seed)
    H = 1 << 21
    buf = rnd(rng, H + ZB)
    lens = [6] * 1500 + [5] * ((ZB - 9000) // 5)
    lens[-1] += ZB - sum(lens)
    rng.shuffle(lens)
    p, nxt = H, None
    for i, ln in enumerate(lens):
        lo, hi = ((1 << 19) + 64, (1 << 20) - 64) if i < near else ((1 << 20) + 64, (1 << 21) - 64)
        while True:
            s = p - int(rng.integers(lo, hi))
            if nxt is None or buf[s] != nxt:
                break
        buf[p: p + ln] = buf[s: s + ln]
        nxt = buf[s + ln]
        p += ln
    return buf, 4 << 20, None


def seq_bitbuf_cases():
    mk = lambda k: far_block(70, k)
    fit = lambda e: any(ev["seq_body"] + 8 == 12288 and not ev["raw_reason"] for ev in e)
    over = lambda e: any(ev["seq_body"] + 8 == 12289 and ev["raw_reason"] == ze.RAW_BITBUF for ev in e)
    return [
        Case("seq_bitbuf_12288", 9, mk, _seq_ks, fit, lambda k: k - 8, "seq_body + 8 == 12288: compressed"),
        Case("seq_bitbuf_12289", 9, mk, _seq_ks, over, lambda k: k + 8, "seq_body + 8 == 12289: raw (bit buffer)"),
    ]


def _seq_ks():
    """Knob values for the far-copy block, nearest the buffer first: the number of copies at offset code 19 that would
    bring the sequence bits of the block to the buffer (one bit each), then its neighbours."""
    src, chunk, _ = far_block(70, 0)
    rows, lits, raw, last = ze.chunk_blocks(src[: (1 << 21) + ZB], 9)[-1]
    body = ze.block_b200(rows, lits, raw, last)[1].seq_body
    k0 = max(0, (body + 8 - 12288) * 8)
    order = [k0]
    for d in range(1, 40):
        order += [k0 + 4 * d, max(0, k0 - 4 * d)]
    return order


# ------------------------------------------------------------------------------------------------- FSE chains
def runs_block(seed, n, gap=24):
    """n runs of 8 equal bytes in random data, one every `gap` bytes: n sequences (literal length gap - 8, offset 1,
    match length 7) in one sub-block."""
    rng = np.random.default_rng(seed)
    x = rnd(rng, n * gap + 64)
    for j in range(n):
        p = 32 + j * gap
        x[p: p + 8] = x[p - 1] ^ 0x55
    return x, 1 << 20, None


def norepeat(rng, n, bits=2):
    """n literals without a repeated 4-gram: groups (x, x', counter high, counter low), x of `bits` random bits."""
    g = np.arange((n + 3) // 4)
    x = rnd(rng, 2 * g.size, 1 << bits)
    return np.stack([x[0::2], x[1::2], (64 + (g >> 8)).astype(np.uint8), (g & 255).astype(np.uint8)], axis=1).reshape(-1)[:n]


def nseq_cases():
    out = [Case("nseq1", 3, lambda k: copy_block(41, k), range(20, 30), lambda e: one(e, nseq=1, raw_reason=0),
                lambda k: 0, "nseq 1")]
    for n in (2, 31, 32, 33, 512, 513):
        extra = {33: dict(lanes_busy=17), 512: dict(lanes_exact=2), 513: dict(lanes_exact=1)}.get(n, {})
        ms = range(n - 2, n + 3) if n < 100 else range(int(n * 0.85), n + 3)        # a run can take two sequences
        out.append(Case("nseq%d" % n, 3, lambda k: runs_block(80 + k // 1000, k % 1000), [s * 1000 + m for s in range(4) for m in ms],
                        lambda e, n=n, extra=extra: one(e, nseq=n, raw_reason=0, **extra),
                        lambda k: k - 1 if n == 512 else k + 1, "nseq %d" % n))
    return out


def token_block(seed, ntok, tlen, n=ZB):
    """Tokens of tlen bytes from a dictionary of ntok, back to back: runs of short sequences with literal length 0 and
    match length tlen, the symbols of normalised count 4 (LL code 0) or 3 (ML codes 1-2) whose state chains can keep
    two different states for many steps, so the warp's warm-up guesses wrong."""
    rng = np.random.default_rng(seed)
    toks = [rnd(rng, tlen) for _ in range(ntok)]
    out = [rnd(rng, 64)]
    size = 64
    while size < n:
        t = toks[int(rng.integers(0, ntok))]
        out.append(t); size += t.size
    return np.concatenate(out)[:n], 1 << 20, None


def chain_cases():
    """The speculative chains of the LL stream on runs every 120 bytes (literal length code 25, normalised count 3),
    those of the ML stream on back-to-back tokens.  The knock-out: 130 runs every 40 bytes, where every guess is right."""
    out = []
    for stream in ("LL", "ML"):
        for what, f in (("wrong", lambda ev, s: ev.get("spec_wrong_" + s, 0) > 0),
                        ("rounds2", lambda ev, s: ev.get("repair_rounds_" + s, 0) >= 2),
                        ("rerun_from_wrong", lambda ev, s: ev.get("rerun_from_wrong_" + s, 0) > 0 and ev.get("rerun_twice_" + s, 0) > 0)):
            mk = token_or_runs if stream == "ML" else (lambda k: runs_block(200 + k, 130, 120) if k >= 0 else runs_block(80, 130, 40))
            out.append(Case("chain_%s_%s" % (stream, what), 3, mk, range(0, 40),
                            lambda e, f=f, s=stream: any(f(ev, s) for ev in e),
                            lambda k: -1, "%s chain: %s" % (stream, what)))
    for what, f in (("wrong", lambda ev: ev.get("spec_wrong_OF", 0) > 0),
                    ("rounds31", lambda ev: ev.get("repair_rounds_OF", 0) == 31)):
        out.append(Case("chain_OF_%s" % what, 9, lambda k: of_run_block(170 + abs(k), 700, far=k >= 0), range(0, 10),
                        lambda e, f=f: any(f(ev) for ev in e), lambda k: -1 - k, "OF chain: %s" % what))
    return out


def of_run_block(seed, R, far=True):
    """Level 9: R pieces of 6 random literals and a 5-byte copy of the literals of the piece 6 back (offset 72, offset
    code 6), then (far) an 8-byte copy from 1500 back (offset code 10).  Offset code 6 has count 2 in the 32-cell OF
    table, at cells 1 and 24, so encoding it from a cell below 16 lands on cell 1 and from 16 or above on cell 24; code
    10's one cell is 25.  The far copy, encoded first, puts the serial chain at cell 25, and it stays at 24 through the
    whole run, while every lane's warm-up starts at init_state(6) = cell 1 and stays there: all 31 speculative lanes
    guess wrong, and the repair fixes one lane per round.  Without the far copy the serial chain sits at cell 1 too."""
    rng = np.random.default_rng(seed)
    x = rnd(rng, ZB)
    B = 200
    for i in range(6, R):
        P, S = B + 11 * i, B + 11 * (i - 6)
        x[P + 6: P + 11] = x[S: S + 5]
        if x[P + 5] == x[S - 1]:
            x[P + 5] ^= 0x5A
        if x[P + 11] == x[S + 5]:
            x[P + 11] ^= 0x5A
    p = B + 11 * R + 6
    if far:
        x[p: p + 8] = x[p - 1500: p + 8 - 1500]
        if x[p + 8] == x[p + 8 - 1500]:
            x[p + 8] ^= 0x5A
    return x, 1 << 20, None


def token_or_runs(k):
    """token_block for k >= 0; the knock-out (k < 0): 130 runs every 40 bytes, where every guess is right."""
    return token_block(90 + k, 40 + k % 5 * 10, 4 + k % 2) if k >= 0 else runs_block(80, 130, 40)


# ------------------------------------------------------------------------------------------------- Huffman placement
def huf_block(seed, n, A=16):
    """n random literals over 0..A-1 then 2000 zeros: a Huffman-coded literal section of about n literals."""
    return alpha_block(seed, n, A)


def huffman_cases():
    out = []
    for r in range(4):
        out.append(Case("huf_nlit_mod4_%d" % r, 3, lambda k: huf_block(100, k), range(200, 240),
                        lambda e, r=r: one(e, lit_mode=2, raw_reason=0, huf_nlit_mod4=r), lambda k: k + 1, "nlit = %d mod 4" % r))
    out.append(Case("huf_short_stream", 3, lambda k: huf_block(101, k), range(64, 200),
                    lambda e: one(e, lit_mode=2, raw_reason=0, huf_empty_runs=lambda v: v and v > 0,
                                  huf_min_stream_lits=lambda v: v is not None and v < 56), lambda k: 400, "a stream under 56 literals"))
    out.append(Case("huf_bits_mod8_0", 3, lambda k: huf_block(102 + k, 300), range(0, 60),
                    lambda e: one(e, lit_mode=2, raw_reason=0, huf_bits_mod8_0=lambda v: v and v > 0), None,
                    "a stream of 0 mod 8 bits"))
    out.append(Case("huf_bits_mod32_31", 3, lambda k: huf_block(103 + k, 300), range(0, 200),
                    lambda e: one(e, lit_mode=2, raw_reason=0, huf_bits_mod32_31=lambda v: v and v > 0), None,
                    "a stream of 31 mod 32 bits"))
    return out


def fib_block(seed, n):
    """n literals with Fibonacci counts over 17 symbols (a tree deeper than 11: 11-bit codes) and no repeated 4-gram,
    then zeros."""
    rng = np.random.default_rng(seed)
    fib = [1, 1]
    while len(fib) < 17:
        fib.append(fib[-1] + fib[-2])
    x = np.repeat(np.arange(1, 18, dtype=np.uint8), fib)
    g = np.arange(n // 4 + 1)
    x = rng.permutation(np.concatenate([x, np.full(max(0, 2 * g.size - x.size), 17, np.uint8)]))[: 2 * g.size]
    lits = np.stack([x[0::2], x[1::2], (32 + (g >> 7) % 64).astype(np.uint8), (128 + (g & 127)).astype(np.uint8)], axis=1).reshape(-1)[:n]
    return np.concatenate([lits, np.zeros(2000, np.uint8)]), 1 << 20, None


def noform_block(seed, bump):
    """Symbols 0..191 ten times each and symbol 192 640 times, permuted, then zeros.  The tree gives the 192 symbols
    length 8 and symbol 192 length 2 (maxbits 8), so all 192 listed weights are 1: the FSE form of the weights has
    nothing to code (z_fse_weights returns 0), direct weights cannot list 192 symbols, and the literals go raw although
    Huffman would pay.  bump > 0: symbol 5 occurs bump more times, its weight differs and the FSE form exists."""
    rng = np.random.default_rng(seed)
    x = np.concatenate([np.repeat(np.arange(192, dtype=np.uint8), 10), np.full(640, 192, np.uint8), np.full(bump, 5, np.uint8)])
    return np.concatenate([rng.permutation(x), np.zeros(2000, np.uint8)]), 1 << 20, None


def tree_cases():
    out = [Case("huf_noform", 3, lambda k: noform_block(160 + k // 100, k % 100), range(0, 300, 100),
                lambda e: any(ev["lit_reason"] == ze.LIT_NOFORM and ev["lit_mode"] == 0 and ev["est"] < ev["nlit"]
                              and not ev["raw_reason"] for ev in e),
                lambda k: k + 10, "no weight description although Huffman pays: raw literals"),
           Case("huf_straddle11", 3, lambda k: fib_block(110 + k, 14000), range(0, 30),
                lambda e: one(e, lit_mode=2, raw_reason=0, huf_straddle11_shared=lambda v: v and v > 0), None,
                "an 11-bit code across a word two runs share")]
    for top in (127, 128):                                          # direct weights: maxsym odd / even
        out.append(Case("direct_maxsym%d" % top, 3, lambda k, top=top: _top_block(120 + k, top if k >= 0 else top - 1), range(0, 20),
                        lambda e, top=top: one(e, lit_mode=2, raw_reason=0, maxsym=top, wdesc_len=0), lambda k: -1 - k,
                        "direct weights, maxsym %d" % top))
    for top in (201, 202):                                          # FSE-coded weights: odd / even weight count
        out.append(Case("fse_weights_%d" % top, 3, lambda k, top=top: _top_block(130 + k, top if k >= 0 else 128, skew=True), range(0, 20),
                        lambda e, top=top: one(e, lit_mode=2, raw_reason=0, maxsym=top, wdesc_len=lambda v: v and v > 0), lambda k: -1 - k,
                        "FSE-coded weights, %d weights" % top))
    return out


def _top_block(seed, top, skew=False, n=3000):
    """n literals over 0..top (top present), the lower half four times as frequent with skew; then zeros."""
    rng = np.random.default_rng(abs(seed))
    p = np.ones(top + 1)
    if skew:
        p[: (top + 1) // 2] = 4
    x = rng.choice(top + 1, n, p=p / p.sum()).astype(np.uint8)
    x[n // 2] = top
    return np.concatenate([x, np.zeros(2000, np.uint8)]), 1 << 20, None


# ------------------------------------------------------------------------------------------------- sequences
def nseq0_block(seed, n):
    """n literals without a repeated 4-gram and zeros to 20 KiB: the cut at 16 KiB falls at the zeros' match, so the
    first sub-block holds the literals alone (a compressed block without sequences).  n = 0: 4 KiB only, no cut."""
    rng = np.random.default_rng(seed)
    if n == 0:
        return np.concatenate([norepeat(rng, 1000), np.zeros(3000, np.uint8)]), 1 << 20, None
    return np.concatenate([norepeat(rng, n), np.zeros(20480 - n, np.uint8)]), 1 << 20, None


def ll_block(seed, lls):
    """Level 9: a first 16 KiB block of 12-byte strings, then one sequence per literal length in lls: lls[i] random
    literals and a copy of the next string.  The boundaries go up to 8192: a 16 KiB block cannot hold 16384 literals
    and a match (long_ll_window reaches the longer ones at level 3).  The pieces are packed into 16 KiB blocks, none across a block boundary,
    so each literal length is counted from the end of the previous copy or from the block's start."""
    rng = np.random.default_rng(seed)
    strs = rnd(rng, ZB)
    blocks, cur, i = [strs], [], 0
    for ll in lls:
        piece = np.concatenate([rnd(rng, ll), strs[12 * i: 12 * i + 12]])
        i += 1
        if sum(x.size for x in cur) + piece.size > ZB - 16:
            blocks.append(np.concatenate(cur + [rnd(rng, ZB - sum(x.size for x in cur))]))
            cur = []
        cur.append(piece)
    if cur:
        blocks.append(np.concatenate(cur + [rnd(rng, ZB - sum(x.size for x in cur))]))
    return np.concatenate(blocks), 1 << 20, None


def long_ll_window(seed, ll, d):
    """Level 3: one 64 KiB window with a literal run of ll bytes.  A run of zeros across the 16 KiB mark is the match
    pending there, so no later mark cuts the sub-block before another match starts; then ll random literals, a 12-byte
    copy of the run's own bytes d back, and zeros before the next mark (so the cut falls after the copy, which keeps its
    literal run).  The source must still be in its hash-table slot when the copy is parsed: at d = 400 it is, at
    d = 200 it is not (same candidate round), and the copy stays literals."""
    rng = np.random.default_rng(seed)
    x = rnd(rng, 1 << 16)
    x[15000:16600] = 0
    q = 16600 + ll
    x[q: q + 12] = x[q - d: q - d + 12]
    if x[q + 12] == x[q - d + 12]:
        x[q + 12] ^= 0x5A
    x[q + 100: q + 400] = 0
    return x


LONG_LL = (16383, 16384, 32767, 32768)


LL_BOUNDS = [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192]


def seq_cases():
    lls = sorted({v for b in LL_BOUNDS for v in (b - 1, b)})
    return [
        Case("nseq0_compressed", 3, lambda k: nseq0_block(140, k), range(15000, 16300, 97),
             lambda e: one(e, nseq=0, raw_reason=0, lit_mode=2), lambda k: 0, "a compressed block without sequences"),
        Case("ll_codes_long", 3, lambda k: (np.concatenate([long_ll_window(7, ll, k) for ll in LONG_LL]), 1 << 20, None),
             [400, 500, 700], lambda e: set(LONG_LL) <= set(r for ev in e for r in ev.get("lls", ())), lambda k: 200,
             "both sides of literal-length codes 33 and 34 (16384, 32768) at level 3"),
        Case("ll_codes", 9, lambda k: ll_block(150, lls) if k else ll_block(150, []), [1],
             lambda e: {b - 1 for b in LL_BOUNDS} | set(LL_BOUNDS) <= set(r for ev in e for r in ev.get("lls", ())),
             lambda k: 0, "both sides of every literal-length code boundary a 16 KiB block allows"),
    ]


def cases():
    out = []
    out += size_cases(3) + size_cases(9) + est_cases(3)
    out += huf_bitbuf_cases() + seq_bitbuf_cases() + nseq_cases() + chain_cases() + huffman_cases() + tree_cases() + seq_cases()
    return out
