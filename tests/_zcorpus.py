"""A corpus of zstd frames at the edges of the format, written by libzstd itself from parses the tests dictate.

Every frame is produced by the image's libzstd (libzstd.so.1) through ZSTD_compressSequences: the test chooses the
sequences (literal length, offset, match length), builds the source those sequences describe (build_from_seqs), and
libzstd chooses everything else — block splits, literal and table modes, repeat-offset codes, Huffman and FSE tables.
Content and parse agree by construction, and nothing is hand-encoded.  Each case names the edge it exists for as a
predicate on the oracle's block trace (orc_zstd_trace); the CPU tests assert that it holds.

`reference_ultra` is the exception: its parse is libzstd's own (level 3, long-distance matching) on data that repeats
more than 32 MiB apart."""
import ctypes
import functools

import numpy as np
import pytest

import _oracle as o

c_sz, c_vp, c_int = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int

# ZSTD_cParameter ids.  The stable ones are fixed by zstd.h; the experimental ones are checked through their bounds below.
P_LEVEL, P_WINDOWLOG, P_LDM = 100, 101, 160
P_CHECKSUM = 201
P_LITMODE, P_MAXBLOCK = 1002, 1015                 # ZSTD_c_literalCompressionMode, ZSTD_c_maxBlockSize (experimental)
EXPECT_BOUNDS = {P_LITMODE: (0, 2), P_MAXBLOCK: (1024, 131072)}


class _Bounds(ctypes.Structure):
    _fields_ = [("error", c_sz), ("lowerBound", c_int), ("upperBound", c_int)]


class Seq(ctypes.Structure):
    """ZSTD_Sequence: offset is the real distance (0 with matchLength 0 for trailing literals); rep is ignored on input."""
    _fields_ = [("offset", ctypes.c_uint), ("litLength", ctypes.c_uint), ("matchLength", ctypes.c_uint), ("rep", ctypes.c_uint)]


def _err(r):
    return r > (1 << 63)


@functools.lru_cache(maxsize=None)
def zstd():
    """libzstd.so.1 with the entry points the corpus uses (the test module skips when it is absent)."""
    try:
        L = ctypes.CDLL("libzstd.so.1")
    except OSError:
        pytest.skip("libzstd.so.1 not present")
    L.ZSTD_versionNumber.restype = ctypes.c_uint
    L.ZSTD_createCCtx.restype = c_vp
    L.ZSTD_freeCCtx.argtypes = [c_vp]
    L.ZSTD_CCtx_setParameter.restype = c_sz; L.ZSTD_CCtx_setParameter.argtypes = [c_vp, c_int, c_int]
    L.ZSTD_cParam_getBounds.restype = _Bounds; L.ZSTD_cParam_getBounds.argtypes = [c_int]
    L.ZSTD_compressBound.restype = c_sz; L.ZSTD_compressBound.argtypes = [c_sz]
    L.ZSTD_compressSequences.restype = c_sz
    L.ZSTD_compressSequences.argtypes = [c_vp, c_vp, c_sz, ctypes.POINTER(Seq), c_sz, c_vp, c_sz]
    L.ZSTD_compress2.restype = c_sz; L.ZSTD_compress2.argtypes = [c_vp, c_vp, c_sz, c_vp, c_sz]
    L.ZSTD_decompress.restype = c_sz; L.ZSTD_decompress.argtypes = [c_vp, c_sz, c_vp, c_sz]
    for pid, want in EXPECT_BOUNDS.items():
        b = L.ZSTD_cParam_getBounds(pid)
        got = (b.lowerBound, b.upperBound)
        if _err(b.error) or got != want:
            raise RuntimeError("libzstd %d: parameter %d has bounds %s, expected %s; the experimental ids differ in this version"
                               % (L.ZSTD_versionNumber(), pid, got, want))
    return L


def compress(src, params, seqs=None):
    """One zstd frame of `src`: ZSTD_compressSequences with the parse `seqs` ((ll, off, ml) rows), or ZSTD_compress2 (libzstd's
    own parser) when seqs is None.  params: {parameter id: value}."""
    L = zstd()
    src = np.ascontiguousarray(src, dtype=np.uint8)
    cctx = L.ZSTD_createCCtx()
    try:
        for k, v in params.items():
            r = L.ZSTD_CCtx_setParameter(cctx, k, v)
            assert not _err(r), (k, v)
        cap = L.ZSTD_compressBound(src.size) + (1 << 16)
        out = np.empty(cap, np.uint8)
        if seqs is None:
            n = L.ZSTD_compress2(cctx, out.ctypes.data, cap, src.ctypes.data, src.size)
        else:
            a = np.asarray(seqs, dtype=np.int64).reshape(-1, 3)
            arr = (Seq * max(1, len(a)))()
            view = np.frombuffer(arr, dtype=np.uint32).reshape(-1, 4)
            view[: len(a), 0] = a[:, 1]; view[: len(a), 1] = a[:, 0]; view[: len(a), 2] = a[:, 2]; view[:, 3] = 0
            n = L.ZSTD_compressSequences(cctx, out.ctypes.data, cap, arr, len(a), src.ctypes.data, src.size)
        assert not _err(n), "libzstd refused the frame (error %d)" % (n - (1 << 64))
        return out[:n].copy()
    finally:
        L.ZSTD_freeCCtx(cctx)


def libzstd_decompress(frame, size):
    L = zstd()
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    out = np.empty(size + 1, np.uint8)
    n = L.ZSTD_decompress(out.ctypes.data, out.size, frame.ctypes.data, frame.size)
    assert not _err(n), "ZSTD_decompress failed (error %d)" % (n - (1 << 64))
    return out[:n]


RANDOM = bytes(range(256))


def build_from_seqs(seqs, tail, literal_alphabet, rng):
    """The source the parse describes: for every (ll, off, ml), ll literals drawn uniformly from `literal_alphabet`, then ml
    bytes copied from `off` back; then `tail` more literals.  literal_alphabet is one byte string for all literals, or a list
    of them: one per sequence, then one for the tail.  An offset reaching before the start of the source is an error."""
    seqs = np.asarray(seqs, dtype=np.int64).reshape(-1, 3)
    total = int(seqs[:, 0].sum() + seqs[:, 2].sum()) + int(tail)
    out = np.empty(total, np.uint8)
    per = isinstance(literal_alphabet, list)
    if per and len(literal_alphabet) != len(seqs) + 1:
        raise ValueError("one alphabet per sequence and one for the tail")
    alphas = {}

    def lits(i, n):
        a = literal_alphabet[i] if per else literal_alphabet
        if a not in alphas:
            alphas[a] = np.frombuffer(bytes(a), np.uint8)
        return alphas[a][rng.integers(0, len(a), n)]

    p = 0
    for i, (ll, off, ml) in enumerate(seqs.tolist()):
        if ll:
            out[p: p + ll] = lits(i, ll); p += ll
        if ml:
            if not 0 < off <= p:
                raise ValueError("offset %d at position %d reaches before the source" % (off, p))
            s = p - off
            if off >= ml:
                out[p: p + ml] = out[s: s + ml]
            else:                                        # overlapping copy: the period repeats
                out[p: p + ml] = np.resize(out[s: p], ml)
            p += ml
    if tail:
        out[p: p + tail] = lits(len(seqs), tail)
    return out


# ---------------------------------------------------------------------------------------------------------------- trace helpers
ZT = o.ZT


def modes(tr):
    """(nblocks, 3) Compression_Modes fields LL, OF, ML per block; -1 where the block has no sequences section."""
    m = tr.col("modes").astype(np.int64)
    out = np.stack([(m >> 6) & 3, (m >> 4) & 3, (m >> 2) & 3], 1)
    out[(m < 0) | (tr.col("nseq") <= 0)] = -1
    return out


def of_codes(tr):
    """Offset_Value codes (floor(log2(Offset_Value))) of every sequence."""
    return np.floor(np.log2(tr.seq[:, 1].astype(np.float64))).astype(np.int64) if len(tr.seq) else np.zeros(0, np.int64)


def seq_blocks(tr):
    """Block index of every sequence of the trace."""
    idx = np.empty(len(tr.seq), np.int64)
    for b in range(len(tr.blk)):
        a, n = int(tr.blk[b, ZT["seq_first"]]), int(tr.blk[b, ZT["nseq"]])
        if a >= 0 and n > 0:
            idx[a: a + n] = b
    return idx


def match_block_distance(tr):
    """Per sequence: how many blocks back the first byte of its match source lies."""
    start = np.concatenate([[0], np.cumsum(tr.col("regen").astype(np.int64))])
    sb = seq_blocks(tr)
    dist = np.zeros(len(tr.seq), np.int64)
    for b in np.unique(sb):
        sel = np.flatnonzero(sb == b)
        q = tr.seq[sel].astype(np.int64)
        lits = np.cumsum(q[:, 0]); mls = np.concatenate([[0], np.cumsum(q[:, 2])[:-1]])
        mpos = start[b] + lits + mls                                     # first byte of each match's destination
        src = mpos - q[:, 3]
        dist[sel] = b - (np.searchsorted(start, src, side="right") - 1)
    return dist


# ---------------------------------------------------------------------------------------------------------------- the cases
MiB = 1 << 20


def _dense():
    """32,768 sequences of 1 literal + a 3-byte match in the first 128 KiB block: a 3-byte Number_of_Sequences."""
    rng = np.random.default_rng(101)
    n = 40000
    seqs = np.stack([np.ones(n, np.int64), rng.integers(4, 2000, n), np.full(n, 3)], 1)
    seqs[:, 1] = np.minimum(seqs[:, 1], np.arange(n) * 4 + 1)          # no match reaches before the start
    src = build_from_seqs(seqs, 100, b"abcdefghijklmnop", rng)
    return src, seqs, {P_LEVEL: 3}


def _far_parse(rng, lead, lead_ll, far, pick_off):
    """`lead` bytes of literals (runs drawn from lead_ll) with short matches, one run of a single byte up to `far`, then far
    matches (offsets from pick_off(position, length)) until 1 MiB past `far`.  No offset repeats one of the three before
    it, so libzstd writes no repeat-offset codes."""
    seqs, last = [], [1, 4, 8]                                         # the initial repeat offsets

    def put(ll, off, ml, pos):
        while off in last:
            off = pick_off(pos, ml) if pos >= far else off - 1
        seqs.append((ll, off, ml)); last[:] = [off, last[0], last[1]]
    p = 0
    while p < lead:                                                     # the region the far matches copy from
        ll, ml = int(rng.choice(lead_ll)), int(rng.integers(4, 40))
        put(ll, int(rng.integers(8, p + ll + 1)), ml, p + ll); p += ll + ml
    for _ in range(3):                                                  # three fresh offsets, so that the run's offset 1
        put(4, int(rng.integers(100, 5000)), 8, p + 4); p += 12         #  is no repeat offset (raw blocks keep the history)
    put(1, 1, far - p - 1, p + 1); p = far                              # a run of one byte: RLE blocks
    while p < far + MiB:
        ll, ml = int(rng.integers(1, 300)), int(rng.integers(3000, 20000))
        put(ll, pick_off(p + ll, ml), ml, p + ll); p += ll + ml
    return np.array(seqs, np.int64)


def _far():
    """Matches 16-33 MiB back (Offset_Value codes 24 and 25) in described-table blocks, windowLog 27, content checksum."""
    rng = np.random.default_rng(202)
    lead = MiB

    def pick(pos, ml):
        lo, hi = max(16 * MiB, pos - lead + 1), min(33 * MiB, pos - ml)
        return int(rng.integers(lo, hi + 1)) if rng.random() < 0.6 else int(rng.integers(max(lo, 32 * MiB - 3), hi + 1))
    seqs = _far_parse(rng, lead, np.arange(20, 200), 32 * MiB + 256 * 1024, pick)
    src = build_from_seqs(seqs, 64, b"ETAOINSHRD", rng)
    return src, seqs, {P_LEVEL: 19, P_WINDOWLOG: 27, P_CHECKSUM: 1}


def _far_predef():
    """Far matches (Offset_Value codes 24 and 25, alternating so that no block has a single offset code) in blocks whose
    three tables are the predefined ones, in a frame with no other inter-block state: the lane-per-block sequence decoder
    must hand such a block to the general path."""
    rng = np.random.default_rng(303)
    turn = [0]

    def pick(pos, ml):
        turn[0] ^= 1
        if turn[0]:
            return int(rng.integers(32 * MiB, min(33 * MiB, pos - ml) + 1))
        return int(rng.integers(16 * MiB, 32 * MiB - 4))
    # long literal runs of varied length codes: about 20 sequences per 128 KiB block, so libzstd keeps the predefined tables
    seqs = _far_parse(rng, MiB, np.concatenate([np.arange(30, 300), np.arange(2000, 12000, 7)]), 32 * MiB + 256 * 1024, pick)
    src = build_from_seqs(seqs, 64, b"ETAOINSHRD", rng)
    return src, seqs, {P_LEVEL: 1, P_WINDOWLOG: 27, P_LITMODE: 2}


class Blocks:
    """A parse laid out block by block, for frames cut into blocks of `bsize` bytes (ZSTD_c_maxBlockSize).  add(kind) fills
    the next block with sequences kind(rng, pos) -> (ll, off, ml, alphabet) (pos: where the sequence's literals start) until
    the next one would not fit; the rest of the block is literals carried into the next sequence, which libzstd splits
    at the block boundary.  raw(n) adds n blocks of random literals, which libzstd stores as raw blocks."""

    def __init__(self, rng, bsize):
        self.rng, self.bsize, self.seqs, self.alpha = rng, bsize, [], []
        self.pos, self.carry, self.carry_random = 0, 0, False

    def add(self, kind, n=1, stretch=False):
        """stretch: the block's last match is lengthened to the block end instead (no literals carried over)."""
        for _ in range(n):
            end, first = self.pos + self.bsize, len(self.seqs)
            while True:
                ll, off, ml, alpha = kind(self.rng, self.pos)
                if self.pos + ll + ml > end:
                    break
                assert 0 < off <= self.pos + ll
                self.seqs.append((self.carry + ll, off, ml)); self.alpha.append(RANDOM if self.carry_random else alpha)
                self.carry, self.carry_random = 0, False
                self.pos += ll + ml
            if stretch and len(self.seqs) > first:
                ll, off, ml = self.seqs[-1]; self.seqs[-1] = (ll, off, ml + end - self.pos)
            else:
                self.carry += end - self.pos
            self.pos = end
        return self

    def raw(self, n=1):
        self.carry += n * self.bsize; self.pos += n * self.bsize; self.carry_random = True
        return self

    def build(self, params):
        seqs = np.array(self.seqs, np.int64).reshape(-1, 3)
        src = build_from_seqs(seqs, self.carry, self.alpha + [RANDOM], self.rng)
        return src, seqs, {**params, P_MAXBLOCK: self.bsize}


def _new_off(rng, pos, lo, hi, avoid=()):
    """An offset in [lo, hi] that reaches no further back than pos and is none of `avoid`."""
    while True:
        off = int(rng.integers(lo, max(lo, min(hi, pos)) + 1))
        if off <= pos and off not in avoid:
            return off
        if pos < lo:
            return max(1, pos)


def _reps():
    """Repeat offsets: Offset_Values 1, 2 and 3 with a literal length of zero (rep1 / rep2 swaps and rep0 - 1), repeats in
    the first sequence of a block, and repeat history carried across raw blocks (which do not change it)."""
    rng = np.random.default_rng(404)
    hist = [1, 4, 8]                                # what the parse has used most recently (libzstd finds the repeats itself)

    after_raw = [False]

    def kind(rng, pos):
        ll = int(rng.choice([0, 0, 0, 1, 2, 5, 9]))
        ml = int(rng.integers(4, 24))
        r = rng.random()
        if after_raw[0]:                            # first sequence after a raw block: the previous offset again (rep0)
            after_raw[0] = False
            ll, off = max(ll, 1), hist[0]
        elif r < 0.45 and pos + ll > 1 + max(hist):
            off = hist[int(rng.integers(0, 3))] if rng.random() < 0.8 else hist[0] - 1
        else:
            off = _new_off(rng, pos + ll, 16, 1500, hist)
        off = max(1, min(off, pos + ll))
        hist[:] = [off] + [h for h in hist if h != off][:2]
        return ll, off, ml, b"0123456789abcdef"
    B = Blocks(rng, 2048)
    B.add(kind, 3)
    for _ in range(12):
        B.raw(1 + int(rng.integers(0, 2)))
        after_raw[0] = True
        B.add(kind, 3)
    return B.build({P_LEVEL: 3})


def _tables():
    """Every sequence table in RLE mode, and Repeat_Mode tables whose describing block lies two or more blocks back,
    across raw blocks too."""
    rng = np.random.default_rng(505)
    last = [0, 0, 0]

    def off_in(pos, lo, hi):
        off = _new_off(rng, pos, lo, hi, last)
        last[:] = [off, last[0], last[1]]
        return off

    def ml_any(rng):                                # few match lengths, skewed: described ML tables pay off and can repeat
        return int(rng.choice([4, 5, 6, 7], p=[0.1, 0.5, 0.2, 0.2]))

    def mix(rng, pos):
        ll = int(rng.integers(0, 24)); return ll, off_in(pos + ll, 4, 3000), ml_any(rng), b"abcdefghijklmnopqrstuvwxyz"

    def ll_rle(rng, pos):
        return 6, off_in(pos + 6, 4, 3000), ml_any(rng), b"abcdefghijklmnopqrstuvwxyz"

    def of_rle(rng, pos):
        ll = int(rng.integers(0, 24)); return ll, off_in(pos + ll, 520, 1000), ml_any(rng), b"abcdefghijklmnopqrstuvwxyz"

    def ml_rle(rng, pos):
        ll = int(rng.integers(0, 24)); return ll, off_in(pos + ll, 4, 3000), 9, b"abcdefghijklmnopqrstuvwxyz"
    B = Blocks(rng, 4096)
    B.add(mix, 4).raw().add(mix, 2).add(ll_rle).add(mix, 3).add(of_rle).add(mix, 3).add(ml_rle).add(mix, 3).raw().add(mix, 2)
    return B.build({P_LEVEL: 19})


def _literals():
    """Literal sections in every form: Huffman with direct 4-bit weights, 1-stream Huffman, treeless with 1 and 4
    streams, raw and RLE with the 3-byte header; and an RLE block."""
    rng = np.random.default_rng(606)
    small = bytes(range(10))                        # symbols 0..9: weights go out direct

    def matches(pos, ml):
        return _new_off(rng, pos, max(ml, 64), 60000)

    def rich(rng, pos):                             # ~8 KiB of literals per block, 4 streams
        ll, ml = int(rng.integers(40, 120)), int(rng.integers(30, 90)); return ll, matches(pos + ll, ml), ml, small

    def lean(alpha, lo, hi):                        # ll in [lo, hi) per 300-600 bytes: ~200 literals per block (1 stream),
        def k(rng, pos):                            # or ~550 (4 streams, treeless while the last tree still fits)
            ll, ml = int(rng.integers(lo, hi)), int(rng.integers(300, 600)); return ll, matches(pos + ll, ml), ml, alpha
        return k

    def run_of(alpha, n):                           # one run of n literals of one alphabet, then matches only
        first = [True]

        def k(rng, pos):
            ll, first[0] = (n if first[0] else 0), False
            ml = int(rng.integers(2000, 3000)); return ll, matches(pos + ll, ml), ml, alpha
        return k

    B = Blocks(rng, 16384)
    B.add(rich, 3, True).add(lean(small, 10, 20), 2, True).add(lean(small, 3, 8), 2, True).add(lean(b"QRSTUVWXYZ", 3, 8), 2, True)
    B.add(rich, 2, True)
    B.add(run_of(RANDOM, 5000), 1, True).add(run_of(b"\x07", 5000), 1, True).add(rich, 1, True)
    B.seqs.append((1, 1, B.bsize * 3 - 1)); B.alpha.append(b"\0"); B.pos += B.bsize * 3      # three blocks of zeros
    B.add(rich, 2, True)
    return B.build({P_LEVEL: 1})


def _deep():
    """Matches reaching hundreds of 1 KiB blocks back, in a frame of 700 blocks."""
    rng = np.random.default_rng(707)

    def kind(rng, pos):
        ll, ml = int(rng.integers(0, 16)), int(rng.integers(8, 64))
        far = pos > 200 * 1024 and rng.random() < 0.7
        return ll, _new_off(rng, pos + ll, 100 * 1024 if far else 16, pos + ll if far else 4096), ml, b"abcdefghijklmnopqrstuvwxyz"
    return Blocks(rng, 1024).add(kind, 700).build({P_LEVEL: 3})


def _reference_ultra():
    """libzstd's own parser (level 3, windowLog 27, long-distance matching) on 1 MiB of random bytes that repeats 33 MiB
    later, after a run of zeros."""
    rng = np.random.default_rng(808)
    a = rng.integers(0, 256, MiB, dtype=np.uint8)
    src = np.concatenate([a, np.zeros(32 * MiB, np.uint8), a])
    return src, None, {P_LEVEL: 3, P_WINDOWLOG: 27, P_LDM: 1}


def _reps_predef():
    """Repeat offsets in a frame whose headers show no inter-block state (predefined tables, raw literals): the block
    parallel sequence decoders meet them at run time and send the frame to the frame-sequential pass."""
    rng = np.random.default_rng(909)
    hist = [1, 4, 8]

    def kind(rng, pos):
        ll, ml = int(rng.integers(40, 400)), int(rng.integers(4, 300))
        if rng.random() < 0.3 and pos + ll > max(hist):
            off = hist[int(rng.integers(0, 3))]
        else:
            off = _new_off(rng, pos + ll, 16, 20000, hist)
        hist[:] = [off] + [h for h in hist if h != off][:2]
        return ll, off, ml, b"0123456789"
    return Blocks(rng, 4096).add(kind, 40).build({P_LEVEL: 1, P_LITMODE: 2})


def _reached_reps_predef(tr):
    return bool((tr.col("modes")[tr.col("nseq") > 0] == 0).all() and not (tr.col("lit_type") == 3).any()
                and (tr.seq[:, 1] <= 3).any())


def _reached_reps(tr):
    ov, ll = tr.seq[:, 1], tr.seq[:, 0]
    zero = all(((ov == v) & (ll == 0)).any() for v in (1, 2, 3))
    typ, first = tr.col("type"), tr.col("seq_first")
    after_raw = any(typ[b] == 2 and typ[b - 1] == 0 and tr.blk[b, ZT["nseq"]] > 0 and ov[first[b]] <= 3 for b in range(1, len(typ)))
    return bool(zero and after_raw)


def _reached_tables(tr):
    m = modes(tr)
    both = all((m[:, t] == 1).any() and (m[:, t] == 3).any() for t in range(3))
    return both and any(r["src"] < b - 1 for r in repeat_sources(tr) for b in [r["block"]])


def repeat_sources(tr):
    """For every table of every block in Repeat_Mode: the block whose header describes the table (the last one before it
    with mode 1 or 2 for that table), or 'predef' after a mode-0 block."""
    m, out = modes(tr), []
    cur = [None, None, None]
    for b in range(len(m)):
        for t in range(3):
            if m[b, t] in (1, 2):
                cur[t] = b
            elif m[b, t] == 0:
                cur[t] = "predef"
            elif m[b, t] == 3:
                out.append({"block": b, "table": t, "src": cur[t]})
    return out


def _reached_literals(tr):
    lt, sf, streams, form = tr.col("lit_type"), tr.col("lit_sf"), tr.col("lit_streams"), tr.col("tree_form")
    return bool(((lt == 2) & (streams == 1)).any() and ((lt == 2) & (form == 0)).any()
                and ((lt == 3) & (streams == 1)).any() and ((lt == 3) & (streams == 4)).any()
                and ((lt == 0) & (sf == 3)).any() and ((lt == 1) & (sf == 3)).any() and (tr.col("type") == 1).any())


CASES = {
    "dense": (_dense, lambda tr: bool(((tr.col("nseq") >= 0x7F00) & (tr.col("nseq_bytes") == 3)).any())),
    "far": (_far, lambda tr: of_codes(tr).max() >= 25),
    "far_predef": (_far_predef, lambda tr: any(m == 0 and (of_codes(tr)[seq_blocks(tr) == b] >= 25).any()
                                               for b, m in enumerate(tr.col("modes")))),
    "reps": (_reps, _reached_reps),
    "reps_predef": (_reps_predef, _reached_reps_predef),
    "tables": (_tables, _reached_tables),
    "literals": (_literals, _reached_literals),
    "deep": (_deep, lambda tr: match_block_distance(tr).max() >= 100),
    "reference_ultra": (_reference_ultra, lambda tr: of_codes(tr).max() >= 25),
}


@functools.lru_cache(maxsize=None)
def case(name):
    """(source, frame) of a named case."""
    gen = CASES[name][0]
    src, seqs, params = gen()
    return src, compress(src, params, seqs)


@functools.lru_cache(maxsize=None)
def trace(name):
    return o.zstd_trace(case(name)[1])
