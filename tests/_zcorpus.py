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
import _zxmodel as zx

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


# ---------------------------------------------------------------------------------------------------- GPU schedule edges
# The x_* cases state edges of the execute pass (zx_block) and of the lane-per-block sequence reader, as events of the
# models in _zxmodel.py.  Each execute case is written twice from the same parse: at level 1 with raw literals (predefined
# tables: the lane sequence decoder) and at level 19 (Huffman literals, described tables: the dependent-block route).
class Plan:
    """A parse written block by block: every block of `bsize` bytes is an explicit list of block-relative rows (ll, off,
    ml), then one pad match (or literals) that fills it exactly.  off may be a (lo, hi) range: a fresh offset from it that
    is none of the repeat offsets libzstd would code it as.  raw() and rle() add a block of random literals (stored raw)
    and one of a single byte (an RLE block).  The repeat-offset history is followed as libzstd keeps it (raw and RLE blocks
    leave it unchanged), and dictated offsets that it would code as repeats are counted in `reps`.
    omit: labels of blocks written as pad only — how a test checks that a case's predicate depends on its edge blocks."""
    omit = frozenset()

    def __init__(self, seed, bsize=4096, alpha=b"abcd"):
        self.rng, self.bsize, self.alpha = np.random.default_rng(seed), bsize, alpha
        self.seqs, self.alphas, self.pos, self.carry, self.carry_random = [], [], 0, 0, False
        self.hist, self.reps = [1, 4, 8], 0

    def _is_rep(self, ll, off):
        h = self.hist
        return off in (h[1], h[2]) or (off == h[0] if ll else off == h[0] - 1)

    def fresh(self, at, ll, lo, hi):
        """An offset in [lo, min(hi, at)] that is no repeat offset for a sequence with ll literals at position at."""
        hi = min(hi, at)
        assert lo <= hi, (lo, hi, at)
        while True:
            off = int(self.rng.integers(lo, hi + 1))
            if not self._is_rep(self.carry + ll, off):
                return off

    def _put(self, ll, off, ml, at, track=True):
        if isinstance(off, tuple):
            off = self.fresh(at, ll, *off)
        assert 0 < off <= at, (off, at)
        if track:
            if self._is_rep(self.carry + ll, off):
                self.reps += 1
            else:
                self.hist = [off] + self.hist[:2]
        self.seqs.append((self.carry + ll, off, ml)); self.alphas.append(RANDOM if self.carry_random else self.alpha)
        self.carry, self.carry_random = 0, False

    def block(self, rows, tail=0, label=None):
        if label is not None and label in Plan.omit:
            rows = [(8, (16, 64), 8)]
        p = 0
        for ll, off, ml in rows:
            self._put(ll, off, ml, self.pos + p + ll); p += ll + ml
        rest = self.bsize - p - tail
        assert rest >= 0, (label, p, tail)
        if rest >= 4:
            self._put(1, (64, 4000), rest - 1, self.pos + p + 1)
        else:
            tail += rest
        self.carry += tail; self.pos += self.bsize
        return self

    def seed(self):
        return self.block([(256, (16, 200), 40)], label=None)

    def raw(self):
        self.carry += self.bsize; self.pos += self.bsize; self.carry_random = True
        return self

    def rle(self):
        self._put(1, 1, self.bsize - 1, self.pos + 1, track=False); self.pos += self.bsize
        return self

    def build(self, params):
        seqs = np.array(self.seqs, np.int64).reshape(-1, 3)
        src = build_from_seqs(seqs, self.carry, self.alphas + [RANDOM], self.rng)
        return src, seqs, {**params, P_MAXBLOCK: self.bsize}


LANE_ROUTE = {P_LEVEL: 1, P_LITMODE: 2}
DEP_ROUTE = {P_LEVEL: 19}


def _x_steps(P):
    """Steps ended by the 32-sequence cap, by the span at exactly 2048 bytes and at 2049, a single sequence of 2048
    bytes; lone steps (first sequence above the span): ll > 2048 with a match in its own literals, ml > 2048 at offsets
    >= ml, 33, 32, 31, 3, 2 and 1, first and last in their block, read by the next step."""
    P.seed().block([(0, (64, 300), 40)] * 3)
    P.block([(2, (16, 2000), 10)] * 34, label="cap")
    P.block([(28, (64, 2000), 100)] * 16 + [(1, (64, 2000), 10)], label="span_2048")
    P.block([(28, (64, 2000), 100)] * 15 + [(20, (64, 2000), 106), (0, (64, 2000), 3)], label="span_2049")
    P.block([(48, (64, 200), 2000), (5, (2000, 4000), 10)], label="single_2048")
    P.block([(2100, 50, 20), (3, 1000, 20)], label="lone_lits")
    P.block([(5, (3000, 8000), 2500), (2, 40, 16)], label="lone_straight")
    for off in (33, 32, 31, 3, 2, 1):
        P.block([(5, off, 2100), (3, (100, 1500), 10)], label="lone_off_%d" % off)
    P.block([(10, (64, 2000), 100), (5, (64, 2000), P.bsize - 115)], label="lone_last")
    return P


def _x_lits(P):
    """Literal runs copied by their lane (0, 1, 7, 8, 9, 31, 32) and by the warp (33, 100, 300); a match reading a
    warp-copied run of its own step back through the window; blocks ending with 0, 1 and 40 literals."""
    P.seed()
    rows = [(n, (64, 2000), 12) for n in (0, 1, 7, 8, 9, 31, 32)] + [(33, (64, 2000), 40), (100, (64, 2000), 80), (300, (64, 2000), 200)]
    P.block(rows + [(120, (64, 2000), 30), (2, 100, 20)], label="runs")
    P.block([(5, (64, 2000), 30)] * 4, tail=1, label="trail_1")
    P.block([(5, (64, 2000), 30)] * 4, tail=40, label="trail_40")
    P.block([(5, (64, 2000), 30)] * 4, label="trail_0")
    return P


def _x_matches(P):
    """Own-lane matches with off == ml (ml 3-32) against in-order ones with off == ml - 1; independent matches of 32 and
    33 bytes; own-lane sources split at the step start at every nlow from 0 to ml (ml 3-32); sources ending at an earlier
    destination's start or one byte into it, starting at its end or one byte before; in-order matches reading an earlier
    in-order match of the step, an own-lane match reading one of an earlier step; a chain of 31 dependent matches."""
    P.seed().block([(0, (64, 300), 40)] * 3)
    P.block([(ml, ml, ml) for ml in range(3, 33)], label="off_eq_ml")
    P.block([(ml, ml - 1, ml) for ml in range(3, 33)], label="off_ml_minus_1")
    P.block([(40, 40, 32), (45, 41, 33)], label="indep_32_33")
    pairs = [(ml, k) for ml in range(3, 33) for k in range(ml + 1)]
    for g in range(0, len(pairs), 31):
        rows, mp = [(40, (100, 2000), 8)], 48                       # lane 0: 40 literals at the step start
        for ml, k in pairs[g: g + 31]:
            mp += 1
            rows.append((1, mp + k, ml)); mp += ml                  # source starts k bytes below the step start
        P.block(rows, label="nlow")
    rows = []
    for ll_j, off_i in ((12, 38), (12, 37), (12, 20), (12, 21)):    # 10-byte destination d, then 20 literals and 8 bytes
        rows += [(ll_j, (200, 2000), 10), (20, off_i, 8)]          # from d - 8, d - 7, d + 10 (its end), d + 9
    for t in range(6):                                              # the same one byte into 40-byte destinations, which
        rows += [(12, (200, 2000), 40), (20 + t, 67 + t, 8)]        # the in-order pass writes after the own-lane copies
    P.block(rows, label="dep_edges")
    P.block([(3, 2, 20), (1, 10, 5), (1, (64, 2000), 2030), (2, 2057, 10)], label="inorder_reads")
    P.block([(8, (64, 2000), 4)] + [(1, 5 + i % 4, 4) for i in range(31)], label="chain")
    return P


def _x_cross(P):
    """Sources 1, 2 and 3 or more blocks back and sources straddling the block start, in the first and in later steps,
    for own-lane, in-order and lone matches, across raw and RLE blocks."""
    P.seed().block([(3, (64, 300), 60)] * 4).block([(3, (64, 300), 60)] * 4).block([(3, (64, 300), 60)] * 4)

    def reach(p):
        """Rows starting at block position p whose sources start at the given block positions (negative: earlier
        blocks): own-lane straddling, 2 and 4 blocks back; in-order 1 block back, straddling, 2 and 4 blocks back."""
        b, rows = P.bsize, []
        for ll, sp, ml in ((4, -6, 16), (4, -b - 100, 16), (4, -3 * b - 50, 16), (4, -400, 100), (2, -5, 40),
                           (4, -b - 300, 60), (4, -3 * b - 700, 60)):
            rows.append((ll, p + ll - sp, ml)); p += ll + ml
        return rows, p

    first, p = reach(0)
    later, _ = reach(p + 1901)                                      # after a 1901-byte sequence: a later step
    P.raw().block(first + [(1, (64, 2000), 1900)] + later, label="after_raw")
    P.rle().block(reach(0)[0], label="after_rle")
    P.block([(5, 105, 2100)], label="lone_straddle")
    P.raw().block([(5, P.bsize + 500, 2100)], label="lone_back2")
    P.rle().block([(5, 3 * P.bsize + 200, 2100)], label="lone_back3")
    return P


def _x_case(build, params):
    def gen():
        P = build(Plan(1000 + sum(map(ord, build.__name__))))
        if params is LANE_ROUTE:
            assert P.reps == 0, (build.__name__, "dictated offsets libzstd would write as repeat offsets", P.reps)
        return P.build(params)
    return gen


X_EVENTS = {
    "x_steps": ["step_cap", "step_span_2048", "step_span_2049", "step_single_2048", "lone_reads_own_literals",
                "lone_straight_long", "lone_off_33", "lone_off_32", "lone_off_31", "lone_off_3", "lone_off_2", "lone_off_1",
                "lone_first", "lone_last", "lone_read_next", "lone_chunk32", "lone_modulo"],
    "x_lits": ["lit_lane_%d" % n for n in (0, 1, 7, 8, 9, 31, 32)] + ["lit_warp_33", "lit_warp_long", "reads_warp_literals",
                                                                     "trailing_0", "trailing_1", "trailing_ge33"],
    "x_matches": ["own_off_eq_ml_%d" % m for m in range(3, 33)] + ["inorder_off_ml_minus_1_%d" % m for m in range(3, 33)]
                 + ["nlow_%d_%d" % (m, k) for m in range(3, 33) for k in range(m + 1)]
                 + ["indep_own_32", "indep_inorder_33", "dep_src_end_at_dest", "dep_src_end_one_into_dest",
                    "dep_src_start_at_dest_end", "dep_src_start_one_before_dest_end", "dep_src_end_one_into_inorder_dest",
                    "inorder_reads_inorder",
                    "own_reads_earlier_inorder", "dep_chain_31", "inorder_modulo", "inorder_straight"],
    "x_cross": ["cross_%s_back%d" % (p, k) for p in ("own", "inorder", "lone") for k in (1, 2, 3)]
               + ["cross_%s_straddle" % p for p in ("own", "inorder", "lone")]
               + ["cross_first_step", "cross_later_step", "cross_over_raw", "cross_over_rle"],
}


def lane_route(tr):
    """Every sequence section on the predefined tables, raw or RLE literals, no repeat Offset_Value: the lane decoder."""
    return bool((tr.col("modes")[tr.col("nseq") > 0] == 0).all() and not (tr.col("lit_type") >= 2).any()
                and not (tr.seq[:, 1] <= 3).any())


def dep_route(tr):
    """Some block with a table that is not predefined or treeless literals (the frame the host scan flags), and some
    Huffman-coded literals."""
    return bool((((tr.col("nseq") > 0) & (tr.col("modes") != 0)) | (tr.col("lit_type") == 3)).any() and (tr.col("lit_type") == 2).any())


def _reached_exec(kind, route):
    def pred(tr):
        ev = zx.exec_frame(tr)[1]
        return route(tr) and all(ev[e] > 0 for e in X_EVENTS[kind])
    return pred


def _x_budget():
    """Predefined-table blocks (level 1, raw literals, windowLog 27) whose sequences put the lane reader's bit budget at
    its edges: extra bits (offset + match + literal length) of 40 and 41 with every symbol's state transition at full
    width, at every bit phase of the refill, so that a sequence with 40 extra bits after a refill of 57 valid bits
    leaves no bit; the largest sum a block allows (offset code 24, 16 + 15 extra bits = 55); blocks with one and two
    sequences, whose bit streams are a few bytes."""
    rng = np.random.default_rng(4242)
    params = {**LANE_ROUTE, P_WINDOWLOG: 27}
    seqs, hist, p = [], [1, 4, 8], 0

    def put(ll, off, ml):
        nonlocal p
        while off in hist or (ll == 0 and off == hist[0] - 1):
            off -= 1
        assert 0 < off <= p + ll
        seqs.append((ll, off, ml)); hist[:] = [off] + hist[:2]; p += ll + ml

    def in_code(base, c):
        return int(rng.integers(base[c], base[c + 1]))
    lb = list(zx.LL_BASE) + [1 << 17]; mb = list(zx.ML_BASE) + [1 << 17]
    while p < 1100 * 1024:                                  # history: about 16 sequences of 3-13 KiB per 128 KiB block
        ll = int(rng.integers(20, 3000)); put(ll, int(rng.integers(16, max(17, min(p + ll, 60000)))), int(rng.integers(3000, 10000)))
    # (offset code, ML code, LL code): every symbol has a count of 1 or -1 in its predefined table (17 state bits)
    kinds = {40: [(16, 48, 31), (18, 47, 30), (14, 49, 32)], 41: [(17, 48, 30), (19, 47, 30), (15, 49, 32)]}
    for i in range(240):
        ofc, mc, lc = kinds[40 + i % 2][int(rng.integers(0, 3))]
        ll, ml = in_code(lb, lc), in_code(mb, mc)
        put(ll, int(rng.integers(1 << ofc, 2 << ofc)) - 3, ml)
        for _ in range(int(rng.integers(0, 3))):             # jitter: the next one starts at another bit phase
            ll = int(rng.integers(1, 700)); put(ll, int(rng.integers(16, min(p + ll, 60000))), int(rng.integers(400, 3000)))
    for _ in range(3):
        put(4, int(rng.integers(100, 5000)), 8)
    # one byte up to a block boundary beyond 17 MiB (RLE blocks).  libzstd may end a block early where it splits a
    # sequence, so the boundaries are read from a frame of the parse so far followed by a shorter run.
    probe = np.array(seqs + [(1, 1, 2 * MiB)], np.int64)
    tp = o.zstd_trace(compress(build_from_seqs(probe, 0, b"ETAOINSHRD", np.random.default_rng(0)), params, probe))
    phase = int(zx.block_starts(tp)[-2]) % (1 << 17)
    run_end = (17 << 20) + (phase - (17 << 20)) % (1 << 17)
    put(1, 1, run_end - p - 1)
    ll, ml = 32768 + 1000, 65539 + 2000                      # LL code 34 (15 bits), ML code 52 (16 bits), offset code 24
    if "s1_55" in Plan.omit:
        ll, ml = 1000, 65539 + 2000 + 32768
    put(ll, p + ll - int(rng.integers(1000, 500000)), ml)   # 16.5-17 MiB back: into the history
    put(10, int(rng.integers(300, 90000)), (1 << 17) - ll - ml - 10)                         # the block's 2nd sequence
    put(5, int(rng.integers(300, 90000)), (1 << 17) - 5)                                     # a block of one sequence
    seqs = np.array(seqs, np.int64)
    src = build_from_seqs(seqs, 64, b"ETAOINSHRD", rng)
    return src, seqs, params


BUDGET_EVENTS = (["s1_%d_phase%d" % (s, r) for s in (40, 41) for r in range(8)] + ["slack_0", "s1_55", "second_refill",
                 "short_stream", "refill_aligned", "refill_funnel", "refill_bytes"] + ["section_mod8_%d" % r for r in range(8)])


def _reached_budget(tr):
    lanes, ev = zx.lane_frame(tr.frame)
    slack = [s["slack"] for r in lanes.values() for s in r["seqs"]]
    nblk = int(((tr.col("type") == 2) & (tr.col("nseq") > 0)).sum())
    return lane_route(tr) and len(lanes) == nblk and min(slack) == 0 and all(ev[e] > 0 for e in BUDGET_EVENTS)


X_CASES = {}
for _k, _b in (("x_steps", _x_steps), ("x_lits", _x_lits), ("x_matches", _x_matches), ("x_cross", _x_cross)):
    X_CASES[_k + "_l1"] = (_x_case(_b, LANE_ROUTE), _reached_exec(_k, lane_route))
    X_CASES[_k + "_l19"] = (_x_case(_b, DEP_ROUTE), _reached_exec(_k, dep_route))
X_CASES["x_budget"] = (_x_budget, _reached_budget)

CASES = {
    "dense":(_dense, lambda tr: bool(((tr.col("nseq") >= 0x7F00) & (tr.col("nseq_bytes") == 3)).any())),
    "far": (_far, lambda tr: of_codes(tr).max() >= 25),
    "far_predef": (_far_predef, lambda tr: any(m == 0 and (of_codes(tr)[seq_blocks(tr) == b] >= 25).any()
                                               for b, m in enumerate(tr.col("modes")))),
    "reps": (_reps, _reached_reps),
    "reps_predef": (_reps_predef, _reached_reps_predef),
    "tables": (_tables, _reached_tables),
    "literals": (_literals, _reached_literals),
    "deep": (_deep, lambda tr: match_block_distance(tr).max() >= 100),
    "reference_ultra": (_reference_ultra, lambda tr: of_codes(tr).max() >= 25),
    **X_CASES,
}


@functools.lru_cache(maxsize=None)
def case(name):
    """(source, frame) of a named case."""
    gen = CASES[name][0]
    src, seqs, params = gen()
    return src, compress(src, params, seqs)


@functools.lru_cache(maxsize=None)
def trace(name):
    """The oracle's block trace of a case, with the frame itself as trace.frame."""
    frame = case(name)[1]
    tr = o.zstd_trace(frame)
    tr.frame = frame
    return tr
