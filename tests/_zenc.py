"""Plain-Python restatement of the choices the GPU zstd encoder (lz4_kernels.cu zstd_blocks_kernel, zstd_entropy.cuh)
makes on top of the LZ77 parse it shares with the LZ4 compressor (lz4_pipe.cuh), for tests that hold its output to them:
  - the parse: the LZ4 sequences of the bit-exact CPU twin orc_lz4_block_compress_b200 on the same 64 KiB window;
  - the sub-block cut: every 4 tiles (16 KiB) a block is closed at the start of the match still pending there;
  - the Huffman code: two-queue tree, length-limited to 11 bits (huf_lengths);
  - the whole framed stream (framed_b200): these blocks, or the 16 KiB blocks of the level 6-12 twin (_zlazy), each
    written by the entropy stage's CPU twin (oracle/zstd_enc_twin.c, block_b200), in the frames the frame pack kernel
    writes.
"""
import ctypes

import numpy as np

import _oracle as o

WINDOW = 65536
SUB = 4 * 4096                   # a sub-block is closed every 4 tiles of 4096 positions
HUF_MAXBITS = 11


def lz4_twin_block(win):
    """The CPU twin's LZ4 block for one window."""
    win = np.ascontiguousarray(win, dtype=np.uint8)
    L = o.orc()
    cap = L.orc_lz4_block_bound(win.size)
    out = np.empty(cap, np.uint8)
    n = L.orc_lz4_block_compress_b200(win.ctypes.data, win.size, out.ctypes.data, cap)
    return out[:n]


def lz4_sequences(block):
    """(match start, offset, match length) of every sequence of an LZ4 block, as an (n, 3) int64 array."""
    b = block.tobytes()
    i, pos, n, seqs = 0, 0, len(b), []
    while i < n:
        tok = b[i]; i += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                x = b[i]; i += 1; ll += x
                if x != 255:
                    break
        i += ll; pos += ll
        if i >= n:
            break                                   # the last sequence carries literals only
        off = b[i] | (b[i + 1] << 8); i += 2
        ml = tok & 15
        if ml == 15:
            while True:
                x = b[i]; i += 1; ml += x
                if x != 255:
                    break
        ml += 4
        seqs.append((pos, off, ml)); pos += ml
    return np.array(seqs, dtype=np.int64).reshape(-1, 3)


def sub_blocks(seqs, n):
    """Start positions of the sub-blocks of a window of n bytes whose twin parse is `seqs`: at 16, 32 and 48 KiB (when the
    window goes on) the encoder closes a block at the start of the last match that began before that point."""
    starts, z_pos = [0], 0
    for t1 in range(SUB, n, SUB):
        before = seqs[seqs[:, 0] < t1, 0] if len(seqs) else np.zeros(0, np.int64)
        c = int(before[-1]) if before.size else t1
        if c > z_pos:
            starts.append(c)
            z_pos = c
    return starts


def window_model(win):
    """[(start, end, seqs of the twin whose match starts in [start, end))] for every sub-block of a window."""
    seqs = lz4_sequences(lz4_twin_block(win))
    st = sub_blocks(seqs, len(win)) + [len(win)]
    out = []
    for a, b in zip(st[:-1], st[1:]):
        sel = seqs[(seqs[:, 0] >= a) & (seqs[:, 0] < b)] if len(seqs) else seqs
        out.append((a, b, sel))
    return out


def sub_block_literals(win, a, b, seqs):
    """The literal bytes of sub-block [a, b) with matches `seqs`."""
    keep = np.ones(b - a, bool)
    for s, _, ml in seqs:
        keep[s - a: s - a + ml] = False
    return np.asarray(win[a:b])[keep]


def huf_lengths(hist, limit=True):
    """Code length per symbol (dict) and the largest length, as zstd_entropy.cuh builds them: present symbols in
    ascending (count, symbol) order; two queues (leaves, internal nodes), the leaf taken on ties; depths from the tree;
    then, if the deepest leaf is below 11, clamp to 11, repay the Kraft excess by lengthening the first (rarest) leaf
    whose lengthening fits in what is left, else the rarest still short leaf, and hand back any overshoot by shortening
    11-bit codes, rarest first."""
    order = sorted((int(c), s) for s, c in enumerate(hist) if c)
    n = len(order)
    cnt = [c for c, _ in order] + [0] * (n - 1)
    par = [0] * (2 * n - 1)
    li, ii, ni = 0, n, n
    for _ in range(n - 1):
        pick = []
        for _ in range(2):
            if li < n and (ii >= ni or cnt[li] <= cnt[ii]):
                pick.append(li); li += 1
            else:
                pick.append(ii); ii += 1
        cnt[ni] = cnt[pick[0]] + cnt[pick[1]]; par[pick[0]] = par[pick[1]] = ni; ni += 1
    depth = [0] * (2 * n - 1)
    for v in range(ni - 2, -1, -1):
        depth[v] = depth[par[v]] + 1
    ln = depth[:n]
    maxl = max(ln)
    if limit and maxl > HUF_MAXBITS:
        ln = [min(x, HUF_MAXBITS) for x in ln]
        excess = sum(1 << (HUF_MAXBITS - x) for x in ln) - (1 << HUF_MAXBITS)
        while excess > 0:
            best = -1
            for i in range(n):
                if ln[i] < HUF_MAXBITS:
                    if best < 0:
                        best = i
                    if (1 << (HUF_MAXBITS - 1 - ln[i])) <= excess:
                        best = i
                        break
            if best < 0:
                break
            excess -= 1 << (HUF_MAXBITS - 1 - ln[best]); ln[best] += 1
        for i in range(n):
            if excess >= 0:
                break
            if ln[i] == HUF_MAXBITS:
                ln[i] -= 1; excess += 1
        maxl = HUF_MAXBITS
    return {s: ln[i] for i, (_, s) in enumerate(order)}, maxl


def kraft(lengths, maxbits):
    """Kraft sum in units of 2^-maxbits (complete code: exactly 1 << maxbits)."""
    return sum(1 << (maxbits - x) for x in lengths.values())


# ------------------------------------------------------------------------------------------------- entropy-stage twin
LIT_FEW, LIT_NOFORM, LIT_EST, LIT_BITBUF = 1, 2, 4, 8           # ORC_ZENC_LIT_*: why a literal section is raw
RAW_SIZE, RAW_BITBUF, RAW_NSEQ = 1, 2, 4                        # ORC_ZENC_RAW_*: why a block is raw
BITBUF = 3072 * 4                                               # the entropy stage's bit buffer, bytes


class _ZencTrace(ctypes.Structure):
    _fields_ = [("code", ctypes.c_void_p * 3), ("state", ctypes.c_void_p * 3),
                ("nseq", ctypes.c_uint32), ("nlit", ctypes.c_uint32), ("regen", ctypes.c_uint32),
                ("lit_mode", ctypes.c_uint32), ("lit_reason", ctypes.c_uint32), ("lit_size", ctypes.c_uint32),
                ("nused", ctypes.c_uint32), ("maxsym", ctypes.c_uint32), ("maxbits", ctypes.c_uint32),
                ("tree_bytes", ctypes.c_uint32), ("wdesc_len", ctypes.c_uint32),
                ("tot_bits", ctypes.c_uint32), ("est", ctypes.c_uint32), ("huf_bits", ctypes.c_uint32 * 4),
                ("seq_bits", ctypes.c_uint32), ("seq_body", ctypes.c_uint32), ("bsize", ctypes.c_uint32),
                ("raw_reason", ctypes.c_uint32), ("fin", ctypes.c_uint32 * 3),
                ("hlen", ctypes.c_uint8 * 256), ("hcode", ctypes.c_uint16 * 256)]


class BlockTrace:
    """What the twin decided for one block: the scalar fields of orc_zenc_trace_t as attributes, huf_bits / fin as
    lists, hlen / hcode as arrays, and (with chains=True) codes[k] / states[k] per stream 0 LL, 1 OF, 2 ML in encoding
    order.  rows / lits: the block's input."""

    def __init__(self, t, codes, states, rows, lits):
        for name, _ in _ZencTrace._fields_:
            if name not in ("code", "state"):
                v = getattr(t, name)
                setattr(self, name, list(v) if name in ("huf_bits", "fin") else np.array(v) if name in ("hlen", "hcode") else int(v))
        self.codes, self.states, self.rows, self.lits = codes, states, rows, lits

    @property
    def raw(self):
        return self.raw_reason != 0


def _L():
    L = o.orc()
    if not hasattr(L, "_zenc_ready"):
        L.orc_zstd_block_b200.restype = ctypes.c_long
        L.orc_zstd_block_b200.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                          ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(_ZencTrace)]
        L.orc_zenc_fse_table.restype = ctypes.c_int
        L.orc_zenc_fse_table.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L._zenc_ready = True
    return L


def fse_table(stream):
    """(log, sym, nbBits, baseline) of the predefined decoding table of stream 0 LL / 1 OF / 2 ML, as the twin has it."""
    sym, nb, base = np.zeros(64, np.uint8), np.zeros(64, np.uint8), np.zeros(64, np.uint16)
    log = _L().orc_zenc_fse_table(stream, sym.ctypes.data, nb.ctypes.data, base.ctypes.data)
    return log, sym[: 1 << log].astype(np.int64), nb[: 1 << log].astype(np.int64), base[: 1 << log].astype(np.int64)


def block_b200(rows, lits, raw, last, chains=False):
    """(block bytes, BlockTrace) of orc_zstd_block_b200: rows (n, 3) of (literal length, offset, match length)."""
    rows = np.ascontiguousarray(np.asarray(rows, np.int64).reshape(-1, 3), dtype=np.uint32)
    lits = np.ascontiguousarray(lits, dtype=np.uint8)
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    n = len(rows)
    cap = 3 + raw.size + lits.size + 16 * n + 1024
    out = np.empty(cap, np.uint8)
    t = _ZencTrace()
    codes = states = None
    if chains:
        codes = [np.zeros(max(n, 1), np.uint8) for _ in range(3)]
        states = [np.zeros(max(n, 1), np.uint16) for _ in range(3)]
        for k in range(3):
            t.code[k] = codes[k].ctypes.data
            t.state[k] = states[k].ctypes.data
    r = _L().orc_zstd_block_b200(rows.ctypes.data, n, lits.ctypes.data, lits.size, raw.ctypes.data, raw.size, int(bool(last)),
                                 out.ctypes.data, cap, ctypes.byref(t))
    if r < 0:
        raise ValueError("orc_zstd_block_b200 failed: %d" % r)
    if chains:
        codes = [c[:n].astype(np.int64) for c in codes]
        states = [s[:n].astype(np.int64) for s in states]
    return out[:r], BlockTrace(t, codes, states, rows.astype(np.int64), lits)


def rows_of(seqs, a):
    """(literal length, offset, match length) rows of sub-block [a, ...) from (match start, offset, length) rows."""
    rows, p = [], a
    for s, off, ml in np.asarray(seqs, np.int64).reshape(-1, 3).tolist():
        rows.append((s - p, off, ml)); p = s + ml
    return np.array(rows, np.int64).reshape(-1, 3)


def level3_blocks(content):
    """[(rows, literals, raw content, last)] of every block the level-3 encoder writes for one chunk."""
    out = []
    n = content.size
    for w0 in range(0, n, WINDOW):
        win = content[w0: w0 + WINDOW]
        model = window_model(win)
        for i, (a, e, seqs) in enumerate(model):
            last = w0 + WINDOW >= n and i + 1 == len(model)
            out.append((rows_of(seqs, a), sub_block_literals(win, a, e, seqs), win[a:e], last))
    return out


def lazy_blocks(content, level):
    """[(rows, literals, raw content, last)] of every 16 KiB block of the level 6-12 encoder for one chunk."""
    import _zlazy as zl
    out = []
    n = content.size
    for b, rows in enumerate(zl.twin_sequences(content, level) if n else []):
        b0, b1 = b * zl.BLOCK, min((b + 1) * zl.BLOCK, n)
        out.append((rows.astype(np.int64), literals_of(content[b0:b1], rows), content[b0:b1], b1 == n))
    return out


def literals_of(raw, rows):
    """The literal bytes of a block whose content is `raw` and whose sequences are `rows` (literal length, offset,
    match length): every byte no match covers."""
    keep = np.ones(len(raw), bool)
    p = 0
    for ll, _, ml in np.asarray(rows, np.int64).reshape(-1, 3).tolist():
        p += ll; keep[p: p + ml] = False; p += ml
    return np.asarray(raw)[keep]


def chunk_blocks(content, level):
    return level3_blocks(content) if level < 6 else lazy_blocks(content, level)


def fcs_bytes(n):
    return 1 if n <= 255 else 2 if n <= 65791 else 4


def frame_header(n):
    """Magic, FHD and Frame_Content_Size of a chunk of n bytes: single segment, no checksum, FCS in 1, 2 (n - 256) or 4
    bytes."""
    fl = fcs_bytes(n)
    fhd = {1: 0x20, 2: 0x60, 4: 0xA0}[fl]
    fcs = (n - 256 if fl == 2 else n).to_bytes(fl, "little")
    return (0xFD2FB528).to_bytes(4, "little") + bytes([fhd]) + fcs


def chunks(src, chunk, chunk_bytes=None):
    """The chunks of src: every `chunk` bytes (one empty chunk for an empty input), or chunk c = src[c * chunk:][:chunk_bytes[c]]."""
    if chunk_bytes is None:
        return [src[i: i + chunk] for i in range(0, max(src.size, 1), chunk)]
    return [src[c * chunk: c * chunk + int(b)] for c, b in enumerate(chunk_bytes)]


def framed_b200(src, chunk, level, chunk_bytes=None, blocks=None):
    """The framed stream the GPU zstd encoder writes at `level` (3: the level-3 class, 6-12: the search class), built on
    the CPU: per chunk a 12-byte skippable header, the frame header and every block through block_b200; an empty chunk
    is one empty raw last block.  blocks: a list that receives (chunk index, block index, BlockTrace) of every block."""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    out = []
    for c, content in enumerate(chunks(src, chunk, chunk_bytes)):
        body = []
        for b, (rows, lits, raw, last) in enumerate(chunk_blocks(content, level)):
            blk, tr = block_b200(rows, lits, raw, last)
            body.append(blk.tobytes())
            if blocks is not None:
                blocks.append((c, b, tr))
        if content.size == 0:
            body.append(bytes([1, 0, 0]))
        frame = frame_header(int(content.size)) + b"".join(body)
        out.append((0x184D2A50).to_bytes(4, "little") + (4).to_bytes(4, "little") + len(frame).to_bytes(4, "little") + frame)
    return np.frombuffer(b"".join(out), np.uint8)


def _blocks_of(frame):
    """[(offset, bytes)] of the blocks of one zstd frame written by this encoder (single segment, no checksum)."""
    fl = 1 if frame[4] == 0x20 else 2 if frame[4] == 0x60 else 4
    pos, out = 5 + fl, []
    while pos + 3 <= len(frame):
        h = int(frame[pos]) | int(frame[pos + 1]) << 8 | int(frame[pos + 2]) << 16
        size = (h >> 3) if (h >> 1) & 3 != 1 else 1
        out.append((pos, frame[pos: pos + 3 + size]))
        pos += 3 + size
        if h & 1:
            break
    return out


def first_difference(got, want):
    """Where framed stream `got` first departs from `want`: the frame, the block and the first differing field of the
    oracle's traces of both (or the first differing byte, when the traces agree)."""
    fg, fw = o.mt_frames(got), o.mt_frames(want)
    if len(fg) != len(fw):
        return "%d frames, the twin writes %d" % (len(fg), len(fw))
    for f, (a, b) in enumerate(zip(fg, fw)):
        if np.array_equal(a, b):
            continue
        if not np.array_equal(a[:5], b[:5]):
            return "frame %d: header %s, the twin writes %s" % (f, a[:9].tolist(), b[:9].tolist())
        ba, bb = _blocks_of(a), _blocks_of(b)
        for k, ((pa, xa), (pb, xb)) in enumerate(zip(ba, bb)):
            if np.array_equal(xa, xb):
                continue
            try:
                ta, tb = o.zstd_trace(a), o.zstd_trace(b)
            except ValueError as e:
                return "frame %d block %d (offset %d): %s" % (f, k, pa, e)
            for name in o.ZT_FIELDS:
                if name in ("seq_first", "lit_first"):
                    continue
                va, vb = int(ta.blk[k, o.ZT[name]]), int(tb.blk[k, o.ZT[name]])
                if va != vb:
                    return "frame %d block %d: %s %d, the twin's %d" % (f, k, name, va, vb)
            if not np.array_equal(ta.weights[k], tb.weights[k]):
                return "frame %d block %d: Huffman weights differ" % (f, k)
            n = min(xa.size, xb.size)
            d = int(np.flatnonzero(xa[:n] != xb[:n])[0]) if (xa[:n] != xb[:n]).any() else n
            return "frame %d block %d: byte %d of the block differs (same traced fields)" % (f, k, d)
        return "frame %d: %d blocks, the twin writes %d" % (f, len(ba), len(bb))
    return "streams equal"


def assert_twin(got, src, chunk, level, chunk_bytes=None):
    """The GPU framed stream `got` equals framed_b200 byte for byte.  Returns the twin's (chunk, block, BlockTrace) list."""
    blocks = []
    want = framed_b200(src, chunk, level, chunk_bytes, blocks)
    got = np.asarray(got, np.uint8)
    if not (got.size == want.size and np.array_equal(got, want)):
        raise AssertionError("GPU zstd stream (level %d) differs from the twin: %s" % (level, first_difference(got, want)))
    return blocks


def raw_counts(blocks):
    """{reason: count} of the raw blocks among framed_b200's `blocks`: "size", "bitbuf", "nseq" (a block counts under
    every reason that holds)."""
    out = {"size": 0, "bitbuf": 0, "nseq": 0}
    for _, _, t in blocks:
        for name, bit in (("size", RAW_SIZE), ("bitbuf", RAW_BITBUF), ("nseq", RAW_NSEQ)):
            out[name] += bool(t.raw_reason & bit)
    return out
