"""A corpus of LZ4 frames at the edges of the format and of the GPU decoder, written from parses the tests dictate.

liblz4 has no entry point that takes a parse, so this module writes the LZ4 blocks itself: a block is only tokens,
length bytes, literals and 2-byte offsets.  liblz4 (liblz4.so.1) is the judge: every block must decode with
LZ4_decompress_safe_usingDict into a buffer of exactly its regenerated size (which makes liblz4 enforce the end-of-block
rules: the last match starts at least 12 bytes before the end, the last 5 bytes are literals), and every frame with
LZ4F_decompress, both to the source the parse describes.  The source is built by running the parse
(_zcorpus.build_from_seqs), so content and parse agree by construction.

A frame spec is a dict: blocks (a list of per-block parses: (ll, off, ml) rows ending with the literals-only row
(ll, 0, 0)), bsid (blockSizeID 4-7), linked, csize (content size field), cchk (content checksum), bchk (block
checksums), dict_id, stored (indices of blocks written raw).  Every case is written in two layouts: `full`, where every
non-last block regenerates blockMaxSize (the decoder's two-pass path), and `short`, where a 100-byte first block is put in
front (the frame-sequential fallback).

The models restate two pieces of the decoder (zstdmt_b200/csrc/lz4_decode.cuh) so that the edges of its two passes can
be stated on the oracle's trace (orc_lz4f_trace)."""
import ctypes
import functools

import numpy as np
import pytest

import _oracle as o
import _zcorpus as zc

# lz4_decode.cuh, and match_exec.cuh for what pass B shares with the zstd execute pass (MX_STEP, MX_OWN, MX_SPAN); the
# model's own numbers: test_lz4_decode_corpus.py compares them with the source
LZD_WIN = 512           # compressed bytes pass A stages per step
LZD_NJ = 256            # token positions pass A's jump table covers per step; a step ends at the first token beyond
LZD_SEQS = 32           # sequences per pass-A step, match records per pass-B step (one per lane)
LZD_LONGLIT = 16        # pass A: longer literal runs are copied by the whole warp (>= 64 bytes: coop_copy_g2g)
LZD_LONG = 32           # pass B: longer independent matches are copied by the whole warp
LZX_SPAN = 2048         # pass B: output bytes one step may span
PUBLISH_EVERY = 4       # pass B publishes a linked block's progress every 4 steps
BLKMAX = {4: 1 << 16, 5: 1 << 18, 6: 1 << 20, 7: 1 << 22}
SHORT_PREFIX = 100
LIT_ALPHA = bytes(range(256))


# ---------------------------------------------------------------------------------------------------- liblz4
@functools.lru_cache(maxsize=None)
def lz4():
    try:
        L = ctypes.CDLL("liblz4.so.1")
    except OSError:
        pytest.skip("liblz4.so.1 not present")
    vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    L.LZ4_versionNumber.restype = ci
    L.LZ4_decompress_safe_usingDict.restype = ci
    L.LZ4_decompress_safe_usingDict.argtypes = [vp, vp, ci, ci, vp, ci]
    L.LZ4F_createDecompressionContext.restype = sz
    L.LZ4F_createDecompressionContext.argtypes = [ctypes.POINTER(vp), ctypes.c_uint]
    L.LZ4F_freeDecompressionContext.argtypes = [vp]
    L.LZ4F_decompress.restype = sz
    L.LZ4F_decompress.argtypes = [vp, vp, ctypes.POINTER(sz), vp, ctypes.POINTER(sz), vp]
    L.LZ4F_isError.restype = ctypes.c_uint; L.LZ4F_isError.argtypes = [sz]
    L.LZ4F_getErrorName.restype = ctypes.c_char_p; L.LZ4F_getErrorName.argtypes = [sz]
    return L


def liblz4_block(block, dict_bytes, size):
    """LZ4_decompress_safe_usingDict into exactly `size` bytes: the decoded bytes, or None if liblz4 rejects the block."""
    L = lz4()
    blk = np.ascontiguousarray(block, dtype=np.uint8)
    d = np.ascontiguousarray(dict_bytes, dtype=np.uint8)
    out = np.empty(max(size, 1), np.uint8)
    r = L.LZ4_decompress_safe_usingDict(blk.ctypes.data, out.ctypes.data, blk.size, size, d.ctypes.data if d.size else None, d.size)
    return out[:size] if r == size else None


def liblz4_frame(frame, cap):
    """LZ4F_decompress over the whole frame: (decoded bytes, bytes consumed), or (error name, 0)."""
    L = lz4()
    fr = np.ascontiguousarray(frame, dtype=np.uint8)
    ctx = ctypes.c_void_p()
    L.LZ4F_createDecompressionContext(ctypes.byref(ctx), 100)
    try:
        out = np.empty(cap + 1, np.uint8)
        got, pos, used = 0, 0, 0
        while True:
            dn, sn = ctypes.c_size_t(out.size - got), ctypes.c_size_t(fr.size - pos)
            r = L.LZ4F_decompress(ctx, out.ctypes.data + got, ctypes.byref(dn), fr.ctypes.data + pos, ctypes.byref(sn), None)
            if L.LZ4F_isError(r):
                return L.LZ4F_getErrorName(r).decode(), 0
            got += dn.value; pos += sn.value
            if r == 0:
                return out[:got], pos
            if sn.value == 0 and dn.value == 0:
                return "stalled", 0
    finally:
        L.LZ4F_freeDecompressionContext(ctx)


# ---------------------------------------------------------------------------------------------------- writer
def _put_len(out, n):
    while n >= 255:
        out.append(255); n -= 255
    out.append(n)


def write_block(rows, src, p):
    """The LZ4 block of the parse `rows`, whose output starts at src[p]."""
    out = bytearray()
    for ll, off, ml in rows:
        out.append(min(ll, 15) << 4 | (min(ml - 4, 15) if ml else 0))
        if ll >= 15:
            _put_len(out, ll - 15)
        out += src[p: p + ll].tobytes(); p += ll
        if ml:
            out += int(off).to_bytes(2, "little")
            if ml - 4 >= 15:
                _put_len(out, ml - 19)
            p += ml
    return bytes(out)


def regen(rows):
    return int(sum(ll + ml for ll, _, ml in rows))


def layout(spec, name):
    """The spec in layout `full` (as written) or `short` (a 100-byte literals-only first block in front: every later
    block keeps its offsets, which only reach back inside the source)."""
    if name == "full":
        return spec
    s = dict(spec)
    s["blocks"] = [[(SHORT_PREFIX, 0, 0)]] + list(spec["blocks"])
    s["stored"] = {i + 1 for i in spec.get("stored", ())}
    return s


def write_frame(spec, seed):
    """(frame bytes, source, per-block (rows, block bytes, output start)) of one spec."""
    rng = np.random.default_rng(seed)
    blocks = spec["blocks"]
    allrows = [r for b in blocks for r in b]
    src = zc.build_from_seqs(allrows, 0, LIT_ALPHA, rng) if allrows else np.zeros(0, np.uint8)
    bsid, blkmax = spec.get("bsid", 4), BLKMAX[spec.get("bsid", 4)]
    linked, bchk, cchk = spec.get("linked", False), spec.get("bchk", False), spec.get("cchk", False)
    csize, did = spec.get("csize", False), spec.get("dict_id")
    flg = 0x40 | (0 if linked else 0x20) | (0x10 if bchk else 0) | (0x08 if csize else 0) | (0x04 if cchk else 0) | (1 if did is not None else 0)
    hd = bytearray([flg, bsid << 4])
    if csize:
        hd += int(src.size).to_bytes(8, "little")
    if did is not None:
        hd += int(did).to_bytes(4, "little")
    out = bytearray((0x184D2204).to_bytes(4, "little")) + hd
    out.append((o.xxh32(np.frombuffer(bytes(hd), np.uint8)) >> 8) & 0xFF)
    p, info = 0, []
    for b, rows in enumerate(blocks):
        n = regen(rows)
        if b in spec.get("stored", ()):
            data = src[p: p + n].tobytes(); hdr = n | 0x80000000
        else:
            data = write_block(rows, src, p); hdr = len(data)
        if len(data) > blkmax or (b < len(blocks) - 1 and n > blkmax):
            raise ValueError("block %d: %d bytes for %d of output (blockMaxSize %d)" % (b, len(data), n, blkmax))
        out += hdr.to_bytes(4, "little") + data
        if bchk:
            out += o.xxh32(np.frombuffer(data, np.uint8)).to_bytes(4, "little")
        info.append((rows, data, p))
        p += n
    out += bytes(4)
    if cchk:
        out += o.xxh32(src).to_bytes(4, "little")
    return np.frombuffer(bytes(out), np.uint8).copy(), src, info


# ---------------------------------------------------------------------------------------------------- parse helpers
def close(rows, target, pos0=0, last=16, off=4):
    """rows + filler matches + `last` literals, regenerating exactly `target` bytes.  The filler is matches of offset
    `off` (at least `off` bytes of output must precede them: pos0 = bytes of history available before the block)."""
    rows = list(rows)
    r = target - regen(rows) - last
    if r < 0:
        raise ValueError("block parse longer than its target")
    if 0 < r < 4 + 1:
        last += r; r = 0
    if r:
        lit = max(0, off - pos0 - regen(rows))
        rows.append((lit + 1, off, r - lit - 1))          # one literal keeps the token ahead of the match
    rows.append((last, 0, 0))
    assert regen(rows) == target
    return rows


# ---------------------------------------------------------------------------------------------------- models
def step_walk_a(tokpos, end, abs_src):
    """Pass A's walk over one block (lzd_parse_block): a step starts at the token at ip0, stages the window
    [ip0 - sh, ip0 - sh + LZD_WIN) (sh = 16-byte misalignment of the block's absolute input offset + ip0) and takes the
    chain of sequences whose tokens lie fewer than LZD_NJ bytes past ip0, at most LZD_SEQS of them.  tokpos: block-relative
    token positions; end: block size.  Returns (ip0, sh, first sequence, count, why the step ended) per step."""
    steps, i, n = [], 0, len(tokpos)
    while i < n:
        ip0 = tokpos[i]; sh = (abs_src + ip0) & 15
        j = i
        while j < n and j - i < LZD_SEQS and tokpos[j] - ip0 < LZD_NJ:
            j += 1
        why = "end" if j == n else "cap" if j - i == LZD_SEQS else "span"
        steps.append((ip0, sh, i, j - i, why))
        i = j
    return steps


def steps_b(recs):
    """Pass B's step formation (lz4_exec_blocks_kernel, staged variant) over one block's match records (d, ml, off) in
    order: a step is the longest prefix of the next LZD_SEQS records whose destinations end within LZX_SPAN bytes of the
    first one's (d0); none fits: the first record alone, copied by the whole warp (a `lone` step).  Per record of a step:
    dependent = its source touches the destination of an earlier record of the step; own = copied by its own lane
    (independent, off >= ml, ml <= LZD_LONG); nlow = bytes of an own-lane source below d0 (read from global memory).
    Returns [(kind, d0, span, [(index, dep, own, nlow), ...])]."""
    out, base, n = [], 0, len(recs)
    while base < n:
        cnt = min(LZD_SEQS, n - base)
        d0 = recs[base][0]
        nfit = 0
        while nfit < cnt and recs[base + nfit][0] + recs[base + nfit][1] - d0 <= LZX_SPAN:
            nfit += 1
        if nfit == 0:
            out.append(("lone", d0, recs[base][1], [(base, False, False, 0)])); base += 1
            continue
        rs = []
        for k in range(nfit):
            d, ml, off = recs[base + k]
            sp = d - off
            dep = any(recs[base + j][0] < sp + ml and recs[base + j][0] + recs[base + j][1] > sp for j in range(k))
            own = off >= ml and not dep and ml <= LZD_LONG
            nlow = (0 if sp >= d0 else min(d0 - sp, ml)) if own else 0
            rs.append((base + k, dep, own, nlow))
        last = recs[base + nfit - 1]
        out.append(("step", d0, last[0] + last[1] - d0, rs))
        base += nfit
    return out


def publications(steps):
    """Progress values a linked block publishes (every PUBLISH_EVERY steps; lone steps do not count): the destination of
    the next record after the 4th, 8th, ... step."""
    pub, cnt = [], 0
    for i, (kind, *_r) in enumerate(steps):
        if kind != "step":
            continue
        cnt += 1
        if cnt % PUBLISH_EVERY == 0 and i + 1 < len(steps):
            pub.append(steps[i + 1][1])
    return pub


# ---------------------------------------------------------------------------------------------------- cases
def _rand_rows(rng, n, pos, hist, small=True):
    """n random sequences starting at block position pos with `hist` bytes of history: short literal runs, short
    matches, offsets inside the reachable window."""
    rows = []
    for _ in range(n):
        ll = int(rng.integers(0, 9)) if small else int(rng.choice([rng.integers(0, 11), rng.integers(20, 80), rng.integers(200, 400)], p=None))
        pos += ll
        reach = min(pos + hist, 65535)
        if reach < 1:
            ll += 1; pos += 1; reach = min(pos + hist, 65535)
        ml = int(rng.integers(4, 41))
        rows.append((ll, int(rng.integers(1, reach + 1)), ml))
        pos += ml
    return rows


def c_lengths():
    lls = list(range(0, 15)) + [15, 16, 17, 63, 64, 256, 257, 269, 270, 524, 525, 1000]
    mls = list(range(4, 19)) + [19, 273, 274, 528, 529, 1000]
    offs = [1, 7, 16, 100, 1000, 3000]
    rows = [(32, 5, 10)]
    for i in range(2 * len(lls)):
        ll, ml = lls[i % len(lls)], mls[i % len(mls)]
        rows.append((ll, min(offs[i % len(offs)], regen(rows) + ll), ml))
    b0 = close(rows, BLKMAX[4])
    b1 = [(40, 3, 300), (0, 40, 524)] + rows[1:20] + [(300, 0, 0)]
    return [dict(blocks=[b0, b1], csize=True, cchk=True)]


def c_window():
    rng = np.random.default_rng(11)
    blocks = []
    for b in range(3):
        rows = [(16, 4, 8)] + [(int(rng.integers(0, 4)), 16, int(rng.integers(4, 19))) for _ in range(300)]
        while regen(rows) < 50000:
            p = regen(rows)
            ll = int(rng.choice([rng.integers(0, 11), rng.integers(0, 11), rng.integers(20, 80), rng.integers(200, 400)]))
            ml = int(rng.integers(4, 41))
            rows.append((ll, int(rng.integers(1, min(p + ll, 65535) + 1)), ml))
        blocks.append(close(rows, BLKMAX[4]) if b < 2 else rows + [(37, 0, 0)])
    return [dict(blocks=blocks, cchk=True)]


def c_dense():
    rng = np.random.default_rng(12)
    blocks = []
    for b in range(4):
        rows = [(8, 8, 4)] if b == 0 else []
        while regen(rows) < BLKMAX[4] - 5 - 40:
            rows.append((0, int(rng.integers(1, 65536)) if b else int(rng.integers(1, 9)), int(rng.integers(4, 19))))
        r = BLKMAX[4] - 5 - regen(rows)
        while r:                                            # finish with 3-byte sequences; the last match starts 12 bytes before the end
            m = r if r <= 18 else min(18, r - 7)
            rows.append((0, 1, m)); r -= m
        blocks.append(rows + [(5, 0, 0)])
    return [dict(blocks=blocks, linked=True)]


def c_periods():
    rows = [(70000, 1, 4)]
    rows += [(3, off, 100) for off in range(1, 34)]
    rows += [(2, off, ml) for ml in (8, 20, 33, 100) for off in (ml - 1, ml, ml + 1)]
    rows += [(2, off, 3000) for off in (1, 31, 32, 33, 2047, 65535)]
    b1 = rows[1:] + [(16, 0, 0)]
    b1[0] = (65600, 1, 100)
    return [dict(blocks=[close(rows, BLKMAX[5]), b1], bsid=5, csize=True)]


def c_steps():
    lone = (0, 2500, 3000)
    rows = [(3000, 1000, 4), lone]
    rows += [(0, 2500, 512)] * 4 + [(1, 2500, 4)]           # a step spanning exactly 2048 bytes; the next record starts at 2049
    rows += [lone, (0, 3000, 20)] + [(2, 3000, ml) for ml in range(4, 34)]     # own-lane sources below d0; ml 32 / 33
    rows += [lone, (0, 3000, 8), (4, 20, 8)]                # source ends exactly at the step's first destination
    rows += [lone, (0, 3000, 8), (4, 19, 8)]                # ... one byte later: dependent
    return [dict(blocks=[close(rows, BLKMAX[4]), rows[:8] + [(20, 0, 0)]])]


def c_linked():
    rng = np.random.default_rng(14)
    dists = [1, 2, 3, 4, 7, 8, 31, 32, 33, 255, 256, 2047, 2048, 4096, 32768, 65534, 65535]
    blocks = []
    for b in range(64):
        if b == 0:
            head = [(5, 5, 4)]                              # offset == op + hist (hist 0 in block 0)
        elif b == 20:                                       # a match longer than LZX_SPAN reading the previous block
            head = [(0, 8, 20), (0, 60000, 3000)]
        else:                                               # the predecessor at distance D, then its last 4 bytes
            head = [(0, dists[b % len(dists)], 4), (0, 8, 20)]
        rows = head + _rand_rows(rng, 400, regen(head), 65536 if b else 0)
        blocks.append(close(rows, BLKMAX[4], pos0=65536 if b else 0) if b < 63 else rows + [(16, 0, 0)])
    big = []
    for bsid in (5, 6, 7):
        n = BLKMAX[bsid]
        b0 = close([(64, 8, 100)] + _rand_rows(rng, 200, 164, 0), n)
        b1 = [(0, 8, 20), (0, 65535, 100), (0, 3000, 2600)] + _rand_rows(rng, 200, 2720, 65536) + [(16, 0, 0)]
        big.append(dict(blocks=[b0, b1], bsid=bsid, linked=True))
    stored = [close([(64, 8, 100)], BLKMAX[4]), close([(0, 10, 50), (3, 65535, 40)], BLKMAX[4], pos0=65536),
              [(0, 7, 30), (0, 65535, 100), (16, 0, 0)]]
    return [dict(blocks=blocks, linked=True, cchk=True), dict(blocks=stored, linked=True, stored={0, 1})] + big


def c_ends():
    out = [dict(blocks=[[(20, 10, 30), (3, 9, 7), (5, 0, 0)]]),                      # last match 12 bytes before the end
           dict(blocks=[[(20, 10, 30), (300, 0, 0)]], csize=True)]                    # extended last literal run
    out += [dict(blocks=[close([(16, 8, 4)], BLKMAX[s])], bsid=s) for s in (4, 5, 6, 7)]
    out += [dict(blocks=[], csize=True, cchk=True), dict(blocks=[], dict_id=0x12345678),
            dict(blocks=[[(20, 10, 30), (12, 0, 0)]], dict_id=0xCAFEF00D, cchk=True)]
    # zero-size stored blocks (header 0x80000000): between full blocks, and as the last block before the end mark
    out += [dict(blocks=[close([(16, 8, 4)], BLKMAX[4]), [], [(20, 10, 30), (12, 0, 0)]], stored={1}, cchk=True),
            dict(blocks=[[(20, 10, 30), (12, 0, 0)], []], stored={1}, csize=True)]
    return out


CASES = {"lengths": c_lengths, "window": c_window, "dense": c_dense, "periods": c_periods, "steps": c_steps,
         "linked": c_linked, "ends": c_ends}
LAYOUTS = ("full", "short")


@functools.lru_cache(maxsize=None)
def case(name, lay="full", bchk=False):
    """[(frame, source, per-block info)] of one case in one layout; bchk: written with FLG.BC."""
    out = []
    for i, spec in enumerate(CASES[name]()):
        s = layout(spec, lay)
        if bchk:
            s = dict(s, bchk=True)
        out.append(write_frame(s, seed=1000 * i + len(name)))
    return out


@functools.lru_cache(maxsize=None)
def traces(name, lay="full"):
    return [o.lz4f_trace(f, s.size) for f, s, _ in case(name, lay)]


def block_view(tr, b, abs_base=12):
    """One block of a trace, in the models' terms: (block-relative token positions, block size, match records
    (d, ml, off), absolute input offset of the block data when the frame sits behind a 12-byte header at abs_base - 12)."""
    sq = tr.block_seqs(b)
    foff = int(tr.blk[b, o.L4B["foff"]])
    tok = [int(t) - foff for t in sq[:, o.L4S["tokpos"]]]
    recs = [(int(r[o.L4S["dst"]]), int(r[o.L4S["ml"]]), int(r[o.L4S["off"]])) for r in sq if r[o.L4S["ml"]]]
    return tok, int(tr.blk[b, o.L4B["bsize"]]), recs, abs_base + foff


def expect_path_is_sequential(lay, tr):
    """What the layouts promise: a `short` frame of two or more blocks, and any frame with a zero-size block, goes to the
    frame-sequential pass; every other frame stays on the two-pass path."""
    return (lay == "short" and len(tr.blk) > 1) or bool((tr.col("bsize") == 0).any())


def expect_fallback(tr, bsid):
    """The frame-sequential pass takes a frame iff a non-last block does not regenerate blockMaxSize (or a block is empty)."""
    rg = tr.col("regen")
    return bool((rg[:-1] != BLKMAX[bsid]).any() or (tr.col("bsize") == 0).any())
