"""The LZ4 high-compression class of levels 10-12 (zstdmt_b200/csrc/lz4_hc_rule.h) restated in Python, and the
binding of its C twin (oracle/lz4_hc_twin.c, built into oracle/liblz4hc_twin.so).

The restatement keeps the chains as a dict of position lists and finds best[] by brute force over them; it is slow and
meant for inputs of up to about 100 KiB.  Both give, per block, the merged sequences as (literal length, offset, match
length); the twin also writes whole framed streams, and `frame` here encodes the restatement's sequences the same way."""
import ctypes
import os
import struct

import numpy as np

from _zlazy import _match_len, hash_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLOCK, LCAP, MINMATCH, MFLIMIT, LASTLIT, WINDOW, LEN_BITS = 65536, 256, 4, 12, 5, 65535, 9
PARAMS = {10: (64, 2), 11: (128, 2), 12: (256, 2)}          # (chain depth, lazy depth)
LEVELS = sorted(PARAMS)


def sequences(data, level, W=None, block=BLOCK):
    """Per block, the list of merged sequences (literal length, offset, match length) of one chunk."""
    src = bytes(np.ascontiguousarray(data, dtype=np.uint8).tobytes())
    depth, lazy = PARAMS[level]
    W = W or WINDOW
    n = len(src)
    chains, rank, key = {}, [0] * n, [None] * n            # rank[p]: index of p in its hash's list
    for p in range(n - MINMATCH + 1):
        k = hash_(int.from_bytes(src[p: p + MINMATCH], "little"), MINMATCH)
        lst = chains.setdefault(k, [])
        key[p], rank[p] = k, len(lst)
        lst.append(p)
    out = []
    for b0 in range(0, n, block):
        b1 = min(b0 + block, n)
        best = {}
        for p in range(b0, b1 - MFLIMIT + 1):
            cap = min(LCAP, b1 - LASTLIT - p)
            lst = chains[key[p]]
            bl = bo = 0
            for q in reversed(lst[max(0, rank[p] - depth): rank[p]]):      # the depth nearest earlier positions
                if p - q > W:
                    break
                ln = _match_len(src, q, p, cap)
                if ln >= MINMATCH and ln > bl:
                    bl, bo = ln, p - q
            if bl:
                best[p] = (bl, bo)
        L = lambda q: best[q][0] if q in best else 0
        seqs, anchor, p = [], b0, b0
        while p < b1:
            m = best.get(p)
            if m is None or L(p + 1) > m[0] + 1 or (lazy >= 2 and L(p + 2) > m[0] + 2):
                p += 1
                continue
            ln, off = m
            if p == anchor and seqs and seqs[-1][1] == off:
                seqs[-1] = (seqs[-1][0], off, seqs[-1][2] + ln)
            else:
                seqs.append((p - anchor, off, ln))
            p += ln
            anchor = p
        out.append(seqs)
    return out


def _lenbytes(x):
    return b"\xff" * (x // 255) + bytes([x % 255])


def encode_block(blk, seqs):
    """The LZ4 block of `blk` (bytes) from its sequences, the last sequence literals only."""
    out, pos = bytearray(), 0
    for ll, off, ml in seqs:
        m = ml - MINMATCH
        out.append((min(ll, 15) << 4) | min(m, 15))
        if ll >= 15:
            out += _lenbytes(ll - 15)
        out += blk[pos: pos + ll]
        out += struct.pack("<H", off)
        if m >= 15:
            out += _lenbytes(m - 15)
        pos += ll + ml
    ll = len(blk) - pos
    out.append(min(ll, 15) << 4)
    if ll >= 15:
        out += _lenbytes(ll - 15)
    out += blk[pos:]
    return bytes(out)


def frame(data, level, xxh32):
    """One chunk as the class frames it (12-byte container header included), from the restatement's sequences;
    xxh32: a function of bytes (the oracle's)."""
    src = bytes(np.ascontiguousarray(data, dtype=np.uint8).tobytes())
    n = len(src)
    hdr = bytes([0x4C if n else 0x44, 0x40]) + (struct.pack("<Q", n) if n else b"")
    body = bytearray(struct.pack("<I", 0x184D2204) + hdr + bytes([(xxh32(hdr) >> 8) & 0xFF]))
    for b, seqs in enumerate(sequences(data, level) if n else []):
        blk = src[b * BLOCK: (b + 1) * BLOCK]
        enc = encode_block(blk, seqs)
        body += struct.pack("<I", len(enc)) + enc if len(enc) < len(blk) else struct.pack("<I", len(blk) | 0x80000000) + blk
    body += struct.pack("<II", 0, xxh32(src))
    return struct.pack("<III", 0x184D2A50, 4, len(body)) + bytes(body)


def replay(data, blocks, block=BLOCK):
    """Rebuild the content from each block's sequences, the literal bytes taken from `data` where no match covers them;
    matches may reach into earlier blocks (linked blocks)."""
    src = bytes(np.ascontiguousarray(data, dtype=np.uint8).tobytes())
    out = bytearray()
    for i, seqs in enumerate(blocks):
        b0, b1 = i * block, min((i + 1) * block, len(src))
        p = b0
        for ll, off, ml in seqs:
            out += src[p: p + ll]
            p += ll
            assert 1 <= off <= len(out)
            for _ in range(ml):
                out.append(out[-off])
            p += ml
        assert not seqs or p <= b1 - LASTLIT
        out += src[p: b1]
    return bytes(out)


def _getlen(b, i, x):
    if x == 15:
        while True:
            c = b[i]; i += 1; x += c
            if c != 255:
                break
    return x, i


def parse_block(b):
    """Sequences (literal length, offset, match length) of an LZ4 block and its trailing literal count."""
    seqs, i = [], 0
    while True:
        tok = b[i]; i += 1
        ll, i = _getlen(b, i, tok >> 4)
        i += ll
        if i == len(b):
            return seqs, ll
        off = b[i] | (b[i + 1] << 8); i += 2
        ml, i = _getlen(b, i, tok & 15)
        seqs.append((ll, off, ml + MINMATCH))


def parse_stream(framed):
    """Every frame of a framed stream: (FLG, BD, [(raw, content bytes, sequences or None)]) per frame."""
    b = bytes(np.ascontiguousarray(framed, dtype=np.uint8).tobytes())
    frames, pos = [], 0
    while pos < len(b):
        magic, four, cs = struct.unpack_from("<III", b, pos)
        assert magic == 0x184D2A50 and four == 4
        f = b[pos + 12: pos + 12 + cs]
        assert struct.unpack_from("<I", f, 0)[0] == 0x184D2204
        flg, bd = f[4], f[5]
        i = 4 + 2 + (8 if flg & 8 else 0) + 1
        blocks = []
        while True:
            h = struct.unpack_from("<I", f, i)[0]; i += 4
            if h == 0:
                break
            sz = h & 0x7FFFFFFF
            if h >> 31:
                blocks.append((True, sz, None))
            else:
                seqs, last = parse_block(f[i: i + sz])
                blocks.append((False, sum(a + c for a, _, c in seqs) + last, seqs))
            i += sz
        assert i + 4 == len(f)
        frames.append((flg, bd, blocks))
        pos += 12 + cs
    return frames


def check_structure(framed, parts):
    """The class's frame layout, frame by frame against the chunk contents `parts`: FLG 0x4C (0x44 empty), BD 0x40,
    64 KiB blocks (the last one may be short), offsets <= 65535 and within the chunk, match starts <= blockEnd - 12,
    matches end at or before blockEnd - 5.  Returns the number of matches that reach into an earlier block."""
    frames = parse_stream(framed)
    assert len(frames) == len(parts)
    back = 0
    for (flg, bd, blocks), content in zip(frames, parts):
        n = int(np.asarray(content).size)
        assert (flg, bd) == ((0x4C if n else 0x44), 0x40)
        assert [c for _, c, _ in blocks] == [min(BLOCK, n - i) for i in range(0, n, BLOCK)]
        for k, (raw, bn, seqs) in enumerate(blocks):
            if raw:
                continue
            b0, p = k * BLOCK, k * BLOCK
            for ll, off, ml in seqs:
                p += ll
                assert 1 <= off <= WINDOW and off <= p
                assert p + MFLIMIT <= b0 + bn and p + ml <= b0 + bn - LASTLIT
                back += p - off < b0
                p += ml
    return back


_twin = None


def twin():
    global _twin
    if _twin is None:
        L = ctypes.CDLL(os.path.join(ROOT, "oracle", "liblz4hc_twin.so"))
        L.orc_lz4_hc_sequences.restype = ctypes.c_long
        L.orc_lz4_hc_sequences.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32,
                                           ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
        L.orc_lz4_hc_compress.restype = ctypes.c_size_t
        L.orc_lz4_hc_compress.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t]
        _twin = L
    return _twin


def twin_sequences(data, level, W=0, block=0):
    """orc_lz4_hc_sequences: per block, an (n, 3) uint32 array of (literal length, offset, match length)."""
    src = np.ascontiguousarray(data, dtype=np.uint8)
    n = int(src.size)
    nb = -(-n // (block or BLOCK))
    ms = n // 4 + 2
    seq = np.empty((ms, 3), np.uint32)
    per = np.zeros(max(nb, 1), np.uint32)
    r = twin().orc_lz4_hc_sequences(src.ctypes.data, n, level, W, block, seq.ctypes.data, ms, per.ctypes.data, per.size)
    if r < 0:
        raise RuntimeError("orc_lz4_hc_sequences failed")
    starts = np.concatenate([[0], np.cumsum(per[:nb].astype(np.int64))])
    return [seq[starts[b]: starts[b + 1]] for b in range(nb)]


def twin_compress(data, chunk, level):
    """orc_lz4_hc_compress: the framed stream of `data` cut every `chunk` bytes."""
    src = np.ascontiguousarray(data, dtype=np.uint8)
    n = int(src.size)
    nch = max(1, -(-n // chunk))
    cap = n + nch * (64 + 300 * (chunk // BLOCK + 1)) + 4096
    out = np.empty(cap, np.uint8)
    r = twin().orc_lz4_hc_compress(src.ctypes.data if n else None, n, chunk, level, out.ctypes.data, cap)
    if r == 0:
        raise RuntimeError("orc_lz4_hc_compress failed")
    return out[:r].copy()
