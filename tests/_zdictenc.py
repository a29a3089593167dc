"""The zstd search class of levels 6-12 compressing against a dictionary (zmt_zstd_compress_dict_device; rule:
zstdmt_b200/csrc/zstd_lazy_rule.h), restated in Python, the binding of its C twin (zstdmt_b200/harness/zlazy_dict_twin.c)
and the framed stream the GPU writes, built on the CPU from the twin's sequences and the entropy twin (_zenc).

A dictionary here is its content D: the whole buffer for raw content, the bytes behind the entropy section for a
formatted one (content()).  The chains run over D followed by the chunk; a dictionary candidate q lies p + len(D) - q
back, and its match ends at the end of D at the latest.  Both restatements count the edges of the walk (EDGES) into an
optional `stats` array, for the tests to show that a corpus reaches them."""
import ctypes
import os

import numpy as np

import _zenc as ze
import _zlazy as zl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLOCK, LCAP = zl.BLOCK, zl.LCAP
DICT_MAGIC = 0xEC30A437
# the counters of zlazy_dict_twin.c's ZDT_* enum, in order
EDGES = ("switch_after_0", "switch_after_depth_minus_1", "depth_used_in_chunk", "dist_W", "dist_W_plus_1", "capped_then_longer",
         "skip_at_dict_end")


def content(d):
    """The content of dictionary `d` (formatted: behind its entropy section, as libzstd's ZDICT_getDictHeaderSize says;
    raw: all of it)."""
    import _zdict as zd
    d = np.ascontiguousarray(d, np.uint8)
    if d.size >= 8 and int(d[:4].view("<u4")[0]) == DICT_MAGIC:
        L = zd.zstd()
        L.ZDICT_getDictHeaderSize.restype = ctypes.c_size_t
        L.ZDICT_getDictHeaderSize.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
        h = L.ZDICT_getDictHeaderSize(d.ctypes.data, d.size)
        assert not zd.err(h), "ZDICT_getDictHeaderSize refused the dictionary"
        return d[h:].copy()
    return d.copy()


def _hashes(buf, mm):
    """h(p) of every p with p + mm <= len(buf) (numpy: the multiply wraps at 64 bits as the C one does)."""
    n = len(buf) - mm + 1
    if n <= 0:
        return np.zeros(0, np.uint64)
    b = np.frombuffer(buf, np.uint8).astype(np.uint64)
    v = np.zeros(n, np.uint64)
    for k in range(mm):
        v |= b[k: k + n] << np.uint64(8 * k)
    return ((v << np.uint64(24)) * np.uint64(889523592379)) >> np.uint64(64 - zl.HASHLOG)


def _match_len(buf, q, g, cap):
    return zl._match_len(buf, q, g, cap) if cap > 0 else 0


def sequences(data, level, dictionary=None, W=None, block=BLOCK, stats=None):
    """Per block, the merged sequences (literal length, offset, match length) of one chunk compressed against the
    content `dictionary` (None or empty: the rule without a dictionary, _zlazy.sequences)."""
    src = bytes(np.ascontiguousarray(data, dtype=np.uint8).tobytes())
    D = bytes(np.ascontiguousarray(dictionary if dictionary is not None else [], dtype=np.uint8).tobytes())
    mm, depth, lazy = zl.params(level)
    W = W or zl.window(level)
    dlen, n = len(D), len(src)
    buf = D + src
    ch, dh = _hashes(src, mm), _hashes(D, mm)            # chunk positions; linked dictionary positions (q + mm <= dlen)
    chains = {}
    if dh.size and ch.size:
        for q in np.flatnonzero(np.isin(dh, ch)).tolist():
            chains.setdefault(int(dh[q]), []).append(q)
    rank = [0] * n
    for p, h in enumerate(ch.tolist()):
        lst = chains.setdefault(h, [])
        rank[p] = len(lst)
        lst.append(dlen + p)
    out = []
    for b0 in range(0, n, block):
        b1 = min(b0 + block, n)
        best = {}
        for p in range(b0, b1 - mm + 1):
            g, cap = dlen + p, min(LCAP, b1 - p)
            lst = chains[int(ch[p])]
            bl = bo = 0
            chunk_steps, in_dict, capped, steps, stopped = 0, False, False, 0, False
            for q in reversed(lst[max(0, rank[p] - depth): rank[p]]):      # the depth nearest earlier positions
                dist = g - q
                if q < dlen and not in_dict:
                    in_dict = True
                    if stats is not None and chunk_steps == 0:
                        stats[0] += 1
                    if stats is not None and depth > 1 and chunk_steps == depth - 1:
                        stats[1] += 1
                if dist > W:
                    if stats is not None and q < dlen and dist == W + 1:
                        stats[4] += 1
                    stopped = True
                    break
                steps += 1
                if q >= dlen:
                    chunk_steps += 1
                qcap = min(cap, dlen - q) if q < dlen else cap
                if q < dlen and bl and bl >= qcap:
                    if stats is not None:
                        stats[6] += 1
                    continue
                if stats is not None and q < dlen and dist == W:
                    stats[3] += 1
                ln = _match_len(buf, q, g, qcap)
                if ln >= mm and ln > bl:
                    if stats is not None and capped:
                        stats[5] += 1
                    capped = q < dlen and ln == qcap < cap
                    bl, bo = ln, dist
                    if ln == cap:
                        stopped = True
                        break
            if stats is not None and not stopped and steps == depth and not in_dict and rank[p] > depth:
                q = lst[rank[p] - depth - 1]                               # the next candidate the depth did not reach
                if q < dlen and g - q <= W:
                    stats[2] += 1
            if bl:
                best[p] = (bl, bo)
        seqs, anchor, p = [], b0, b0
        while p < b1:
            m = best.get(p)
            if m is None:
                p += 1
                continue
            gn = zl.gain(*m)
            m1, m2 = best.get(p + 1), best.get(p + 2)
            if (m1 and zl.gain(*m1) > gn + 4) or (lazy >= 2 and m2 and zl.gain(*m2) > gn + 7):
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


def replay(data, blocks, dictionary=None, block=BLOCK):
    """Rebuild the content from each block's sequences with `dictionary`'s content before it; literal bytes from `data`."""
    src = bytes(np.ascontiguousarray(data, dtype=np.uint8).tobytes())
    D = bytes(np.ascontiguousarray(dictionary if dictionary is not None else [], dtype=np.uint8).tobytes())
    out = bytearray(D)
    for i, seqs in enumerate(blocks):
        p = i * block
        for ll, off, ml in seqs:
            out += src[p: p + ll]
            p += ll
            assert 1 <= off <= len(out)
            for _ in range(ml):
                out.append(out[-off])
            p += ml
        out += src[p: min((i + 1) * block, len(src))]
    return bytes(out[len(D):])


_twin = None


def twin():
    global _twin
    if _twin is None:
        L = ctypes.CDLL(os.path.join(ROOT, "zstdmt_b200", "libzlazy_dict_twin.so"))
        vp, sz, u32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32
        L.orc_zstd_lazy_sequences_dict.restype = ctypes.c_long
        L.orc_zstd_lazy_sequences_dict.argtypes = [vp, sz, vp, sz, ctypes.c_int, u32, u32, vp, sz, vp, sz, vp]
        L.orc_zstd_lazy_best_dict.restype = ctypes.c_int
        L.orc_zstd_lazy_best_dict.argtypes = [vp, sz, vp, sz, ctypes.c_int, u32, u32, vp, vp]
        _twin = L
    return _twin


def _arr(x):
    return np.ascontiguousarray(x if x is not None else np.zeros(0, np.uint8), dtype=np.uint8)


def twin_best(data, level, dictionary=None, W=0, block=0, stats=None):
    """orc_zstd_lazy_best_dict: the chunk's best[] (uint32, length | offset << 9, 0: no match)."""
    src, d = _arr(data), _arr(dictionary)
    best = np.zeros(max(int(src.size), 1), np.uint32)
    st = stats if stats is not None else np.zeros(len(EDGES), np.uint64)
    if twin().orc_zstd_lazy_best_dict(d.ctypes.data, d.size, src.ctypes.data, src.size, level, W, block, best.ctypes.data, st.ctypes.data):
        raise RuntimeError("orc_zstd_lazy_best_dict failed")
    return best[: src.size]


def twin_sequences(data, level, dictionary=None, W=0, block=0, stats=None):
    """orc_zstd_lazy_sequences_dict: per block, an (n, 3) uint32 array of (literal length, offset, match length).
    stats: None or a uint64 array of len(EDGES) counters, added to."""
    src, d = _arr(data), _arr(dictionary)
    n = int(src.size)
    nb = -(-n // (block or BLOCK))
    ms = n // 4 + 2
    seq = np.empty((ms, 3), np.uint32)
    per = np.zeros(max(nb, 1), np.uint32)
    st = stats if stats is not None else np.zeros(len(EDGES), np.uint64)
    assert st.dtype == np.uint64 and st.size == len(EDGES)
    r = twin().orc_zstd_lazy_sequences_dict(d.ctypes.data, d.size, src.ctypes.data, n, level, W, block, seq.ctypes.data, ms,
                                            per.ctypes.data, per.size, st.ctypes.data)
    if r < 0:
        raise RuntimeError("orc_zstd_lazy_sequences_dict failed")
    starts = np.concatenate([[0], np.cumsum(per[:nb].astype(np.int64))])
    return [seq[starts[b]: starts[b + 1]] for b in range(nb)]


def did_bytes(dict_id):
    """Size of the Dictionary_ID field libzstd writes for dict_id: none for 0, then 1, 2 or 4 bytes."""
    return 0 if dict_id == 0 else 1 if dict_id < 256 else 2 if dict_id < 65536 else 4


def frame_header(n, dict_id=0):
    """_zenc.frame_header with the Dictionary_ID field: FHD bits 0-1 = 1, 2, 3 for a 1, 2, 4-byte ID, the ID before
    Frame_Content_Size."""
    h = ze.frame_header(n)
    dl = did_bytes(dict_id)
    if not dl:
        return h
    return h[:4] + bytes([h[4] | {1: 1, 2: 2, 4: 3}[dl]]) + dict_id.to_bytes(dl, "little") + h[5:]


def framed_b200(src, chunk, level, chunk_bytes=None, dictionary=None, dict_id=0, blocks=None):
    """The framed stream zmt_zstd_compress_dict_device writes at `level` (6-22) against content `dictionary`, naming
    dict_id: _zenc.framed_b200's layout with the dictionary's sequences and header.  blocks: as in _zenc.framed_b200."""
    src = np.ascontiguousarray(src, dtype=np.uint8)
    out = []
    for c, cont in enumerate(ze.chunks(src, chunk, chunk_bytes)):
        body = []
        n = int(cont.size)
        for b, rows in enumerate(twin_sequences(cont, level, dictionary) if n else []):
            b0, b1 = b * BLOCK, min((b + 1) * BLOCK, n)
            blk, tr = ze.block_b200(rows.astype(np.int64), ze.literals_of(cont[b0:b1], rows), cont[b0:b1], b1 == n)
            body.append(blk.tobytes())
            if blocks is not None:
                blocks.append((c, b, tr))
        if n == 0:
            body.append(bytes([1, 0, 0]))
        frame = frame_header(n, dict_id) + b"".join(body)
        out.append((0x184D2A50).to_bytes(4, "little") + (4).to_bytes(4, "little") + len(frame).to_bytes(4, "little") + frame)
    return np.frombuffer(b"".join(out), np.uint8)


def frames(stream):
    """The zstd frames of a container stream (12-byte headers stripped)."""
    s = np.asarray(stream, np.uint8)
    out, pos = [], 0
    while pos < s.size:
        sz = int(s[pos + 8: pos + 12].view("<u4")[0])
        out.append(s[pos + 12: pos + 12 + sz])
        pos += 12 + sz
    return out
