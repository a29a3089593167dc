"""The zstd search class of levels 6-12 (zstdmt_b200/csrc/zstd_lazy_rule.h) restated in Python, and the binding of its
C twin (oracle/chain_twin.c, built into oracle/libchain_twin.so).

The restatement keeps the chains as a dict of position lists and finds best[] by brute force over them; it is slow and
meant for inputs of up to about 100 KiB.  Both return, per block, the merged sequences as (literal length, offset,
match length)."""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLOCK, LCAP, HASHLOG, LEN_BITS = 16384, 256, 22, 9
PARAMS = {6: (5, 8, 1), 7: (5, 16, 1), 8: (5, 16, 2), 9: (5, 32, 2), 10: (5, 48, 2), 11: (5, 56, 2), 12: (5, 64, 2)}
M64 = (1 << 64) - 1


def params(level):
    """(minMatch, chain depth, lazy depth); levels above 12 use level 12's row."""
    return PARAMS[min(max(level, 6), 12)]


def window(level):
    return 1 << 22 if min(level, 12) >= 10 else 1 << 21


def hash_(v, mm):
    if mm == 4:
        return ((v * 2654435761) & 0xFFFFFFFF) >> (32 - HASHLOG)
    return ((((v << 24) & M64) * 889523592379) & M64) >> (64 - HASHLOG)


def gain(length, off):
    return 4 * length - ((off + 3).bit_length() - 1)


def _match_len(src, q, p, cap):
    if src[q: q + cap] == src[p: p + cap]:
        return cap
    lo, hi = 0, cap                      # equal for lo bytes, not for hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if src[q: q + mid] == src[p: p + mid]:
            lo = mid
        else:
            hi = mid
    return lo


def sequences(data, level, W=None, block=BLOCK):
    """Per block, the list of merged sequences (literal length, offset, match length) of one chunk."""
    src = bytes(np.ascontiguousarray(data, dtype=np.uint8).tobytes())
    mm, depth, lazy = params(level)
    W = W or window(level)
    n = len(src)
    chains, rank = {}, [0] * n           # rank[p]: index of p in its hash's list
    key = [None] * n
    for p in range(n - mm + 1):
        k = hash_(int.from_bytes(src[p: p + mm], "little"), mm)
        lst = chains.setdefault(k, [])
        key[p], rank[p] = k, len(lst)
        lst.append(p)
    out = []
    for b0 in range(0, n, block):
        b1 = min(b0 + block, n)
        best = {}
        for p in range(b0, b1 - mm + 1):
            cap = min(LCAP, b1 - p)
            lst = chains[key[p]]
            bl = bo = 0
            for q in reversed(lst[max(0, rank[p] - depth): rank[p]]):      # the depth nearest earlier positions
                if p - q > W:
                    break
                ln = _match_len(src, q, p, cap)
                if ln >= mm and ln > bl:
                    bl, bo = ln, p - q
            if bl:
                best[p] = (bl, bo)
        seqs, anchor, p = [], b0, b0
        while p < b1:
            m = best.get(p)
            if m is None:
                p += 1
                continue
            g = gain(*m)
            m1, m2 = best.get(p + 1), best.get(p + 2)
            if (m1 and gain(*m1) > g + 4) or (lazy >= 2 and m2 and gain(*m2) > g + 7):
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


def replay(data, blocks, block=BLOCK):
    """Rebuild the content from each block's sequences, the literal bytes taken from `data` where no match covers them."""
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
        assert p <= b1
        out += src[p: b1]
    return bytes(out)


_twin = None


def twin():
    global _twin
    if _twin is None:
        L = ctypes.CDLL(os.path.join(ROOT, "oracle", "libchain_twin.so"))
        L.orc_zstd_lazy_sequences.restype = ctypes.c_long
        L.orc_zstd_lazy_sequences.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32,
                                              ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
        L.orc_zstd_lazy_best.restype = ctypes.c_int
        L.orc_zstd_lazy_best.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p]
        _twin = L
    return _twin


def twin_best(data, level, W=0, block=0):
    """orc_zstd_lazy_best: the chunk's best[] (uint32, length | offset << LEN_BITS, 0: no match)."""
    src = np.ascontiguousarray(data, dtype=np.uint8)
    best = np.zeros(max(int(src.size), 1), np.uint32)
    if twin().orc_zstd_lazy_best(src.ctypes.data, src.size, level, W, block, best.ctypes.data) != 0:
        raise RuntimeError("orc_zstd_lazy_best failed")
    return best[: src.size]


def twin_sequences(data, level, W=0, block=0):
    """orc_zstd_lazy_sequences: per block, an (n, 3) uint32 array of (literal length, offset, match length)."""
    src = np.ascontiguousarray(data, dtype=np.uint8)
    n = int(src.size)
    nb = -(-n // (block or BLOCK))
    ms = n // 4 + 2
    seq = np.empty((ms, 3), np.uint32)
    per = np.zeros(max(nb, 1), np.uint32)
    r = twin().orc_zstd_lazy_sequences(src.ctypes.data, n, level, W, block, seq.ctypes.data, ms, per.ctypes.data, per.size)
    if r < 0:
        raise RuntimeError("orc_zstd_lazy_sequences failed")
    starts = np.concatenate([[0], np.cumsum(per[:nb].astype(np.int64))])
    return [seq[starts[b]: starts[b + 1]] for b in range(nb)]
