"""zstd dictionaries and frames written against them by the image's libzstd (libzstd.so.1), for the dictionary tests.

Dictionaries come from fixed seeds: trained (ZDICT_trainFromBuffer), finalized from chosen content (ZDICT_finalizeDictionary)
or raw content.  Frames come from ZSTD_compress2 on a context with the dictionary loaded (libzstd's own parse), or from
ZSTD_compressSequences on such a context with a parse the test dictates, whose offsets may reach into the dictionary's
content.  libzstd's ZSTD_decompress_usingDict is the reference decoder."""
import ctypes
import functools

import numpy as np

import _zcorpus as zc

c_sz, c_vp, c_int, c_uint = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int, ctypes.c_uint

P_CONTENTSIZE, P_CHECKSUM, P_DICTID = 200, 201, 202             # ZSTD_c_contentSizeFlag, ZSTD_c_checksumFlag, ZSTD_c_dictIDFlag
DCT_AUTO, DCT_RAW, DCT_FULL = 0, 1, 2                           # ZSTD_dictContentType_e
DICT_MAGIC = 0xEC30A437
ZB_SELF, ZB_PREDEF, ZB_NONE, ZB_DICT = 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD, 0xFFFFFFFC
ZF_NEEDS_SEQ, ZF_DICT = 1, 8


class ZdictParams(ctypes.Structure):
    _fields_ = [("compressionLevel", c_int), ("notificationLevel", c_uint), ("dictID", c_uint)]


def err(r):
    return r > (1 << 63)


@functools.lru_cache(maxsize=None)
def zstd():
    L = zc.zstd()
    L.ZDICT_trainFromBuffer.restype = c_sz
    L.ZDICT_trainFromBuffer.argtypes = [c_vp, c_sz, c_vp, ctypes.POINTER(c_sz), c_uint]
    L.ZDICT_finalizeDictionary.restype = c_sz
    L.ZDICT_finalizeDictionary.argtypes = [c_vp, c_sz, c_vp, c_sz, c_vp, ctypes.POINTER(c_sz), c_uint, ZdictParams]
    L.ZDICT_isError.restype = c_uint; L.ZDICT_isError.argtypes = [c_sz]
    L.ZSTD_CCtx_loadDictionary_advanced.restype = c_sz
    L.ZSTD_CCtx_loadDictionary_advanced.argtypes = [c_vp, c_vp, c_sz, c_int, c_int]
    L.ZSTD_createDCtx.restype = c_vp
    L.ZSTD_freeDCtx.argtypes = [c_vp]
    L.ZSTD_decompress_usingDict.restype = c_sz
    L.ZSTD_decompress_usingDict.argtypes = [c_vp, c_vp, c_sz, c_vp, c_sz, c_vp, c_sz]
    L.ZSTD_DCtx_loadDictionary.restype = c_sz
    L.ZSTD_DCtx_loadDictionary.argtypes = [c_vp, c_vp, c_sz]
    return L


def records(seed, count, lo=200, hi=4096):
    """Small records that share vocabulary and layout, as rows or messages do: what dictionaries are for."""
    rng = np.random.default_rng(seed)
    words = [bytes(rng.integers(97, 123, rng.integers(3, 10)).astype(np.uint8)) for _ in range(400)]
    out = []
    for i in range(count):
        n = int(rng.integers(lo, hi + 1))
        parts, size = [], 0
        while size < n:
            w = b'{"id": %d, "name": "%s", "tags": ["%s", "%s"], "v": %d}\n' % (
                int(rng.integers(0, 1 << 20)), words[rng.integers(0, 400)], words[rng.integers(0, 400)], words[rng.integers(0, 40)],
                int(rng.integers(0, 1000)))
            parts.append(w); size += len(w)
        out.append(np.frombuffer(b"".join(parts)[:n], np.uint8))
    return out


def _samples(recs):
    buf = np.concatenate(recs)
    sizes = (c_sz * len(recs))(*[r.size for r in recs])
    return buf, sizes


def train(seed, size, nrec=600):
    """ZDICT_trainFromBuffer on records(seed): a formatted dictionary of at most `size` bytes."""
    L = zstd()
    buf, sizes = _samples(records(seed, nrec))
    out = np.empty(size, np.uint8)
    n = L.ZDICT_trainFromBuffer(out.ctypes.data, size, buf.ctypes.data, sizes, len(sizes))
    assert not L.ZDICT_isError(n), "ZDICT_trainFromBuffer failed"
    return out[:n].copy()


def finalize(seed, content, size, level=3, dict_id=0):
    """ZDICT_finalizeDictionary: `content` as the dictionary's content, entropy tables from records(seed)."""
    L = zstd()
    buf, sizes = _samples(records(seed, 400))
    content = np.ascontiguousarray(content, np.uint8)
    out = np.empty(size, np.uint8)
    n = L.ZDICT_finalizeDictionary(out.ctypes.data, size, content.ctypes.data, content.size, buf.ctypes.data, sizes, len(sizes),
                                   ZdictParams(level, 0, dict_id))
    assert not L.ZDICT_isError(n), "ZDICT_finalizeDictionary failed"
    return out[:n].copy()


def dict_id(d):
    d = np.asarray(d, np.uint8)
    return int(d[4:8].view("<u4")[0]) if d.size >= 8 and int(d[:4].view("<u4")[0]) == DICT_MAGIC else 0


def compress(src, d, level=3, checksum=0, content_size=1, dict_id_flag=1, kind=DCT_AUTO, seqs=None, params=None):
    """One frame of `src` against dictionary `d` (kind: how libzstd reads it)."""
    L = zstd()
    src = np.ascontiguousarray(src, np.uint8)
    d = np.ascontiguousarray(d, np.uint8)
    cctx = L.ZSTD_createCCtx()
    try:
        p = {zc.P_LEVEL: level, P_CHECKSUM: checksum, P_CONTENTSIZE: content_size, P_DICTID: dict_id_flag}
        p.update(params or {})
        for k, v in p.items():
            assert not err(L.ZSTD_CCtx_setParameter(cctx, k, v)), (k, v)
        assert not err(L.ZSTD_CCtx_loadDictionary_advanced(cctx, d.ctypes.data, d.size, 0, kind)), "dictionary refused"
        cap = L.ZSTD_compressBound(src.size) + (1 << 16)
        out = np.empty(cap, np.uint8)
        if seqs is None:
            n = L.ZSTD_compress2(cctx, out.ctypes.data, cap, src.ctypes.data, src.size)
        else:
            a = np.asarray(seqs, dtype=np.int64).reshape(-1, 3)
            arr = (zc.Seq * max(1, len(a)))()
            view = np.frombuffer(arr, dtype=np.uint32).reshape(-1, 4)
            view[: len(a), 0] = a[:, 1]; view[: len(a), 1] = a[:, 0]; view[: len(a), 2] = a[:, 2]; view[:, 3] = 0
            n = L.ZSTD_compressSequences(cctx, out.ctypes.data, cap, arr, len(a), src.ctypes.data, src.size)
        assert not err(n), "libzstd refused the frame (error %d)" % (n - (1 << 64))
        return out[:n].copy()
    finally:
        L.ZSTD_freeCCtx(cctx)


def decompress(frame, d, size):
    """ZSTD_decompress_usingDict: (error flag, bytes)."""
    L = zstd()
    frame = np.ascontiguousarray(frame, np.uint8)
    d = np.ascontiguousarray(d, np.uint8)
    dctx = L.ZSTD_createDCtx()
    try:
        out = np.empty(size + 1, np.uint8)
        n = L.ZSTD_decompress_usingDict(dctx, out.ctypes.data, out.size, frame.ctypes.data, frame.size, d.ctypes.data, d.size)
        return (True, None) if err(n) else (False, out[:n].copy())
    finally:
        L.ZSTD_freeDCtx(dctx)


def libzstd_accepts(d):
    """ZSTD_DCtx_loadDictionary's verdict on `d`."""
    L = zstd()
    d = np.ascontiguousarray(d, np.uint8)
    dctx = L.ZSTD_createDCtx()
    try:
        return not err(L.ZSTD_DCtx_loadDictionary(dctx, d.ctypes.data, d.size))
    finally:
        L.ZSTD_freeDCtx(dctx)


def container(frames):
    """Frames behind 12-byte container headers."""
    out = []
    for f in frames:
        out.append(np.array([0x184D2A50, 4, f.size], "<u4").view(np.uint8)); out.append(f)
    return np.concatenate(out) if out else np.zeros(0, np.uint8)


def plain(frames, seed=0):
    """Frames back to back with skippable frames of random size between some of them."""
    rng = np.random.default_rng(seed)
    out = []
    for i, f in enumerate(frames):
        if i % 3 == 1:
            k = int(rng.integers(0, 40))
            out.append(np.array([0x184D2A50 + int(rng.integers(0, 16)), k], "<u4").view(np.uint8))
            out.append(rng.integers(0, 256, k).astype(np.uint8))
        out.append(f)
    return np.concatenate(out) if out else np.zeros(0, np.uint8)
