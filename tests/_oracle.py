"""ctypes bindings to the TEST-ONLY oracle: oracle/liboracle.so (CPU restatement) and
oracle/_ref/libzstdmt_ref.so (the unmodified reference wrapper + liblz4/libzstd)."""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
c_sz = ctypes.c_size_t
c_vp = ctypes.c_void_p

CODEC_LZ4, CODEC_ZSTD = 1, 2
_orc = None
_ref = None


def orc():
    global _orc
    if _orc is None:
        L = ctypes.CDLL(os.path.join(ROOT, "oracle", "liboracle.so"))
        L.orc_xxh32.restype = ctypes.c_uint32; L.orc_xxh32.argtypes = [c_vp, c_sz, ctypes.c_uint32]
        L.orc_mt_decode.restype = ctypes.c_int; L.orc_mt_decode.argtypes = [ctypes.c_int, c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz)]
        L.orc_mt_encode_lz4_b200.restype = c_sz; L.orc_mt_encode_lz4_b200.argtypes = [c_vp, c_sz, c_sz, c_vp, c_sz]
        L.orc_lz4f_decode.restype = ctypes.c_int; L.orc_lz4f_decode.argtypes = [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz), ctypes.POINTER(c_sz)]
        L.orc_zstd_decode.restype = ctypes.c_int; L.orc_zstd_decode.argtypes = [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz), ctypes.POINTER(c_sz)]
        L.orc_lz4_block_compress_b200.restype = c_sz; L.orc_lz4_block_compress_b200.argtypes = [c_vp, c_sz, c_vp, c_sz]
        L.orc_lz4_block_bound.restype = c_sz; L.orc_lz4_block_bound.argtypes = [c_sz]
        L.orc_lz4_block_decode.restype = ctypes.c_long; L.orc_lz4_block_decode.argtypes = [c_vp, c_sz, c_vp, c_sz, c_sz]
        L.orc_mt_scan.restype = ctypes.c_long; L.orc_mt_scan.argtypes = [c_vp, c_sz, c_vp, c_vp, c_sz]
        _orc = L
    return _orc


def have_ref():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libzstdmt_ref.so"))


def ref():
    global _ref
    if _ref is None:
        L = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libzstdmt_ref.so"))
        for f in ("ref_lz4_compress_mem", "ref_zstd_compress_mem"):
            getattr(L, f).restype = c_sz
            getattr(L, f).argtypes = [ctypes.c_int] * 3 + [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz)]
        for f in ("ref_lz4_decompress_mem", "ref_zstd_decompress_mem"):
            getattr(L, f).restype = c_sz
            getattr(L, f).argtypes = [ctypes.c_int] * 2 + [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz)]
        _ref = L
    return _ref


def _arr(data):
    return np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data, dtype=np.uint8)


def ref_compress(codec, data, threads=1, level=1, chunk=1 << 20):
    """The real reference: {LZ4MT,ZSTDCB}_compressCCtx -> liblz4 / libzstd."""
    data = _arr(data)
    cap = data.size + data.size // 64 + 65536 + 64 * (data.size // chunk + 2)
    out = np.empty(cap, np.uint8); st = (c_sz * 5)()
    fn = ref().ref_lz4_compress_mem if codec == CODEC_LZ4 else ref().ref_zstd_compress_mem
    rc = fn(threads, level, chunk, data.ctypes.data, data.size, out.ctypes.data, cap, st)
    return rc, out[: st[0]].copy(), list(st)


def ref_decompress(codec, data, out_cap, threads=1):
    data = _arr(data)
    out = np.empty(out_cap + 1, np.uint8); st = (c_sz * 5)()
    fn = ref().ref_lz4_decompress_mem if codec == CODEC_LZ4 else ref().ref_zstd_decompress_mem
    rc = fn(threads, 0, data.ctypes.data, data.size, out.ctypes.data, out_cap + 1, st)
    return rc, out[: st[0]].copy(), list(st)


def orc_decode(codec, data, out_cap):
    data = _arr(data)
    out = np.empty(out_cap + 1, np.uint8); got = c_sz(0)
    rc = orc().orc_mt_decode(codec, data.ctypes.data, data.size, out.ctypes.data, out_cap + 1, ctypes.byref(got))
    return rc, out[: got.value]


def orc_encode_lz4(data, chunk=1 << 20):
    data = _arr(data)
    cap = data.size + data.size // 100 + 4096 + 64 * (data.size // chunk + 2)
    out = np.empty(cap, np.uint8)
    n = orc().orc_mt_encode_lz4_b200(data.ctypes.data, data.size, chunk, out.ctypes.data, cap)
    return out[:n].copy()


def xxh32(data, seed=0):
    data = _arr(data)
    return orc().orc_xxh32(data.ctypes.data, data.size, seed)


# ---- zstd block trace (orc_zstd_trace) ----
# columns of ZstdTrace.blk, in the order of the ORC_ZT_* enum of oracle/oracle.h
ZT_FIELDS = ("type", "last", "bsize", "regen", "lit_type", "lit_sf", "lit_hdr", "lit_regen", "lit_comp", "lit_streams",
             "s1", "s2", "s3", "s4", "tree_form", "tree_bytes", "nweights", "maxbits", "nseq", "nseq_bytes", "modes",
             "seq_first", "lit_first")
ZT = {name: i for i, name in enumerate(ZT_FIELDS)}


class _ZTrace(ctypes.Structure):
    _fields_ = [("max_blocks", c_sz), ("max_seqs", c_sz), ("max_lits", c_sz),
                ("blk", c_vp), ("weights", c_vp), ("seq", c_vp), ("lits", c_vp),
                ("nblocks", c_sz), ("nseqs", c_sz), ("nlits", c_sz)]


class ZstdTrace:
    """What every block of one zstd frame contained, as numpy arrays.
    blk[b, ZT[field]] (int32, -1 where the field does not apply); weights[b] (256 Huffman weights, the implied last one
    included); seq[i] = (literal length, Offset_Value as coded, match length, resolved offset); lits: the decoded literal
    sections of the compressed blocks back to back (block b's start at blk[b, ZT["lit_first"]]); content: the frame's
    decoded bytes."""

    def __init__(self, blk, weights, seq, lits, content, consumed):
        self.blk, self.weights, self.seq, self.lits, self.content, self.consumed = blk, weights, seq, lits, content, consumed

    def col(self, name):
        return self.blk[:, ZT[name]]

    def block_lits(self, b):
        a = int(self.blk[b, ZT["lit_first"]])
        return self.lits[a: a + int(self.blk[b, ZT["lit_regen"]])]

    def block_seqs(self, b):
        a = int(self.blk[b, ZT["seq_first"]])
        return self.seq[a: a + max(0, int(self.blk[b, ZT["nseq"]]))]


def zstd_trace(frame, out_cap=None):
    """orc_zstd_trace on one zstd frame (starting at the zstd magic).  Raises on a decode error."""
    frame = _arr(frame)
    L = orc()
    if not hasattr(L, "_zt_ready"):
        L.orc_zstd_trace.restype = ctypes.c_int
        L.orc_zstd_trace.argtypes = [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz), ctypes.POINTER(c_sz), ctypes.POINTER(_ZTrace)]
        L.orc_zstd_content_size.restype = ctypes.c_uint64; L.orc_zstd_content_size.argtypes = [c_vp, c_sz]
        L._zt_ready = True
    if out_cap is None:
        fcs = L.orc_zstd_content_size(frame.ctypes.data, frame.size)
        out_cap = int(fcs) if fcs != (1 << 64) - 1 else 128 << 20
    mb, ms, ml = frame.size // 3 + 2, out_cap // 3 + 2, out_cap + 1
    blk = np.empty((mb, len(ZT_FIELDS)), np.int32); w = np.empty((mb, 256), np.uint8)
    seq = np.empty((ms, 4), np.uint32); lits = np.empty(ml, np.uint8); out = np.empty(out_cap + 1, np.uint8)
    t = _ZTrace(mb, ms, ml, blk.ctypes.data, w.ctypes.data, seq.ctypes.data, lits.ctypes.data, 0, 0, 0)
    got, used = c_sz(0), c_sz(0)
    rc = L.orc_zstd_trace(frame.ctypes.data, frame.size, out.ctypes.data, out.size, ctypes.byref(got), ctypes.byref(used), ctypes.byref(t))
    if rc != 0:
        raise ValueError("orc_zstd_trace failed: %d" % rc)
    return ZstdTrace(blk[: t.nblocks].copy(), w[: t.nblocks].copy(), seq[: t.nseqs].copy(), lits[: t.nlits].copy(),
                     out[: got.value].copy(), used.value)


def mt_frames(framed):
    """The zstd / LZ4 frames of a framed stream (each after its 12-byte skippable header)."""
    framed = _arr(framed)
    cap = framed.size // 12 + 1
    offs = np.empty(cap, np.uint64); cs = np.empty(cap, np.uint32)
    n = orc().orc_mt_scan(framed.ctypes.data, framed.size, offs.ctypes.data, cs.ctypes.data, cap)
    if n < 0:
        raise ValueError("orc_mt_scan failed: %d" % n)
    return [framed[int(offs[i]) + 12: int(offs[i]) + 12 + int(cs[i])] for i in range(n)]


# ---- LZ4 frame trace (orc_lz4f_trace) ----
# columns of Lz4Trace.blk / .seq, in the order of the ORC_L4B_* / ORC_L4S_* enums of oracle/oracle.h
L4B_FIELDS = ("foff", "bsize", "stored", "regen", "linked", "bchk", "bchk_ok", "seq_first", "nseq", "dst")
L4S_FIELDS = ("tokpos", "llext", "mlext", "ll", "off", "ml", "dst")
L4B = {name: i for i, name in enumerate(L4B_FIELDS)}
L4S = {name: i for i, name in enumerate(L4S_FIELDS)}


class _L4Trace(ctypes.Structure):
    _fields_ = [("max_blocks", c_sz), ("max_seqs", c_sz), ("blk", c_vp), ("seq", c_vp), ("nblocks", c_sz), ("nseqs", c_sz)]


class Lz4Trace:
    """What every block of one LZ4 frame contained, as int64 numpy arrays: blk[b, L4B[field]] and seq[i, L4S[field]]
    (token position in the frame, extension byte counts, literal length, offset, match length, block-relative
    destination of the match; offset and match length 0 for a literals-only last sequence); content: the decoded bytes."""

    def __init__(self, blk, seq, content, consumed):
        self.blk, self.seq, self.content, self.consumed = blk, seq, content, consumed

    def col(self, name):
        return self.blk[:, L4B[name]]

    def s(self, name):
        return self.seq[:, L4S[name]]

    def block_seqs(self, b):
        a = int(self.blk[b, L4B["seq_first"]])
        return self.seq[a: a + int(self.blk[b, L4B["nseq"]])]


def lz4f_trace(frame, out_cap):
    """orc_lz4f_trace on one LZ4 frame (starting at its magic).  Raises on a decode error."""
    frame = _arr(frame)
    L = orc()
    if not hasattr(L, "_l4t_ready"):
        L.orc_lz4f_trace.restype = ctypes.c_int
        L.orc_lz4f_trace.argtypes = [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz), ctypes.POINTER(c_sz), ctypes.POINTER(_L4Trace)]
        L._l4t_ready = True
    mb, ms = frame.size // 4 + 2, frame.size + 2                      # a block costs >= 4 header bytes, a sequence >= 1 byte
    blk = np.empty((mb, len(L4B_FIELDS)), np.int64); seq = np.empty((ms, len(L4S_FIELDS)), np.int64)
    out = np.empty(out_cap + 1, np.uint8)
    t = _L4Trace(mb, ms, blk.ctypes.data, seq.ctypes.data, 0, 0)
    got, used = c_sz(0), c_sz(0)
    rc = L.orc_lz4f_trace(frame.ctypes.data, frame.size, out.ctypes.data, out.size, ctypes.byref(got), ctypes.byref(used), ctypes.byref(t))
    if rc != 0:
        raise ValueError("orc_lz4f_trace failed: %d" % rc)
    return Lz4Trace(blk[: t.nblocks].copy(), seq[: t.nseqs].copy(), out[: got.value].copy(), used.value)


def lz4f_decode(frame, out_cap):
    """orc_lz4f_decode on one LZ4 frame: (rc, decoded bytes, bytes consumed)."""
    frame = _arr(frame)
    out = np.empty(out_cap + 1, np.uint8); got, used = c_sz(0), c_sz(0)
    rc = orc().orc_lz4f_decode(frame.ctypes.data, frame.size, out.ctypes.data, out.size, ctypes.byref(got), ctypes.byref(used))
    return rc, out[: got.value].copy(), used.value
