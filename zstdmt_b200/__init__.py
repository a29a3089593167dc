"""zstdmt_b200 — GPU-native (H100) replacement for zstdmt's per-chunk LZ4 / Zstandard hot path.

The product is the C-ABI shared library ``libzstdmt_b200.so`` (CUDA kernels for sm_90a +
host pipeline exporting LZ4MT_* / ZSTDCB_* / ZSTDMT_*, see include/).  This module is only
the thin ctypes binding used by tests and bench.py; it never computes anything itself and it
raises if the native library is missing (no Python / CPU fallback).
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ZMT_LIB") or os.path.join(_HERE, "libzstdmt_b200.so")

c_sz = ctypes.c_size_t
c_u64 = ctypes.c_uint64
c_u32 = ctypes.c_uint32
c_vp = ctypes.c_void_p

CODEC_LZ4, CODEC_ZSTD = 1, 2
GEN_ZEROS, GEN_TEXT, GEN_MIX, GEN_RANDOM = 0, 1, 2, 3

ST_NAMES = {0: "ok", 1: "truncated", 2: "bad_magic", 3: "bad_header", 4: "hdr_checksum", 5: "block", 6: "dst_small",
            7: "content_checksum", 8: "content_size", 9: "trailing", 10: "unsupported", 11: "cuda", 12: "bad_arg"}

GEN_LIB_PATH = os.path.join(_HERE, "libzmt_datagen.so")
MEMIO_LIB_PATH = os.path.join(_HERE, "libzmt_memio.so")

_lib = None
_gen = None
_memio = None


class Buffer(ctypes.Structure):
    """LZ4MT_Buffer / ZSTDCB_Buffer (include/zstdmt_b200_lz4.h)."""
    _fields_ = [("buf", c_vp), ("size", c_sz), ("allocated", c_sz)]


RW_FN = ctypes.CFUNCTYPE(ctypes.c_int, c_vp, ctypes.POINTER(Buffer))


class RdWr(ctypes.Structure):
    """LZ4MT_RdWr_t / ZSTDCB_RdWr_t."""
    _fields_ = [("fn_read", RW_FN), ("arg_read", c_vp), ("fn_write", RW_FN), ("arg_write", c_vp)]


def lib():
    """Load libzstdmt_b200.so (building it with nvcc if the .so is absent)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        from . import build as _b
        _b.build_product()
    L = ctypes.CDLL(LIB_PATH)
    L.zmt_chunk_count.restype = c_u32; L.zmt_chunk_count.argtypes = [c_u64, c_u32]
    L.zmt_lz4c_workspace_bytes.restype = c_sz; L.zmt_lz4c_workspace_bytes.argtypes = [c_u32, c_u32]
    L.zmt_lz4c_out_bound.restype = c_u64; L.zmt_lz4c_out_bound.argtypes = [c_u32, c_u32]
    L.zmt_lz4_compress_device.restype = ctypes.c_int
    L.zmt_lz4_compress_device.argtypes = [c_vp, c_u64, c_u32, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstdc_workspace_bytes.restype = c_sz; L.zmt_zstdc_workspace_bytes.argtypes = [c_u32, c_u32]
    L.zmt_zstdc_out_bound.restype = c_u64; L.zmt_zstdc_out_bound.argtypes = [c_u32, c_u32]
    L.zmt_zstd_compress_device.restype = ctypes.c_int
    L.zmt_zstd_compress_device.argtypes = [c_vp, c_u64, c_u32, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstd_blk_desc_bytes.restype = c_sz; L.zmt_zstd_blk_desc_bytes.argtypes = []
    L.zmt_zstd_scan_frame_host.restype = ctypes.c_int
    L.zmt_zstd_scan_frame_host.argtypes = [c_vp, c_sz, c_u64, c_u32, c_vp, ctypes.POINTER(c_u32), c_u32, ctypes.POINTER(c_u64), ctypes.POINTER(c_u64), ctypes.POINTER(c_u32)]
    L.zmt_zstdd_workspace_bytes.restype = c_sz; L.zmt_zstdd_workspace_bytes.argtypes = [c_u32, c_u32, c_u64]
    L.zmt_zstd_decompress_device.restype = ctypes.c_int
    L.zmt_zstd_decompress_device.argtypes = [c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_lz4d_workspace_bytes.restype = c_sz; L.zmt_lz4d_workspace_bytes.argtypes = [c_u32, c_u32, c_u64]
    L.zmt_lz4_decompress_device.restype = ctypes.c_int
    L.zmt_lz4_decompress_device.argtypes = [c_vp, c_u64, c_vp, c_vp, c_u32, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    for pre, api in (("LZ4MT", "lz4"), ("ZSTDCB", "zstd"), ("ZSTDMT", "zstd")):
        getattr(L, pre + "_createCCtx").restype = c_vp; getattr(L, pre + "_createCCtx").argtypes = [ctypes.c_int] * 3
        getattr(L, pre + "_createDCtx").restype = c_vp; getattr(L, pre + "_createDCtx").argtypes = [ctypes.c_int] * 2
        for k in ("compressCCtx", "decompressDCtx"):
            f = getattr(L, pre + "_" + k); f.restype = c_sz; f.argtypes = [c_vp, ctypes.POINTER(RdWr)]
        for k in ("GetFramesCCtx", "GetInsizeCCtx", "GetOutsizeCCtx", "GetFramesDCtx", "GetInsizeDCtx", "GetOutsizeDCtx"):
            f = getattr(L, pre + "_" + k); f.restype = c_sz; f.argtypes = [c_vp]
        for k in ("freeCCtx", "freeDCtx"):
            f = getattr(L, pre + "_" + k); f.restype = None; f.argtypes = [c_vp]
        getattr(L, pre + "_isError").restype = ctypes.c_uint; getattr(L, pre + "_isError").argtypes = [c_sz]
        getattr(L, pre + "_getErrorString").restype = ctypes.c_char_p; getattr(L, pre + "_getErrorString").argtypes = [c_sz]
    _lib = L
    return L


def gen_lib():
    """libzmt_datagen.so: the synthetic input generator (harness, no dependency on the product library)."""
    global _gen
    if _gen is None:
        if not os.path.exists(GEN_LIB_PATH):
            from . import build as _b
            _b.build_harness()
        G = ctypes.CDLL(GEN_LIB_PATH)
        G.zmt_gen_stream.restype = None
        G.zmt_gen_stream.argtypes = [ctypes.c_int, c_u64, c_u64, c_sz, c_vp, c_sz, ctypes.c_int]
        G.zmt_gen_stream_dealt.restype = None
        G.zmt_gen_stream_dealt.argtypes = [ctypes.c_int, c_u64, c_u64, c_u64, c_sz, c_vp, c_sz, ctypes.c_int]
        _gen = G
    return _gen


def memio_lib():
    """libzmt_memio.so: in-memory fn_read / fn_write drivers of LZ4MT_* / ZSTDCB_* (harness; links the product library)."""
    global _memio
    if _memio is None:
        lib()
        if not os.path.exists(MEMIO_LIB_PATH):
            from . import build as _b
            _b.build_harness()
        M = ctypes.CDLL(MEMIO_LIB_PATH)
        for name in ("lz4_compress_mem", "zstd_compress_mem"):
            f = getattr(M, "zmt_" + name); f.restype = c_sz
            f.argtypes = [ctypes.c_int] * 3 + [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz)]
        for name in ("lz4_decompress_mem", "zstd_decompress_mem"):
            f = getattr(M, "zmt_" + name); f.restype = c_sz
            f.argtypes = [ctypes.c_int] * 2 + [c_vp, c_sz, c_vp, c_sz, ctypes.POINTER(c_sz)]
        _memio = M
    return _memio


# ------------------------------------------------------------------ synthetic inputs
def gen_stream(kind, nbytes, chunk, first=0, stride=1, threads=None, out=None, deal=None):
    """Deterministic synthetic stream (harness/datagen.c).  Returns a numpy uint8 array.
    deal=(rank, world, batch): the share of consumer `rank` when the global stream is dealt in batches of chunks."""
    if out is None:
        out = np.empty(nbytes, dtype=np.uint8)
    if threads is None:
        threads = min(32, os.cpu_count() or 1)
    if nbytes and deal is not None:
        gen_lib().zmt_gen_stream_dealt(kind, deal[0], deal[1], deal[2], chunk, out.ctypes.data, nbytes, threads)
    elif nbytes:
        gen_lib().zmt_gen_stream(kind, first, stride, chunk, out.ctypes.data, nbytes, threads)
    return out


# ------------------------------------------------------------------ memory-to-memory driver of the callback API
def _mem_call(fn, ints, data, cap):
    data = np.ascontiguousarray(data, dtype=np.uint8)
    out = np.empty(cap, dtype=np.uint8)
    st = (c_sz * 5)()
    rc = fn(*ints, data.ctypes.data, data.size, out.ctypes.data, cap, st)
    return rc, out[: st[0]], {"out_bytes": st[0], "frames": st[1], "insize": st[2], "outsize": st[3],
                              "reads": st[4] >> 32, "writes": st[4] & 0xFFFFFFFF}


def mt_bound(n, chunk):
    nch = max(1, -(-n // chunk))
    return n + n // 128 + nch * (64 + 4 * (chunk // 65536 + 1)) + 4096


def compress_mem(codec, data, threads=4, level=1, chunk=1 << 20):
    """{LZ4MT,ZSTDCB}_compressCCtx through in-memory callbacks (harness/memio_glue.c)."""
    L = memio_lib()
    fn = L.zmt_lz4_compress_mem if codec == CODEC_LZ4 else L.zmt_zstd_compress_mem
    return _mem_call(fn, (threads, level, chunk), data, mt_bound(len(data), chunk))


def decompress_mem(codec, data, out_cap, threads=4, inputsize=0):
    L = memio_lib()
    fn = L.zmt_lz4_decompress_mem if codec == CODEC_LZ4 else L.zmt_zstd_decompress_mem
    return _mem_call(fn, (threads, inputsize), data, out_cap)


# ------------------------------------------------------------------ device-resident batch API (torch only as allocator / stream owner)
def _torch():
    import torch
    return torch


def scan_frames(framed):
    """Walk a framed stream on the host: offsets of the 12-byte headers, payload sizes."""
    b = np.ascontiguousarray(framed, dtype=np.uint8)
    offs, sizes, pos, n = [], [], 0, b.size
    while pos < n:
        if n - pos < 12:
            raise ValueError("truncated skippable header")
        magic, four, cs = np.frombuffer(b[pos:pos + 12].tobytes(), dtype="<u4")
        if magic != 0x184D2A50 or four != 4:
            raise ValueError("bad skippable header at %d" % pos)
        offs.append(pos); sizes.append(int(cs)); pos += 12 + int(cs)
    if pos != n:
        raise ValueError("truncated payload")
    return np.array(offs, dtype=np.uint64), np.array(sizes, dtype=np.uint32)


class Lz4DeviceCompressor:
    """Pre-allocated device buffers + one call per batch: zmt_lz4_compress_device."""

    def __init__(self, in_bytes, chunk, device="cuda"):
        torch = _torch(); L = lib()
        self.chunk, self.in_bytes = chunk, in_bytes
        self.nchunks = L.zmt_chunk_count(in_bytes, chunk)
        self.work = torch.empty(L.zmt_lz4c_workspace_bytes(self.nchunks, chunk), dtype=torch.uint8, device=device)
        self.out = torch.empty(L.zmt_lz4c_out_bound(self.nchunks, chunk), dtype=torch.uint8, device=device)
        self.frame_off = torch.zeros(self.nchunks + 1, dtype=torch.int64, device=device)

    def run(self, d_in, stream=None):
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        rc = lib().zmt_lz4_compress_device(d_in.data_ptr(), self.in_bytes, self.chunk, None, self.nchunks,
                                           self.work.data_ptr(), self.out.data_ptr(), self.frame_off.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_lz4_compress_device failed: %s" % ST_NAMES.get(rc, rc))
        return self.out, self.frame_off


class ZstdDeviceCompressor:
    """zmt_zstd_compress_device: same layout contract as the LZ4 twin, Zstandard frames out."""

    def __init__(self, in_bytes, chunk, device="cuda"):
        torch = _torch(); L = lib()
        self.chunk, self.in_bytes = chunk, in_bytes
        self.nchunks = L.zmt_chunk_count(in_bytes, chunk)
        self.work = torch.empty(L.zmt_zstdc_workspace_bytes(self.nchunks, chunk), dtype=torch.uint8, device=device)
        self.out = torch.empty(L.zmt_zstdc_out_bound(self.nchunks, chunk), dtype=torch.uint8, device=device)
        self.frame_off = torch.zeros(self.nchunks + 1, dtype=torch.int64, device=device)

    def run(self, d_in, stream=None):
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        rc = lib().zmt_zstd_compress_device(d_in.data_ptr(), self.in_bytes, self.chunk, None, self.nchunks,
                                            self.work.data_ptr(), self.out.data_ptr(), self.frame_off.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_zstd_compress_device failed: %s" % ST_NAMES.get(rc, rc))
        return self.out, self.frame_off


class Lz4DeviceDecompressor:
    """zmt_lz4_decompress_device over a device-resident framed stream."""

    def __init__(self, frame_off, frame_csize, out_sizes, device="cuda"):
        torch = _torch(); L = lib()
        self.n = len(frame_off)
        self.d_off = torch.from_numpy(np.asarray(frame_off, dtype=np.int64)).to(device)
        self.d_cs = torch.from_numpy(np.asarray(frame_csize, dtype=np.int32)).to(device)
        oo = np.zeros(self.n + 1, dtype=np.int64); oo[1:] = np.cumsum(np.asarray(out_sizes, dtype=np.int64))
        self.out_total = int(oo[-1])
        osz = np.asarray(out_sizes, dtype=np.int64)
        self.nslots = int(np.maximum(1, (osz + 65535) // 65536).sum()) if len(osz) else 1
        self.d_out_off = torch.from_numpy(oo).to(device)
        self.out = torch.empty(max(self.out_total, 1), dtype=torch.uint8, device=device)
        self.out_size = torch.zeros(self.n, dtype=torch.int64, device=device)
        self.status = torch.zeros(self.n, dtype=torch.int32, device=device)
        self.in_bytes_cap = int((np.asarray(frame_off, dtype=np.int64) + 12 + np.asarray(frame_csize, dtype=np.int64)).max()) if self.n else 0
        self.work = torch.empty(L.zmt_lz4d_workspace_bytes(self.n, self.nslots, self.in_bytes_cap), dtype=torch.uint8, device=device)

    def run(self, d_framed, stream=None):
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        rc = lib().zmt_lz4_decompress_device(d_framed.data_ptr(), d_framed.numel(), self.d_off.data_ptr(), self.d_cs.data_ptr(), self.n,
                                             self.nslots, self.out.data_ptr(), self.d_out_off.data_ptr(), self.out_size.data_ptr(),
                                             self.status.data_ptr(), self.work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_lz4_decompress_device failed: %s" % ST_NAMES.get(rc, rc))
        return self.out, self.status


class ZstdDeviceDecompressor:
    """zmt_zstd_decompress_device.  The block table is built on the host from the framed bytes
    (zmt_zstd_scan_frame_host: frame + block headers only), as the host pipeline does while reading."""

    def __init__(self, framed_host, device="cuda"):
        torch = _torch(); L = lib()
        fb = np.ascontiguousarray(framed_host, dtype=np.uint8)
        offs, sizes = scan_frames(fb)
        self.n = len(offs)
        dsz = L.zmt_zstd_blk_desc_bytes()
        cap = int(fb.size // 3 + self.n + 16)              # every block costs at least its 3-byte header
        blocks = np.zeros(cap * dsz, dtype=np.uint8)
        nblk = c_u32(0); scr = c_u64(0)
        first = np.zeros(self.n + 1, dtype=np.uint32); expect = np.zeros(max(self.n, 1), dtype=np.uint64)
        fseq = np.zeros(max(self.n, 1), dtype=np.uint32)
        self.scan_status = []
        for i in range(self.n):
            first[i] = nblk.value
            cs = c_u64(0); nsq = c_u32(0)
            rc = L.zmt_zstd_scan_frame_host(fb[int(offs[i]) + 12:].ctypes.data, int(sizes[i]), int(offs[i]) + 12, i, blocks.ctypes.data,
                                            ctypes.byref(nblk), cap, ctypes.byref(scr), ctypes.byref(cs), ctypes.byref(nsq))
            self.scan_status.append(rc)
            expect[i] = cs.value; fseq[i] = nsq.value
        first[self.n] = nblk.value
        self.nblk = nblk.value
        self.scan_ok = all(rc == 0 for rc in self.scan_status)
        oo = np.zeros(self.n + 1, dtype=np.int64); oo[1:] = np.cumsum(expect[: self.n].astype(np.int64))
        self.out_total = int(oo[-1])
        self.d_blocks = torch.from_numpy(blocks[: max(1, self.nblk) * dsz].copy()).to(device)
        self.d_first = torch.from_numpy(first.astype(np.int32)).to(device)
        self.d_expect = torch.from_numpy(expect.astype(np.int64)).to(device)
        self.d_fseq = torch.from_numpy(fseq.astype(np.int32)).to(device)
        self.n_seq_frames = int(fseq.sum())
        self.d_out_off = torch.from_numpy(oo).to(device)
        self.out = torch.empty(max(self.out_total, 1), dtype=torch.uint8, device=device)
        self.out_size = torch.zeros(max(self.n, 1), dtype=torch.int64, device=device)
        self.status = torch.zeros(max(self.n, 1), dtype=torch.int32, device=device)
        self.work = torch.empty(L.zmt_zstdd_workspace_bytes(self.n, self.nblk, scr.value), dtype=torch.uint8, device=device)

    def run(self, d_framed, stream=None):
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        rc = lib().zmt_zstd_decompress_device(d_framed.data_ptr(), self.d_blocks.data_ptr(), self.nblk, self.d_first.data_ptr(), self.d_expect.data_ptr(),
                                              self.d_fseq.data_ptr(), self.n, self.out.data_ptr(), self.d_out_off.data_ptr(), self.out_size.data_ptr(), self.status.data_ptr(),
                                              self.work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_zstd_decompress_device failed: %s" % ST_NAMES.get(rc, rc))
        return self.out, self.status
