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
            7: "content_checksum", 8: "content_size", 9: "trailing", 10: "unsupported", 11: "cuda", 12: "bad_arg", 13: "dict_wrong"}

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
    L.zmt_lz4c_level_workspace_bytes.restype = c_sz; L.zmt_lz4c_level_workspace_bytes.argtypes = [c_u32, c_u32, ctypes.c_int]
    L.zmt_lz4_compress_level_device.restype = ctypes.c_int
    L.zmt_lz4_compress_level_device.argtypes = [c_vp, c_u64, c_u32, c_vp, c_u32, ctypes.c_int, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstdc_workspace_bytes.restype = c_sz; L.zmt_zstdc_workspace_bytes.argtypes = [c_u32, c_u32]
    L.zmt_zstdc_out_bound.restype = c_u64; L.zmt_zstdc_out_bound.argtypes = [c_u32, c_u32]
    L.zmt_zstd_compress_device.restype = ctypes.c_int
    L.zmt_zstd_compress_device.argtypes = [c_vp, c_u64, c_u32, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstdc_level_workspace_bytes.restype = c_sz; L.zmt_zstdc_level_workspace_bytes.argtypes = [c_u32, c_u32, ctypes.c_int]
    L.zmt_zstd_compress_level_device.restype = ctypes.c_int
    L.zmt_zstd_compress_level_device.argtypes = [c_vp, c_u64, c_u32, c_vp, c_u32, ctypes.c_int, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstd_blk_desc_bytes.restype = c_sz; L.zmt_zstd_blk_desc_bytes.argtypes = []
    L.zmt_zstd_scan_frame_host.restype = ctypes.c_int
    L.zmt_zstd_scan_frame_host.argtypes = [c_vp, c_sz, c_u64, c_u32, c_vp, ctypes.POINTER(c_u32), c_u32, ctypes.POINTER(c_u64), ctypes.POINTER(c_u64), ctypes.POINTER(c_u32)]
    L.zmt_zstdd_workspace_bytes.restype = c_sz; L.zmt_zstdd_workspace_bytes.argtypes = [c_u32, c_u32, c_u64]
    L.zmt_zstd_decompress_device.restype = ctypes.c_int
    L.zmt_zstd_decompress_device.argtypes = [c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_lz4d_workspace_bytes.restype = c_sz; L.zmt_lz4d_workspace_bytes.argtypes = [c_u32, c_u32, c_u64]
    L.zmt_lz4_decompress_device.restype = ctypes.c_int
    L.zmt_lz4_decompress_device.argtypes = [c_vp, c_u64, c_vp, c_vp, c_u32, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_lz4_decompress_segments_device.restype = ctypes.c_int
    L.zmt_lz4_decompress_segments_device.argtypes = [c_vp, c_u64, c_vp, c_vp, c_u32, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_lz4f_segment_host.restype = ctypes.c_int
    L.zmt_lz4f_segment_host.argtypes = [c_vp, c_sz, c_sz, c_u32, c_u32, c_sz, c_u64, ctypes.POINTER(c_sz), ctypes.POINTER(c_u64), ctypes.POINTER(c_u32)]
    L.zmt_zstd_decompress_segments_device.restype = ctypes.c_int
    L.zmt_zstd_decompress_segments_device.argtypes = [c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstd_segment_host.restype = ctypes.c_int
    L.zmt_zstd_segment_host.argtypes = [c_vp, c_sz, c_u64, c_u32, ctypes.POINTER(ZstdWalk), c_sz, c_u64, c_vp, ctypes.POINTER(c_u32), c_u32,
                                        ctypes.POINTER(c_u64), ctypes.POINTER(c_sz), ctypes.POINTER(c_u64), ctypes.POINTER(c_u32), ctypes.POINTER(c_u32)]
    L.zmt_zstd_segment_sources.restype = c_u32
    L.zmt_zstd_segment_sources.argtypes = [ctypes.POINTER(ZstdWalk), ctypes.POINTER(c_u64), ctypes.POINTER(c_u32)]
    L.zmt_index_workspace_bytes.restype = c_sz; L.zmt_index_workspace_bytes.argtypes = [c_u32]
    L.zmt_lz4_index_device.restype = ctypes.c_int
    L.zmt_lz4_index_device.argtypes = [c_vp, c_u64, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstd_index_device.restype = ctypes.c_int
    L.zmt_zstd_index_device.argtypes = [c_vp, c_u64, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_lz4_index_plain_device.restype = ctypes.c_int
    L.zmt_lz4_index_plain_device.argtypes = L.zmt_lz4_index_device.argtypes
    L.zmt_zstd_index_plain_device.restype = ctypes.c_int
    L.zmt_zstd_index_plain_device.argtypes = L.zmt_zstd_index_device.argtypes
    L.zmt_zstd_blocks_device.restype = ctypes.c_int
    L.zmt_zstd_blocks_device.argtypes = [c_vp, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_vp]
    L.zmt_zstd_ddict_bytes.restype = c_sz; L.zmt_zstd_ddict_bytes.argtypes = []
    L.zmt_zstd_ddict_load_device.restype = ctypes.c_int; L.zmt_zstd_ddict_load_device.argtypes = [c_vp, c_u64, c_vp, c_vp, c_vp]
    L.zmt_zstd_scan_frame_dict_host.restype = ctypes.c_int
    L.zmt_zstd_scan_frame_dict_host.argtypes = L.zmt_zstd_scan_frame_host.argtypes + [ctypes.POINTER(DictInfo)]
    for k in ("index", "index_plain", "blocks", "decompress"):
        f = getattr(L, "zmt_zstd_%s_dict_device" % k); f.restype = ctypes.c_int
        f.argtypes = getattr(L, "zmt_zstd_%s_device" % k).argtypes + [c_vp]
    L.zmt_zstd_cdict_bytes.restype = c_sz; L.zmt_zstd_cdict_bytes.argtypes = [c_u64]
    L.zmt_zstd_cdict_build_device.restype = ctypes.c_int; L.zmt_zstd_cdict_build_device.argtypes = [c_vp, c_u64, c_vp, c_vp]
    L.zmt_zstd_compress_dict_device.restype = ctypes.c_int
    L.zmt_zstd_compress_dict_device.argtypes = L.zmt_zstd_compress_level_device.argtypes + [c_vp]
    L.zmt_range_workspace_bytes.restype = c_sz; L.zmt_range_workspace_bytes.argtypes = [c_u32, c_u32]
    L.zmt_lz4_content_offsets_device.restype = ctypes.c_int
    L.zmt_lz4_content_offsets_device.argtypes = [c_vp, c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstd_content_offsets_device.restype = ctypes.c_int
    L.zmt_zstd_content_offsets_device.argtypes = [c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_lz4_range_plan_device.restype = ctypes.c_int
    L.zmt_lz4_range_plan_device.argtypes = [c_u32, c_vp, c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstd_range_plan_device.restype = ctypes.c_int
    L.zmt_zstd_range_plan_device.argtypes = [c_u32, c_vp, c_vp, c_vp, c_vp, c_vp, c_u32, c_vp, c_vp, c_vp, c_vp]
    for k in ("lz4", "zstd"):
        f = getattr(L, "zmt_%s_range_read_workspace_bytes" % k); f.restype = c_sz; f.argtypes = [ctypes.POINTER(RangePlan)]
    L.zmt_lz4_range_read_device.restype = ctypes.c_int
    L.zmt_lz4_range_read_device.argtypes = [c_vp, c_vp, c_vp, ctypes.POINTER(RangePlan), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.zmt_zstd_range_read_device.restype = ctypes.c_int
    L.zmt_zstd_range_read_device.argtypes = [c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.POINTER(RangePlan), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
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


class FrameIndex(ctypes.Structure):
    """zmt_frame_index (include/zstdmt_b200_dev.h): the summary of a device frame index."""
    _fields_ = [("status", c_u32), ("bad_frame", c_u32), ("bad_offset", c_u64), ("nframes", c_u32), ("nblocks", c_u32),
                ("out_bytes", c_u64), ("scratch_bytes", c_u64)]

    def __repr__(self):
        return "FrameIndex(%s)" % ", ".join("%s=%s" % (k, getattr(self, k)) for k, _ in self._fields_)


class DictInfo(ctypes.Structure):
    """zmt_zstd_dict_info (include/zstdmt_b200_dev.h): the summary of a dictionary loaded on the device."""
    _fields_ = [("status", c_u32), ("dict_id", c_u32), ("kind", c_u32), ("reserved", c_u32), ("content_bytes", c_u64), ("content_off", c_u64)]

    def __repr__(self):
        return "DictInfo(%s)" % ", ".join("%s=%s" % (k, getattr(self, k)) for k, _ in self._fields_)


class RangePlan(ctypes.Structure):
    """zmt_range_plan (include/zstdmt_b200_dev.h): the summary of a range-read plan, read back once per batch."""
    _fields_ = [("status", c_u32), ("bad_range", c_u32), ("nframes", c_u32), ("nranges", c_u32), ("nsel", c_u32), ("nunits", c_u32),
                ("packed_bytes", c_u64), ("scratch_bytes", c_u64), ("dec_scratch", c_u64), ("dst_bytes", c_u64), ("npieces", c_u64)]

    def __repr__(self):
        return "RangePlan(%s)" % ", ".join("%s=%s" % (k, getattr(self, k)) for k, _ in self._fields_)


# The plain index writes its tables for a base this many bytes below the stream: the decode calls address a frame as
# one behind a 12-byte container header (include/zstdmt_b200_dev.h, "Layout convention").
PLAIN_PAD = 12


def _device_index(d_framed, max_frames, stream, zstd, plain=False, dictionary=None):
    """Run zmt_{lz4,zstd}_index_device (plain: zmt_{lz4,zstd}_index_plain_device; with a ZstdDictionary: the zstd
    *_dict_device calls) over a stream in device memory.  Only the summary struct is read back; on ZMT_ST_DST_SMALL the
    index runs once more with the exact frame count.  Returns (summary, device tables by name)."""
    torch = _torch(); L = lib()
    s = stream if stream is not None else torch.cuda.current_stream()
    dev, nbytes = d_framed.device, d_framed.numel()
    cap = int(max_frames) if max_frames is not None else min(nbytes // (9 if plain else 12), 1 << 16)
    for attempt in range(2):
        e = lambda n, dt: torch.empty(max(n, 1), dtype=dt, device=dev)
        t = {"frame_off": e(cap, torch.int64), "frame_csize": e(cap, torch.int32), "out_off": e(cap + 1, torch.int64)}
        if zstd:
            t.update(first_blk=e(cap + 1, torch.int32), frame_scratch=e(cap + 1, torch.int64), expect=e(cap, torch.int64),
                     frame_seq=e(cap, torch.int32))
        wb = L.zmt_index_workspace_bytes(cap)
        if wb == 0:
            raise ValueError("no index workspace size for %d frames" % cap)
        work = torch.empty(wb, dtype=torch.uint8, device=dev)
        d_info = torch.zeros(ctypes.sizeof(FrameIndex), dtype=torch.uint8, device=dev)
        p = lambda k: t[k].data_ptr()
        if zstd:
            args = (d_framed.data_ptr(), nbytes, cap, p("frame_off"), p("frame_csize"), p("first_blk"), p("frame_scratch"),
                    p("expect"), p("frame_seq"), p("out_off"), d_info.data_ptr(), work.data_ptr(), s.cuda_stream)
            if dictionary is not None:
                fn = L.zmt_zstd_index_plain_dict_device if plain else L.zmt_zstd_index_dict_device
                rc = fn(*args, dictionary.d_ddict.data_ptr())
            else:
                fn = L.zmt_zstd_index_plain_device if plain else L.zmt_zstd_index_device
                rc = fn(*args)
        else:
            fn = L.zmt_lz4_index_plain_device if plain else L.zmt_lz4_index_device
            rc = fn(d_framed.data_ptr(), nbytes, cap, p("frame_off"), p("frame_csize"), p("out_off"), d_info.data_ptr(),
                    work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("frame index failed: %s" % ST_NAMES.get(rc, rc))
        s.synchronize()
        info = FrameIndex.from_buffer_copy(d_info.cpu().numpy().tobytes())
        if info.status == 6 and attempt == 0:                               # ZMT_ST_DST_SMALL: info.nframes is the true count
            cap = info.nframes
            continue
        break
    if info.status != 0:
        raise ValueError("%s stream rejected: %s in frame %d at offset %d" % ("plain" if plain else "framed", ST_NAMES.get(info.status, info.status),
                                                                            info.bad_frame, info.bad_offset))
    return info, t


class Lz4DeviceCompressor:
    """Pre-allocated device buffers + one call per batch: zmt_lz4_compress_level_device.  Levels 1-9 run the level-1
    encoder (zmt_lz4_compress_device, independent blocks), levels 10-12 the high-compression class with linked blocks."""

    def __init__(self, in_bytes, chunk, device="cuda", level=1):
        torch = _torch(); L = lib()
        self.chunk, self.in_bytes, self.level = chunk, in_bytes, level
        self.nchunks = L.zmt_chunk_count(in_bytes, chunk)
        wb = L.zmt_lz4c_level_workspace_bytes(self.nchunks, chunk, level)
        if wb == 0:
            raise ValueError("no workspace size for %d chunks of %d bytes at level %d" % (self.nchunks, chunk, level))
        self.work = torch.empty(wb, dtype=torch.uint8, device=device)
        self.out = torch.empty(L.zmt_lz4c_out_bound(self.nchunks, chunk), dtype=torch.uint8, device=device)
        self.frame_off = torch.zeros(self.nchunks + 1, dtype=torch.int64, device=device)

    def run(self, d_in, stream=None):
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        rc = lib().zmt_lz4_compress_level_device(d_in.data_ptr(), self.in_bytes, self.chunk, None, self.nchunks, self.level,
                                                 self.work.data_ptr(), self.out.data_ptr(), self.frame_off.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_lz4_compress_level_device failed: %s" % ST_NAMES.get(rc, rc))
        return self.out, self.frame_off


class ZstdDeviceCompressor:
    """zmt_zstd_compress_level_device: same layout contract as the LZ4 twin, Zstandard frames out.  Levels 1-5 run the
    level-3 encoder (zmt_zstd_compress_device), levels 6-22 the hash-chain class with a lazy parse.  With a
    ZstdDictionary (levels 6-22) the chains continue into its content and the frames name its ID
    (zmt_zstd_compress_dict_device); the dictionary must outlive the compressor, which keeps a reference to it."""

    def __init__(self, in_bytes, chunk, device="cuda", level=3, dictionary=None):
        torch = _torch(); L = lib()
        if dictionary is not None and level < 6:
            raise ValueError("compressing with a dictionary needs level 6 or above (level %d)" % level)
        self.chunk, self.in_bytes, self.level, self.dictionary = chunk, in_bytes, level, dictionary
        self.nchunks = L.zmt_chunk_count(in_bytes, chunk)
        wb = L.zmt_zstdc_level_workspace_bytes(self.nchunks, chunk, level)
        if wb == 0:
            raise ValueError("no workspace size for %d chunks of %d bytes at level %d" % (self.nchunks, chunk, level))
        self.work = torch.empty(wb, dtype=torch.uint8, device=device)
        self.out = torch.empty(L.zmt_zstdc_out_bound(self.nchunks, chunk), dtype=torch.uint8, device=device)
        self.frame_off = torch.zeros(self.nchunks + 1, dtype=torch.int64, device=device)

    def run(self, d_in, stream=None, chunk_bytes=None):
        """chunk_bytes: a device uint32 tensor of the chunks' lengths (one per chunk; chunk c starts at c * chunk), for a
        batch of records in fixed slots."""
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        cb = None
        if chunk_bytes is not None:
            if (chunk_bytes.dtype not in (torch.int32, torch.uint32) or not chunk_bytes.is_cuda or not chunk_bytes.is_contiguous()
                    or chunk_bytes.numel() != self.nchunks):
                raise ValueError("chunk_bytes: a contiguous device tensor of %d 32-bit lengths" % self.nchunks)
            cb = chunk_bytes.data_ptr()
        args = (d_in.data_ptr(), self.in_bytes, self.chunk, cb, self.nchunks, self.level, self.work.data_ptr(), self.out.data_ptr(),
                self.frame_off.data_ptr(), s.cuda_stream)
        if self.dictionary is not None:
            name = "zmt_zstd_compress_dict_device"
            rc = lib().zmt_zstd_compress_dict_device(*args, self.dictionary.cdict(s).data_ptr())
        else:
            name = "zmt_zstd_compress_level_device"
            rc = lib().zmt_zstd_compress_level_device(*args)
        if rc != 0:
            raise RuntimeError("%s failed: %s" % (name, ST_NAMES.get(rc, rc)))
        return self.out, self.frame_off


class Lz4DeviceDecompressor:
    """zmt_lz4_decompress_device over a device-resident framed stream (from_device: also a plain .lz4 stream)."""
    pad = 0                 # bytes from the decoder's base to the stream (PLAIN_PAD for a plain stream)

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

    @classmethod
    def from_device(cls, d_framed, max_frames=None, stream=None, plain=False):
        """A decoder for a framed stream that is already in device memory: the frame tables are built on the GPU
        (zmt_lz4_index_device) and only the summary comes back to the host, as .index_info.  run(d_framed) decodes.
        max_frames sizes the first attempt (default: up to 65536 frames); a larger stream is indexed once more at its
        exact count.  Raises ValueError naming the status, frame and offset of a stream the index rejects.
        plain=True: d_framed is a plain .lz4 stream (LZ4F and skippable frames back to back, zmt_lz4_index_plain_device);
        frame offsets are then the frames' own, and run() passes the decoder the base the tables are written for."""
        torch = _torch(); L = lib()
        info, t = _device_index(d_framed, max_frames, stream, zstd=False, plain=plain)
        self = cls.__new__(cls)
        self.pad = PLAIN_PAD if plain else 0
        self.index_info, self.n, self.nslots, self.out_total = info, info.nframes, max(info.nblocks, 1), info.out_bytes
        self.d_off, self.d_cs, self.d_out_off = t["frame_off"], t["frame_csize"], t["out_off"]
        self.out = torch.empty(max(self.out_total, 1), dtype=torch.uint8, device=d_framed.device)
        self.out_size = torch.zeros(max(self.n, 1), dtype=torch.int64, device=d_framed.device)
        self.status = torch.zeros(max(self.n, 1), dtype=torch.int32, device=d_framed.device)
        self.in_bytes_cap = d_framed.numel() + self.pad
        self.work = torch.empty(L.zmt_lz4d_workspace_bytes(self.n, self.nslots, self.in_bytes_cap), dtype=torch.uint8, device=d_framed.device)
        return self

    def run(self, d_framed, stream=None):
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        rc = lib().zmt_lz4_decompress_device(d_framed.data_ptr() - self.pad, d_framed.numel() + self.pad, self.d_off.data_ptr(), self.d_cs.data_ptr(), self.n,
                                             self.nslots, self.out.data_ptr(), self.d_out_off.data_ptr(), self.out_size.data_ptr(),
                                             self.status.data_ptr(), self.work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_lz4_decompress_device failed: %s" % ST_NAMES.get(rc, rc))
        return self.out, self.status


SEG_FIRST, SEG_LAST = 1, 2


class Lz4Segment(ctypes.Structure):
    """zmt_lz4_segment (include/zstdmt_b200_dev.h): the state of an LZ4F frame decoded as a chain of segments."""
    _fields_ = [("history", c_u64), ("produced", c_u64), ("content_size", c_u64), ("flags", c_u32), ("flg", ctypes.c_uint8),
                ("bd", ctypes.c_uint8), ("pending_len", ctypes.c_uint16), ("acc", c_u32 * 4), ("pending", ctypes.c_uint8 * 16)]


def lz4f_segment(seg_bytes, start, flg, bd, max_in, max_out):
    """zmt_lz4f_segment_host: (status, end, room, last) of the segment whose bytes begin seg_bytes (first block header at start)."""
    b = np.ascontiguousarray(seg_bytes, dtype=np.uint8)
    end, room, last = c_sz(0), c_u64(0), c_u32(0)
    rc = lib().zmt_lz4f_segment_host(b.ctypes.data, b.size, start, flg, bd, max_in, max_out, ctypes.byref(end), ctypes.byref(room), ctypes.byref(last))
    return rc, end.value, room.value, last.value


def lz4_decode_segments(frame, cuts, device="cuda"):
    """Decodes one LZ4F frame (host bytes) through zmt_lz4_decompress_segments_device as the chain of segments that ends
    at the frame offsets `cuts` (block boundaries, increasing; the frame's length is appended).  Each segment's output
    goes 64 KiB above the start of a fresh buffer, with the frame's last 64 KiB of content copied below it first.
    Returns (content, status): the decoded bytes (numpy) and the ZMT_ST_* of the first failing segment, or 0."""
    torch = _torch(); L = lib()
    fb = np.ascontiguousarray(frame, dtype=np.uint8)
    flg, bd = int(fb[4]), int(fb[5])
    H = 65536
    seg = torch.zeros(ctypes.sizeof(Lz4Segment), dtype=torch.uint8, device=device)
    ends = [int(c) for c in cuts] + [fb.size]
    parts, prev, hist = [], 0, torch.zeros(0, dtype=torch.uint8, device=device)
    for k, end in enumerate(ends):
        first, last = k == 0, k == len(ends) - 1
        rc, e2, room, is_last = lz4f_segment(fb[prev:], (7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)) if first else 0, flg, bd,
                                             end - prev, 1 << 62)
        if rc != 0 or e2 != end - prev or bool(is_last) != last:
            raise ValueError("cut %d is not a block boundary (walk: rc %d end %d last %d)" % (end, rc, prev + e2, is_last))
        d_in = torch.zeros(12 + (end - prev) + 256, dtype=torch.uint8, device=device)
        d_in[12:12 + end - prev] = torch.from_numpy(fb[prev:end].copy()).to(device)
        out = torch.zeros(H + room + 256, dtype=torch.uint8, device=device)
        if hist.numel():
            out[H - hist.numel():H] = hist
        foff = torch.zeros(1, dtype=torch.int64, device=device)
        fcs = torch.tensor([end - prev], dtype=torch.int32, device=device)
        ooff = torch.tensor([H, H + room], dtype=torch.int64, device=device)
        osz = torch.zeros(1, dtype=torch.int64, device=device)
        st = torch.zeros(1, dtype=torch.int32, device=device)
        nslots = max(1, (room + 65535) // 65536)
        work = torch.empty(L.zmt_lz4d_workspace_bytes(1, nslots, 12 + end - prev), dtype=torch.uint8, device=device)
        rec = Lz4Segment.from_buffer_copy(bytes(seg.cpu().numpy()))
        rec.history, rec.flags = hist.numel(), (SEG_FIRST if first else 0) | (SEG_LAST if last else 0)
        seg.copy_(torch.frombuffer(bytearray(bytes(rec)), dtype=torch.uint8))
        s = torch.cuda.current_stream()
        rc = L.zmt_lz4_decompress_segments_device(d_in.data_ptr(), d_in.numel(), foff.data_ptr(), fcs.data_ptr(), 1, nslots, out.data_ptr(),
                                                  ooff.data_ptr(), osz.data_ptr(), st.data_ptr(), seg.data_ptr(), work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_lz4_decompress_segments_device failed: %s" % ST_NAMES.get(rc, rc))
        torch.cuda.synchronize()
        if int(st.item()) != 0:
            return np.concatenate(parts) if parts else np.zeros(0, np.uint8), int(st.item())
        n = int(osz.item())
        parts.append(out[H:H + n].cpu().numpy())
        hist = torch.cat([hist, out[H:H + n]])[-H:].clone()
        prev = end
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8), 0


class ZstdWalk(ctypes.Structure):
    """zmt_zstd_walk (include/zstdmt_b200_dev.h): where the segment walk of a zstd frame stands, and the frame's table sources."""
    _fields_ = [("pos", c_u64), ("content_size", c_u64), ("window", c_u64), ("flags", c_u32), ("nblk", c_u32), ("done", c_u32),
                ("reserved", c_u32), ("src_off", c_u64 * 4), ("src_len", c_u32 * 4)]


class ZstdSegment(ctypes.Structure):
    """zmt_zstd_segment (include/zstdmt_b200_dev.h): the device state of a zstd frame decoded as a chain of segments."""
    _fields_ = [("history", c_u64), ("produced", c_u64), ("content_size", c_u64), ("flags", c_u32), ("rep", c_u32 * 3),
                ("acc", c_u64 * 4), ("pending_len", c_u32), ("reserved", c_u32), ("pending", ctypes.c_uint8 * 32)]


def zstd_segment_sources(walk):
    """zmt_zstd_segment_sources: [(frame offset, length)] of the table sources a segment starting at `walk` carries."""
    off, ln = (c_u64 * 4)(), (c_u32 * 4)()
    k = lib().zmt_zstd_segment_sources(ctypes.byref(walk), off, ln)
    return [(int(off[i]), int(ln[i])) for i in range(k)]


def zstd_segment(seg_bytes, walk, max_in, max_out, base_off=0, frame_idx=0):
    """zmt_zstd_segment_host on the frame's bytes from walk.pos on: (status, end, room, flags, last, descriptors).  `walk`
    (a ZstdWalk) advances on success.  descriptors: the segment's block descriptors as bytes (zmt_zstd_blk_desc_bytes()
    each), the carried table sources first; seg_bytes[0] lies at base_off in the decoder input, the carry area below."""
    L = lib()
    b = np.ascontiguousarray(seg_bytes, dtype=np.uint8)
    dsz = L.zmt_zstd_blk_desc_bytes()
    cap = int(min(b.size, max_in + (1 << 17)) // 3 + 16)
    while True:
        out = np.zeros(cap * dsz, np.uint8)
        nb, scr, end, room, flags, last = c_u32(0), c_u64(0), c_sz(0), c_u64(0), c_u32(0), c_u32(0)
        rc = L.zmt_zstd_segment_host(b.ctypes.data, b.size, base_off, frame_idx, ctypes.byref(walk), max_in, max_out, out.ctypes.data,
                                     ctypes.byref(nb), cap, ctypes.byref(scr), ctypes.byref(end), ctypes.byref(room), ctypes.byref(flags),
                                     ctypes.byref(last))
        if rc != 6:                                          # ZMT_ST_DST_SMALL: a larger table
            return rc, end.value, room.value, flags.value, last.value, out[: nb.value * dsz], scr.value
        cap *= 2


def zstd_decode_segments(frame, cuts, device="cuda"):
    """Decodes one zstd frame (host bytes) through zmt_zstd_decompress_segments_device as the chain of segments that ends
    at the frame offsets `cuts` (block boundaries, increasing; the frame's length is appended).  Each segment's input is
    its carried table sources followed by its bytes; its output goes above the frame's last min(Window_Size, produced)
    content bytes, copied below it first.  Returns (content, status): the decoded bytes (numpy) and the ZMT_ST_* of the
    first failing segment, or 0."""
    torch = _torch(); L = lib()
    fb = np.ascontiguousarray(frame, dtype=np.uint8)
    seg = torch.zeros(ctypes.sizeof(ZstdSegment), dtype=torch.uint8, device=device)
    w = ZstdWalk()
    ends = [int(c) for c in cuts] + [fb.size]
    parts, prev, hist = [], 0, torch.zeros(0, dtype=torch.uint8, device=device)
    for k, end in enumerate(ends):
        first, last = k == 0, k == len(ends) - 1
        carry = b"".join(fb[o:o + n].tobytes() for o, n in zstd_segment_sources(w))
        rc, e2, room, flags, is_last, blk, scr = zstd_segment(fb[prev:], w, end - prev, 1 << 62, base_off=len(carry))
        if rc != 0 or e2 != end - prev or bool(is_last) != last:
            raise ValueError("cut %d is not a block boundary (walk: rc %d end %d last %d)" % (end, rc, prev + e2, is_last))
        nblk = blk.size // L.zmt_zstd_blk_desc_bytes()
        d_in = torch.zeros(len(carry) + (end - prev) + 256, dtype=torch.uint8, device=device)
        d_in[:len(carry) + end - prev] = torch.from_numpy(np.frombuffer(carry + fb[prev:end].tobytes(), np.uint8).copy()).to(device)
        H = hist.numel()
        out = torch.zeros(H + room + 256, dtype=torch.uint8, device=device)
        if H:
            out[:H] = hist
        d_blk = torch.from_numpy(blk.copy()).to(device)
        first_blk = torch.tensor([0, nblk], dtype=torch.int32, device=device)
        expect = torch.tensor([-1 if flags & 4 else w.content_size], dtype=torch.int64, device=device) if first else torch.full((1,), -1, dtype=torch.int64, device=device)
        fseq = torch.tensor([flags], dtype=torch.int32, device=device)
        ooff = torch.tensor([H, H + room], dtype=torch.int64, device=device)
        osz = torch.zeros(1, dtype=torch.int64, device=device)
        st = torch.zeros(1, dtype=torch.int32, device=device)
        work = torch.empty(L.zmt_zstdd_workspace_bytes(1, nblk, scr), dtype=torch.uint8, device=device)
        rec = ZstdSegment.from_buffer_copy(bytes(seg.cpu().numpy()))
        rec.history, rec.flags = H, (SEG_FIRST if first else 0) | (SEG_LAST if last else 0)
        seg.copy_(torch.frombuffer(bytearray(bytes(rec)), dtype=torch.uint8))
        s = torch.cuda.current_stream()
        rc = L.zmt_zstd_decompress_segments_device(d_in.data_ptr(), d_blk.data_ptr(), nblk, first_blk.data_ptr(), expect.data_ptr(), fseq.data_ptr(), 1,
                                                   out.data_ptr(), ooff.data_ptr(), osz.data_ptr(), st.data_ptr(), seg.data_ptr(), work.data_ptr(),
                                                   s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_zstd_decompress_segments_device failed: %s" % ST_NAMES.get(rc, rc))
        torch.cuda.synchronize()
        if int(st.item()) != 0:
            return np.concatenate(parts) if parts else np.zeros(0, np.uint8), int(st.item())
        n = int(osz.item())
        parts.append(out[H:H + n].cpu().numpy())
        hist = torch.cat([hist, out[H:H + n]])[-w.window:].clone() if w.window else hist[:0]
        prev = end
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8), 0


class ZstdDictionary:
    """A zstd dictionary loaded on the device (zmt_zstd_ddict_load_device): `data` (bytes or a uint8 array, formatted or
    raw content) is copied to the device and stays there with the record for as long as this object lives.  .info is
    the load's summary (DictInfo); a dictionary the load rejects raises ValueError with the status name.  The
    compression index (16 MiB and more, zmt_zstd_cdict_build_device) is built on first use by a compressor."""

    _cdict = None

    def __init__(self, data, device="cuda", stream=None):
        torch = _torch(); L = lib()
        b = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8)
        s = stream if stream is not None else torch.cuda.current_stream()
        self.nbytes = int(b.size)
        self.d_dict = torch.from_numpy(np.concatenate([b, np.zeros(1, np.uint8)])).to(device)
        self.d_ddict = torch.zeros(L.zmt_zstd_ddict_bytes(), dtype=torch.uint8, device=device)
        d_info = torch.zeros(ctypes.sizeof(DictInfo), dtype=torch.uint8, device=device)
        rc = L.zmt_zstd_ddict_load_device(self.d_dict.data_ptr(), self.nbytes, self.d_ddict.data_ptr(), d_info.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("zmt_zstd_ddict_load_device failed: %s" % ST_NAMES.get(rc, rc))
        s.synchronize()
        self.info = DictInfo.from_buffer_copy(d_info.cpu().numpy().tobytes())
        if self.info.status != 0:
            raise ValueError("dictionary rejected: %s" % ST_NAMES.get(self.info.status, self.info.status))

    def cdict(self, stream=None):
        """The compression index (device uint8 tensor), built on `stream` the first time it is asked for."""
        if self._cdict is None:
            torch = _torch(); L = lib()
            s = stream if stream is not None else torch.cuda.current_stream()
            nb = L.zmt_zstd_cdict_bytes(self.nbytes)
            if nb == 0:
                raise ValueError("no compression index for a dictionary of %d bytes" % self.nbytes)
            cd = torch.empty(nb, dtype=torch.uint8, device=self.d_ddict.device)
            rc = L.zmt_zstd_cdict_build_device(self.d_ddict.data_ptr(), self.nbytes, cd.data_ptr(), s.cuda_stream)
            if rc != 0:
                raise RuntimeError("zmt_zstd_cdict_build_device failed: %s" % ST_NAMES.get(rc, rc))
            self._cdict = cd
        return self._cdict


class ZstdDeviceDecompressor:
    """zmt_zstd_decompress_device.  The constructor builds the block table on the host from the framed bytes
    (zmt_zstd_scan_frame_host: frame + block headers only), as the host pipeline does while reading; from_device builds
    it on the GPU from a stream already in device memory.  With a ZstdDictionary every frame decodes against it (the
    *_dict calls); the dictionary must outlive the decompressor, which keeps a reference to it."""

    pad = 0                 # as Lz4DeviceDecompressor.pad
    dictionary = None

    def __init__(self, framed_host, device="cuda", dictionary=None):
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
            args = (fb[int(offs[i]) + 12:].ctypes.data, int(sizes[i]), int(offs[i]) + 12, i, blocks.ctypes.data,
                    ctypes.byref(nblk), cap, ctypes.byref(scr), ctypes.byref(cs), ctypes.byref(nsq))
            if dictionary is not None:
                rc = L.zmt_zstd_scan_frame_dict_host(*args, ctypes.byref(dictionary.info))
            else:
                rc = L.zmt_zstd_scan_frame_host(*args)
            self.scan_status.append(rc)
            expect[i] = cs.value; fseq[i] = nsq.value
        first[self.n] = nblk.value
        self.nblk = nblk.value
        self.scan_ok = all(rc == 0 for rc in self.scan_status)
        oo = np.zeros(self.n + 1, dtype=np.int64); oo[1:] = np.cumsum(expect[: self.n].astype(np.int64))
        self.out_total = int(oo[-1])
        expect[: self.n][(fseq[: self.n] & 4) != 0] = ~np.uint64(0)     # ZF_NO_SIZE: the room is a bound, not a size to check
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
        self.dictionary = dictionary

    @classmethod
    def from_device(cls, d_framed, max_frames=None, stream=None, plain=False, dictionary=None):
        """A decoder for a framed stream that is already in device memory: the frame tables and the block table are built
        on the GPU (zmt_zstd_index_device, zmt_zstd_blocks_device) and only the summary comes back to the host, as
        .index_info.  run(d_framed) decodes.  max_frames, plain and the errors as Lz4DeviceDecompressor.from_device
        (plain: a .zst stream, zmt_zstd_index_plain_device)."""
        torch = _torch(); L = lib()
        s = stream if stream is not None else torch.cuda.current_stream()
        info, t = _device_index(d_framed, max_frames, s, zstd=True, plain=plain, dictionary=dictionary)
        dev = d_framed.device
        self = cls.__new__(cls)
        self.pad = PLAIN_PAD if plain else 0
        self.dictionary = dictionary
        self.index_info, self.n, self.nblk, self.out_total = info, info.nframes, info.nblocks, info.out_bytes
        self.d_first, self.d_expect, self.d_fseq, self.d_out_off = t["first_blk"], t["expect"], t["frame_seq"], t["out_off"]
        self.d_blocks = torch.empty(max(1, self.nblk) * L.zmt_zstd_blk_desc_bytes(), dtype=torch.uint8, device=dev)
        rc = L.zmt_zstd_blocks_dict_device(d_framed.data_ptr() - self.pad, self.n, t["frame_off"].data_ptr(), t["frame_csize"].data_ptr(),
                                           self.d_first.data_ptr(), t["frame_scratch"].data_ptr(), self.d_blocks.data_ptr(), self.nblk, s.cuda_stream,
                                           dictionary.d_ddict.data_ptr() if dictionary is not None else None)
        if rc != 0:
            raise RuntimeError("zmt_zstd_blocks_device failed: %s" % ST_NAMES.get(rc, rc))
        self.d_frame_off, self.d_frame_csize, self.d_frame_scratch = t["frame_off"], t["frame_csize"], t["frame_scratch"]
        self.out = torch.empty(max(self.out_total, 1), dtype=torch.uint8, device=dev)
        self.out_size = torch.zeros(max(self.n, 1), dtype=torch.int64, device=dev)
        self.status = torch.zeros(max(self.n, 1), dtype=torch.int32, device=dev)
        self.work = torch.empty(L.zmt_zstdd_workspace_bytes(self.n, self.nblk, info.scratch_bytes), dtype=torch.uint8, device=dev)
        return self

    def run(self, d_framed, stream=None):
        torch = _torch()
        s = stream if stream is not None else torch.cuda.current_stream()
        args = (d_framed.data_ptr() - self.pad, self.d_blocks.data_ptr(), self.nblk, self.d_first.data_ptr(), self.d_expect.data_ptr(),
                self.d_fseq.data_ptr(), self.n, self.out.data_ptr(), self.d_out_off.data_ptr(), self.out_size.data_ptr(), self.status.data_ptr(),
                self.work.data_ptr(), s.cuda_stream)
        if self.dictionary is not None:
            rc = lib().zmt_zstd_decompress_dict_device(*args, self.dictionary.d_ddict.data_ptr())
        else:
            rc = lib().zmt_zstd_decompress_device(*args)
        if rc != 0:
            raise RuntimeError("zmt_zstd_decompress_device failed: %s" % ST_NAMES.get(rc, rc))
        return self.out, self.status


class RangeReader:
    """Byte ranges of a compressed stream that is already in device memory, decoding only the frames that hold them.

    The constructor indexes the stream once on the GPU (as from_device does; plain=True for a plain .lz4 / .zst stream)
    and builds its content table: the content offset of every frame, from the sizes the frames' headers state.  A stream
    with a frame that states no content size cannot be range-read: ValueError names the status and the frame.
    read(ranges) takes an int64 (M, 2) tensor of (start, length) pairs in content coordinates, on the CPU or the GPU, and
    returns CUDA tensors (bytes, dst_off, status): range r's bytes are bytes[dst_off[r]:dst_off[r + 1]], status[r] is its
    ZMT_ST_* code.  Every frame a range touches is decoded once per batch, the others are not read.  Buffers are kept
    across batches and grown when a batch needs more; .plan is the last batch's RangePlan summary."""

    def __init__(self, d_stream, codec, plain=False, max_frames=None, stream=None):
        torch = _torch(); L = lib()
        if codec in ("lz4", CODEC_LZ4):
            self.zstd = False
        elif codec in ("zstd", CODEC_ZSTD):
            self.zstd = True
        else:
            raise ValueError("unknown codec %r" % (codec,))
        s = stream if stream is not None else torch.cuda.current_stream()
        self.d_stream, self.dev = d_stream, d_stream.device
        self.pad = PLAIN_PAD if plain else 0
        self.index_info, self.t = _device_index(d_stream, max_frames, s, zstd=self.zstd, plain=plain)
        self.n = self.index_info.nframes
        self.content_off = torch.empty(self.n + 1, dtype=torch.int64, device=self.dev)
        d_info = torch.zeros(ctypes.sizeof(FrameIndex), dtype=torch.uint8, device=self.dev)
        self.work = torch.empty(L.zmt_range_workspace_bytes(self.n, 0), dtype=torch.uint8, device=self.dev)
        p = lambda k: self.t[k].data_ptr()
        if self.zstd:
            rc = L.zmt_zstd_content_offsets_device(self.n, p("frame_off"), p("frame_csize"), p("expect"), self.content_off.data_ptr(),
                                                   d_info.data_ptr(), self.work.data_ptr(), s.cuda_stream)
        else:
            rc = L.zmt_lz4_content_offsets_device(self._base(), self.n, p("frame_off"), p("frame_csize"), self.content_off.data_ptr(),
                                                  d_info.data_ptr(), self.work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("content table failed: %s" % ST_NAMES.get(rc, rc))
        s.synchronize()
        self.content_info = FrameIndex.from_buffer_copy(d_info.cpu().numpy().tobytes())
        if self.content_info.status != 0:
            raise ValueError("stream cannot be range-read: %s in frame %d at offset %d" % (
                ST_NAMES.get(self.content_info.status, self.content_info.status), self.content_info.bad_frame, self.content_info.bad_offset))
        self.content_size = self.content_info.out_bytes
        self.scratch = torch.empty(1, dtype=torch.uint8, device=self.dev)
        self.read_work = torch.empty(1, dtype=torch.uint8, device=self.dev)
        self.plan = None
        self.read_work_bytes = 0

    def _base(self):
        return self.d_stream.data_ptr() - self.pad

    def _grow(self, name, nbytes):
        torch = _torch()
        if getattr(self, name).numel() < nbytes:
            setattr(self, name, torch.empty(nbytes, dtype=torch.uint8, device=self.dev))
        return getattr(self, name)

    def read(self, ranges, stream=None):
        torch = _torch(); L = lib()
        s = stream if stream is not None else torch.cuda.current_stream()
        r = torch.as_tensor(ranges)
        if r.dtype != torch.int64 or r.dim() != 2 or r.shape[1] != 2:
            raise ValueError("ranges must be an int64 (M, 2) tensor of (start, length)")
        r = r.to(self.dev).contiguous()
        m = r.shape[0]
        work = self._grow("work", L.zmt_range_workspace_bytes(self.n, m))
        dst_off = torch.empty(m + 1, dtype=torch.int64, device=self.dev)
        d_plan = torch.zeros(ctypes.sizeof(RangePlan), dtype=torch.uint8, device=self.dev)
        p = lambda k: self.t[k].data_ptr()
        if self.zstd:
            rc = L.zmt_zstd_range_plan_device(self.n, p("frame_csize"), p("first_blk"), p("frame_scratch"), self.content_off.data_ptr(), r.data_ptr(), m,
                                              dst_off.data_ptr(), d_plan.data_ptr(), work.data_ptr(), s.cuda_stream)
        else:
            rc = L.zmt_lz4_range_plan_device(self.n, p("frame_csize"), self.content_off.data_ptr(), r.data_ptr(), m, dst_off.data_ptr(),
                                             d_plan.data_ptr(), work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("range plan failed: %s" % ST_NAMES.get(rc, rc))
        s.synchronize()
        plan = RangePlan.from_buffer_copy(d_plan.cpu().numpy().tobytes())
        self.plan = plan
        scratch = self._grow("scratch", max(plan.scratch_bytes, 1))
        ws = (L.zmt_zstd_range_read_workspace_bytes if self.zstd else L.zmt_lz4_range_read_workspace_bytes)(ctypes.byref(plan))
        self.read_work_bytes = ws
        read_work = self._grow("read_work", max(ws, 1))
        out = torch.empty(max(plan.dst_bytes, 1), dtype=torch.uint8, device=self.dev)
        status = torch.empty(max(m, 1), dtype=torch.int32, device=self.dev)
        if self.zstd:
            rc = L.zmt_zstd_range_read_device(self._base(), p("frame_off"), p("frame_csize"), p("expect"), p("frame_seq"), ctypes.byref(plan), out.data_ptr(),
                                              dst_off.data_ptr(), status.data_ptr(), scratch.data_ptr(), read_work.data_ptr(), work.data_ptr(), s.cuda_stream)
        else:
            rc = L.zmt_lz4_range_read_device(self._base(), p("frame_off"), p("frame_csize"), ctypes.byref(plan), out.data_ptr(), dst_off.data_ptr(),
                                             status.data_ptr(), scratch.data_ptr(), read_work.data_ptr(), work.data_ptr(), s.cuda_stream)
        if rc != 0:
            raise RuntimeError("range read failed: %s" % ST_NAMES.get(rc, rc))
        return out[: plan.dst_bytes], dst_off, status[:m]
