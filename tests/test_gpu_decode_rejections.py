"""The host's decisions on bad or edge-case input, pinned exactly: for each stream the call's return code, the
*_getErrorString text and the list of fn_write sizes up to the error.

Plain .lz4 / .zst streams are cut into frames on the host (the header checks, the truncation and stray-byte rules, the
zstd block table) and written in pieces of at most one read's size, whole frames and segments alike; a host-side
rejection returns before the frames ahead of it in the same batch are decoded, so nothing of that batch is written.
Container-framed streams are checked by the reader thread (the LZ4F room rule, the zstd frame walk) before a batch is
submitted."""
import ctypes
import struct

import numpy as np
import pytest

import zstdmt_b200 as z
from test_gpu_plain_streams import lz4f, zstd1

pytestmark = pytest.mark.gpu

SMAX = 1 << 64
# (data_error, frame_decompress, library) of each codec (include/lz4-mt.h, include/zstd-mt.h)
DATA, FRAME, LIBRARY = "data", "frame", "library"
ERR = {z.CODEC_LZ4: {DATA: 4, FRAME: 6, LIBRARY: 8}, z.CODEC_ZSTD: {DATA: 5, FRAME: 7, LIBRARY: 9}}
API = {z.CODEC_LZ4: "LZ4MT", z.CODEC_ZSTD: "ZSTDCB"}
MALFORMED, CUT = b"Malformed input", b"Could not decompress frame at once"


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


class Io:
    """fn_read serves `src`; fn_write records every write."""

    def __init__(self, src):
        self.src, self.pos, self.writes = np.ascontiguousarray(src, np.uint8), 0, []
        self.rw = z.RdWr(z.RW_FN(self._rd), None, z.RW_FN(self._wr), None)

    def _rd(self, arg, b):
        take = min(b.contents.size, self.src.size - self.pos)
        if take:
            ctypes.memmove(b.contents.buf, self.src[self.pos:].ctypes.data, take)
        self.pos += take; b.contents.size = take
        return 0

    def _wr(self, arg, b):
        self.writes.append(ctypes.string_at(b.contents.buf, b.contents.size))
        return 0


def decode(codec, stream, inputsize=0):
    """One create / decompress / free; returns (return code, error string or None, sizes written, bytes written)."""
    L = z.lib(); api = API[codec]
    io = Io(stream)
    ctx = getattr(L, api + "_createDCtx")(4, inputsize)
    assert ctx
    rc = getattr(L, api + "_decompressDCtx")(ctx, ctypes.byref(io.rw))
    getattr(L, api + "_freeDCtx")(ctx)
    msg = getattr(L, api + "_getErrorString")(rc) if rc else None
    return rc, msg, [len(w) for w in io.writes], b"".join(io.writes)


def check(codec, stream, err, msg, writes, inputsize=0):
    rc, got_msg, got_writes, _ = decode(codec, stream, inputsize)
    assert (rc, got_msg, got_writes) == (SMAX - ERR[codec][err], msg, writes)


def u8(b):
    return np.frombuffer(bytes(b), np.uint8)


def pieces(n, piece):
    return [piece] * (n // piece) + ([n % piece] if n % piece else [])


# ---------------------------------------------------------------- plain .lz4
@pytest.fixture(scope="module")
def good_lz4(gpu):
    a = z.gen_stream(z.GEN_TEXT, 200000, 1 << 20)
    b = z.gen_stream(z.GEN_MIX, 70000, 1 << 20, first=3)
    return a, b, lz4f(a), lz4f(b, blockMode=1, contentChecksumFlag=1)


def test_plain_lz4_flg_version(good_lz4):
    _, _, fa, fb = good_lz4
    bad = fb.copy(); bad[4] = (bad[4] & 0x3F) | 0x80                           # version 10
    check(z.CODEC_LZ4, bad, LIBRARY, b"ERROR_frameHeader_incomplete", [])
    check(z.CODEC_LZ4, np.concatenate([fa, bad]), LIBRARY, b"ERROR_frameHeader_incomplete", [])


def test_plain_lz4_block_size_id_below_4(good_lz4):
    _, _, fa, fb = good_lz4
    bad = fb.copy(); bad[5] = 3 << 4
    check(z.CODEC_LZ4, bad, LIBRARY, b"ERROR_frameHeader_incomplete", [])
    check(z.CODEC_LZ4, np.concatenate([fa, bad]), LIBRARY, b"ERROR_frameHeader_incomplete", [])


def test_plain_lz4_content_size_above_the_block_bound(good_lz4):
    """One 64 KiB block holding 1000 bytes: a content-size field of 70 000 exceeds the most the blocks decode to."""
    src = z.gen_stream(z.GEN_TEXT, 1000, 1 << 20)
    fr = lz4f(src, blockSizeID=4, contentSize=1000)
    assert fr[4] & 8
    bad = fr.copy(); bad[6:14] = u8(struct.pack("<Q", 70000))
    check(z.CODEC_LZ4, bad, LIBRARY, b"ERROR_frameSize_wrong", [])
    check(z.CODEC_LZ4, np.concatenate([good_lz4[2], bad]), LIBRARY, b"ERROR_frameSize_wrong", [])
    ok = fr.copy(); ok[6:14] = u8(struct.pack("<Q", 65536))                     # at the bound: the device judges the size
    rc, _, _, _ = decode(z.CODEC_LZ4, ok)
    assert rc == SMAX - ERR[z.CODEC_LZ4][LIBRARY]


def test_plain_lz4_cut_short_at_eof(good_lz4):
    _, _, fa, fb = good_lz4
    check(z.CODEC_LZ4, fa[:-3], FRAME, CUT, [])
    check(z.CODEC_LZ4, np.concatenate([fa, fb[:-3]]), FRAME, CUT, [])
    check(z.CODEC_LZ4, np.concatenate([fa, fb[:5]]), DATA, MALFORMED, [])      # FLG / BD not all there


def test_plain_lz4_truncated_skippable_frame(good_lz4):
    _, _, fa, _ = good_lz4
    skip = u8(struct.pack("<II", 0x184D2A53, 100) + b"x" * 99)
    check(z.CODEC_LZ4, np.concatenate([fa, skip]), DATA, MALFORMED, [])
    check(z.CODEC_LZ4, np.concatenate([fa, skip[:6]]), DATA, MALFORMED, [])


def test_plain_lz4_stray_bytes_after_a_good_frame(good_lz4):
    _, _, fa, _ = good_lz4
    check(z.CODEC_LZ4, np.concatenate([fa, u8(b"\x01\x02\x03")]), DATA, MALFORMED, [])


def test_plain_lz4_bad_magic_after_two_good_frames(good_lz4):
    _, _, fa, fb = good_lz4
    check(z.CODEC_LZ4, np.concatenate([fa, fb, u8(b"\x00\x22\x4d\x18" + b"\x00" * 12)]), DATA, MALFORMED, [])


def test_plain_lz4_writes_in_read_sized_pieces(good_lz4):
    """Each frame is written in pieces of at most one read (inputsize, here 100 000 bytes)."""
    a, b, fa, fb = good_lz4
    rc, msg, writes, data = decode(z.CODEC_LZ4, np.concatenate([fa, fb]), inputsize=100000)
    assert rc == 0 and writes == pieces(a.size, 100000) + pieces(b.size, 100000)
    assert data == np.concatenate([a, b]).tobytes()


def test_plain_lz4_segments_write_in_read_sized_pieces(gpu, monkeypatch):
    """Incompressible 64 KiB blocks are stored (65 540 bytes each): with 1 MiB batches a segment ends behind 16 blocks,
    so a 56-block frame decodes as segments of 16, 16, 16 and 8 blocks, each written in pieces of 100 000 bytes."""
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", "1")
    src = z.gen_stream(z.GEN_RANDOM, 56 << 16, 1 << 20)
    fr = lz4f(src, blockSizeID=4, contentChecksumFlag=1)
    assert fr.size == 7 + 56 * 65540 + 4 + 4
    rc, msg, writes, data = decode(z.CODEC_LZ4, fr, inputsize=100000)
    assert rc == 0 and writes == pieces(1 << 20, 100000) * 3 + pieces(8 << 16, 100000)
    assert data == src.tobytes()
    check(z.CODEC_LZ4, fr[:-6], FRAME, CUT, pieces(1 << 20, 100000) * 3, inputsize=100000)


# ---------------------------------------------------------------- plain .zst
@pytest.fixture(scope="module")
def good_zst(gpu):
    a = z.gen_stream(z.GEN_TEXT, 300000, 1 << 20)
    b = z.gen_stream(z.GEN_MIX, 90000, 1 << 20, first=3)
    return a, b, zstd1(a, 3), zstd1(b, 1)


def zst_header(fhd, rest):
    return u8(struct.pack("<IB", 0xFD2FB528, fhd) + rest)


def test_plain_zst_dictionary_id(good_zst):
    bad = zst_header(0x21, b"\x07\x10" + struct.pack("<I", 1 | (16 << 3))[:3] + b"y" * 16)     # 1-byte dictionary ID
    check(z.CODEC_ZSTD, bad, LIBRARY, b"stream type not supported by the GPU path", [])
    check(z.CODEC_ZSTD, np.concatenate([good_zst[2], bad]), LIBRARY, b"stream type not supported by the GPU path", [])


def test_plain_zst_reserved_header_bit(good_zst):
    bad = good_zst[3].copy(); bad[4] |= 0x08
    check(z.CODEC_ZSTD, bad, LIBRARY, b"ERROR_frameHeader_incomplete", [])
    check(z.CODEC_ZSTD, np.concatenate([good_zst[2], bad]), LIBRARY, b"ERROR_frameHeader_incomplete", [])


def test_plain_zst_block_type_3(good_zst):
    bad = zst_header(0x20, b"\x10" + struct.pack("<I", 1 | (3 << 1) | (16 << 3))[:3] + b"z" * 16)
    check(z.CODEC_ZSTD, bad, LIBRARY, b"ERROR_decompressionFailed", [])
    check(z.CODEC_ZSTD, np.concatenate([good_zst[2], bad]), LIBRARY, b"ERROR_decompressionFailed", [])


def test_plain_zst_cut_short_at_eof(good_zst):
    _, _, fa, fb = good_zst
    check(z.CODEC_ZSTD, fa[:-3], FRAME, CUT, [])
    check(z.CODEC_ZSTD, np.concatenate([fa, fb[:-3]]), FRAME, CUT, [])


def test_plain_zst_bad_magic_between_frames(good_zst):
    _, _, fa, fb = good_zst
    check(z.CODEC_ZSTD, np.concatenate([fa, u8(b"\x00\x01\x02\x03" + b"\x00" * 12), fb]), DATA, MALFORMED, [])


def test_plain_zst_frame_of_many_blocks(good_zst):
    """10 000 raw blocks of 16 bytes: more block descriptors than the block table's first growth holds."""
    a, _, fa, _ = good_zst
    many = z.gen_stream(z.GEN_MIX, 10000 * 16, 1 << 20)
    parts = [struct.pack("<IBI", 0xFD2FB528, 0xA0, many.size)]
    for o in range(0, many.size, 16):
        parts += [struct.pack("<I", (16 << 3) | (o + 16 == many.size))[:3], many[o:o + 16].tobytes()]
    fm = u8(b"".join(parts))
    rc, msg, writes, data = decode(z.CODEC_ZSTD, np.concatenate([fa, fm, fa]), inputsize=100000)
    assert rc == 0 and writes == pieces(a.size, 100000) + pieces(many.size, 100000) + pieces(a.size, 100000)
    assert data == np.concatenate([a, many, a]).tobytes()


# ---------------------------------------------------------------- container-framed streams
def wrap(payload):
    return np.concatenate([u8(struct.pack("<III", 0x184D2A50, 4, payload.size)), payload])


@pytest.fixture(scope="module")
def small_frames(gpu):
    src = z.gen_stream(z.GEN_MIX, 5 * 65536 + 17, 1 << 20)
    rc, f4, _ = z.compress_mem(z.CODEC_LZ4, src, threads=4, level=1, chunk=65536)
    assert rc == 0
    rc, fz, _ = z.compress_mem(z.CODEC_ZSTD, src, threads=4, level=3, chunk=65536)
    assert rc == 0
    return {z.CODEC_LZ4: f4, z.CODEC_ZSTD: fz}


@pytest.mark.parametrize("behind", [False, True])
def test_container_lz4_content_size_above_255x(small_frames, behind):
    """LZ4F content size 10^9 in a 19-byte payload: above 255 x payload + 65 536."""
    bad = wrap(u8(b"\x04\x22\x4d\x18\x68\x40" + struct.pack("<Q", 10 ** 9) + b"\x00" + b"\x00" * 4))
    stream = np.concatenate([small_frames[z.CODEC_LZ4], bad]) if behind else np.concatenate([bad, small_frames[z.CODEC_LZ4]])
    check(z.CODEC_LZ4, stream, LIBRARY, b"ERROR_frameHeader_incomplete", [])


@pytest.mark.parametrize("behind", [False, True])
def test_container_zstd_trailing_bytes(small_frames, behind):
    bad = wrap(np.concatenate([zstd1(z.gen_stream(z.GEN_TEXT, 5000, 1 << 20), 3), u8(b"\x00")]))
    stream = np.concatenate([small_frames[z.CODEC_ZSTD], bad]) if behind else np.concatenate([bad, small_frames[z.CODEC_ZSTD]])
    check(z.CODEC_ZSTD, stream, FRAME, CUT, [])


@pytest.mark.parametrize("behind", [False, True])
def test_container_zstd_dictionary_id(small_frames, behind):
    bad = wrap(zst_header(0x21, b"\x07\x00" + struct.pack("<I", 1)[:3]))
    stream = np.concatenate([small_frames[z.CODEC_ZSTD], bad]) if behind else np.concatenate([bad, small_frames[z.CODEC_ZSTD]])
    check(z.CODEC_ZSTD, stream, LIBRARY, b"stream type not supported by the GPU path", [])
