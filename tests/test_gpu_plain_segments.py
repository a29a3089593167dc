"""LZ4F frames larger than a batch, decoded as chains of segments of whole blocks: through the device API
(zmt_lz4_decompress_segments_device) cut at block boundaries, and through LZ4MT_decompressDCtx on plain .lz4 streams with
small batches (ZSTDMT_B200_PLAIN_MB).  Every case compares the GPU's output with the source bytes."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import zstdmt_b200 as z
import _lz4corpus as lc
import _oracle as o
from test_frame_segments import boundaries
from test_gpu_plain_streams import lz4f

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def sample(cuts, k=20):
    if len(cuts) <= k:
        return list(cuts)
    return [cuts[int(i)] for i in np.linspace(0, len(cuts) - 1, k)]


# ---------------------------------------------------------------- 1. the device API, cut at block boundaries
@pytest.mark.parametrize("lay", ["full", "short"])
@pytest.mark.parametrize("bchk", [False, True])
def test_device_segments_on_linked_corpus_frames_at_every_cut(gpu, lay, bchk):
    """_lz4corpus `linked`: block b of the 64-block frame starts with a match at distance D into block b-1, the 2-block
    frames start block 1 with a match at offset 65535.  Cut in front of such a block, those matches read the history the
    earlier segment left below the segment's output."""
    for i, (fr, src, info) in enumerate(lc.case("linked", lay, bchk)):
        cuts, _, _ = boundaries(fr)
        cuts = cuts[:-1]                                    # behind the last block: the end mark alone follows
        for j, c in enumerate(cuts):
            back, st = z.lz4_decode_segments(fr, [c])
            assert st == 0 and np.array_equal(back, src), (i, c)
            rows = info[j + 1][0]
            stored = int.from_bytes(fr[c:c + 4].tobytes(), "little") >> 31
            if lay == "full" and not stored:                 # the segment's first sequence is a match into the history
                assert rows[0][0] == 0 and rows[0][1] > 0, (i, j)
        back, st = z.lz4_decode_segments(fr, cuts)         # every block a segment of its own
        assert st == 0 and np.array_equal(back, src), i
    if lay == "full":                                       # a match at offset 65535 right behind a cut
        assert any(off == 65535 for _, _, info in lc.case("linked", lay, bchk) for rows, _, _ in info[1:2] for _, off, _ in rows[:2])


@pytest.mark.parametrize("prefs", [dict(blockSizeID=4, blockMode=0, contentChecksumFlag=1),
                                   dict(blockSizeID=4, blockMode=0, blockChecksumFlag=1, contentSize=1),
                                   dict(blockSizeID=5, blockMode=1, contentChecksumFlag=1),
                                   dict(blockSizeID=7, blockMode=1, contentChecksumFlag=1, contentSize=1)])
def test_device_segments_on_liblz4_frames(gpu, prefs):
    src = z.gen_stream(z.GEN_MIX, (9 << 20) + 777, 1 << 20, first=4)
    if prefs.get("contentSize"):
        prefs = dict(prefs, contentSize=int(src.size))
    fr = lz4f(src, **prefs)
    cuts = boundaries(fr)[0][:-1]
    for c in sample(cuts):
        back, st = z.lz4_decode_segments(fr, [c])
        assert st == 0 and np.array_equal(back, src), c
    back, st = z.lz4_decode_segments(fr, sample(cuts, 7))
    assert st == 0 and np.array_equal(back, src)
    if prefs.get("contentChecksumFlag"):                      # the checksum runs across the segments: a flipped stored byte fails
        bad = fr.copy(); bad[-2] ^= 0x10
        _, st = z.lz4_decode_segments(bad, sample(cuts, 3))
        assert z.ST_NAMES[st] == "content_checksum"


# ---------------------------------------------------------------- 2. the callback API in small batches
def big_frames():
    a = z.gen_stream(z.GEN_MIX, (24 << 20) + 12345, 1 << 20, first=7)
    b = z.gen_stream(z.GEN_TEXT, (33 << 20) + 99, 1 << 20, first=8)
    return [("linked64k", a, dict(blockSizeID=4, blockMode=0, contentSize=int(a.size))),
            ("indep4m_cchk", b, dict(blockSizeID=7, blockMode=1, contentChecksumFlag=1))]


@pytest.mark.parametrize("idx", [0, 1], ids=["linked64k", "indep4m_cchk"])
def test_callback_api_decodes_frames_larger_than_a_batch(gpu, idx, monkeypatch):
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", "1")
    _, src, prefs = big_frames()[idx]
    small = [z.gen_stream(z.GEN_TEXT, n, 1 << 20, first=n) for n in (1000, 300000)]
    skip = np.frombuffer(bytes.fromhex("502a4d18") + (6).to_bytes(4, "little") + b"abcdef", np.uint8)
    big = lz4f(src, **prefs)
    stream = np.concatenate([lz4f(small[0]), big, skip, lz4f(small[1], blockMode=0), big])
    want = np.concatenate([small[0], src, small[1], src])
    rc, back, st = z.decompress_mem(z.CODEC_LZ4, stream, want.size + 16, threads=4, inputsize=1 << 20)
    assert rc == 0, z.lib().LZ4MT_getErrorString(rc)
    assert back.size == want.size and np.array_equal(back, want)
    assert st["insize"] == stream.size and st["outsize"] == want.size


def test_callback_api_segments_a_small_frame_with_a_large_output(gpu, monkeypatch):
    """A frame far smaller than a batch whose content is more than four batches: cut by its output room (the host's rule:
    a batch of input or four batches of output room, whichever its blocks reach first), so the output stays bounded too."""
    src = np.tile(z.gen_stream(z.GEN_TEXT, 4096, 1 << 20, first=5), 4096)             # 16 MiB of content
    fr = lz4f(src, blockSizeID=4, blockMode=0, contentChecksumFlag=1, contentSize=int(src.size))
    assert fr.size < (1 << 20) // 2
    hl = 7 + 8
    rc, end, room, last = z.lz4f_segment(fr, hl, int(fr[4]), int(fr[5]), 1 << 20, 4 << 20)
    assert rc == 0 and not last and room == 4 << 20 and end < fr.size    # the output room ends the first segment
    small = z.gen_stream(z.GEN_MIX, 70000, 1 << 20, first=6)
    stream = np.concatenate([lz4f(small), fr, lz4f(small, blockMode=0)])
    want = np.concatenate([small, src, small])
    for mb in ("1", "64"):                                   # segmented by output room / one batch, as before
        monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", mb)
        rc, back, st = z.decompress_mem(z.CODEC_LZ4, stream, want.size + 16, threads=4, inputsize=1 << 20)
        assert rc == 0, z.lib().LZ4MT_getErrorString(rc)
        assert np.array_equal(back, want) and st["insize"] == stream.size and st["outsize"] == want.size
    bad = stream.copy(); bad[lz4f(small).size + fr.size - 1] ^= 0x20    # its content checksum, checked on the last segment
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", "1")
    rc, _, _ = z.decompress_mem(z.CODEC_LZ4, bad, want.size + 16, threads=4, inputsize=1 << 20)
    assert b"contentChecksum" in z.lib().LZ4MT_getErrorString(rc)


# ---------------------------------------------------------------- 3. output leaves before the frame's input has all arrived
def test_first_write_comes_before_the_last_read(gpu, monkeypatch):
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", "1")
    src = z.gen_stream(z.GEN_MIX, 32 << 20, 1 << 20, first=9)
    fr = lz4f(src, blockSizeID=4, blockMode=0, contentChecksumFlag=1)
    L = z.lib()
    events, state = [], {"at": 0}
    out = bytearray()

    def rd(_, b):
        n = min(b.contents.size, fr.size - state["at"])
        ctypes.memmove(b.contents.buf, fr.ctypes.data + state["at"], n)
        b.contents.size = n; state["at"] += n
        events.append(("r", state["at"]))
        return 0

    def wr(_, b):
        out.extend(ctypes.string_at(b.contents.buf, b.contents.size))
        events.append(("w", state["at"]))
        return 0

    rdf, wrf = z.RW_FN(rd), z.RW_FN(wr)
    rw = z.RdWr(rdf, None, wrf, None)
    ctx = L.LZ4MT_createDCtx(4, 1 << 20)
    try:
        rc = L.LZ4MT_decompressDCtx(ctx, ctypes.byref(rw))
        assert rc == 0, L.LZ4MT_getErrorString(rc)
        assert L.LZ4MT_GetInsizeDCtx(ctx) == fr.size and L.LZ4MT_GetOutsizeDCtx(ctx) == src.size
    finally:
        L.LZ4MT_freeDCtx(ctx)
    assert bytes(out) == src.tobytes()
    first_w = next(at for kind, at in events if kind == "w")
    assert first_w <= fr.size - (1 << 20), (first_w, fr.size)


# ---------------------------------------------------------------- 4. memory stays bounded (a subprocess without torch)
_RSS_SCRIPT = textwrap.dedent("""
    import ctypes, resource, sys
    sys.path.insert(0, sys.argv[1])
    import zstdmt_b200 as z
    L = z.lib()
    def run(path):
        f = open(path, "rb")
        def rd(_, b):
            buf = (ctypes.c_char * b.contents.size).from_address(b.contents.buf)
            b.contents.size = f.readinto(buf)
            return 0
        def wr(_, b):
            return 0
        rdf, wrf = z.RW_FN(rd), z.RW_FN(wr)
        rw = z.RdWr(rdf, None, wrf, None)
        ctx = L.LZ4MT_createDCtx(4, 1 << 20)
        rc = L.LZ4MT_decompressDCtx(ctx, ctypes.byref(rw))
        out = L.LZ4MT_GetOutsizeDCtx(ctx)
        L.LZ4MT_freeDCtx(ctx); f.close()
        return rc, out
    rc, _ = run(sys.argv[2])
    assert rc == 0, rc
    before = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    rc, out = run(sys.argv[3])
    after = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    print(rc, out, before, after)
""")


def write_lz4_stream(path, total):
    """One linked-block LZ4F frame of `total` content bytes with a content checksum, written by liblz4's streaming API."""
    write_lz4_stream_prefs(path, total, dict(blockSizeID=4, blockMode=0, contentChecksumFlag=1))


def write_lz4_stream_prefs(path, total, kw, piece=8 << 20):
    """One LZ4F frame of `total` content bytes (GEN_MIX), LZ4F preferences `kw`, written by liblz4's streaming API in pieces."""
    L = ctypes.CDLL("liblz4.so.1")
    L.LZ4F_createCompressionContext.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
    L.LZ4F_compressBound.restype = ctypes.c_size_t; L.LZ4F_compressBound.argtypes = [ctypes.c_size_t, ctypes.c_void_p]
    for fn in ("LZ4F_compressBegin", "LZ4F_compressEnd"):
        getattr(L, fn).restype = ctypes.c_size_t
    L.LZ4F_compressBegin.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.LZ4F_compressUpdate.restype = ctypes.c_size_t
    L.LZ4F_compressUpdate.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.LZ4F_compressEnd.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.LZ4F_freeCompressionContext.argtypes = [ctypes.c_void_p]
    from test_gpu_plain_streams import LZ4FPrefs
    prefs = LZ4FPrefs()
    for k, v in kw.items():
        setattr(prefs, k, v)
    cctx = ctypes.c_void_p()
    assert L.LZ4F_createCompressionContext(ctypes.byref(cctx), 100) == 0
    cap = L.LZ4F_compressBound(piece, ctypes.byref(prefs)) + 64
    dst = np.empty(cap, np.uint8)
    with open(path, "wb") as f:
        n = L.LZ4F_compressBegin(cctx, dst.ctypes.data, cap, ctypes.byref(prefs)); assert n < (1 << 62); f.write(dst[:n].tobytes())
        at = 0
        while at < total:
            k = min(piece, total - at)
            src = z.gen_stream(z.GEN_MIX, k, 1 << 20, first=at // (1 << 20))
            n = L.LZ4F_compressUpdate(cctx, dst.ctypes.data, cap, src.ctypes.data, k, None); assert n < (1 << 62); f.write(dst[:n].tobytes())
            at += k
        n = L.LZ4F_compressEnd(cctx, dst.ctypes.data, cap, None); assert n < (1 << 62); f.write(dst[:n].tobytes())
    L.LZ4F_freeCompressionContext(cctx)


def test_memory_is_bounded_for_a_2gib_frame(gpu, tmp_path):
    total = 2 << 30
    big, warm = str(tmp_path / "big.lz4"), str(tmp_path / "warm.lz4")
    write_lz4_stream(big, total)
    write_lz4_stream(warm, 40 << 20)
    env = dict(os.environ, ZSTDMT_B200_PLAIN_MB="16")
    r = subprocess.run([sys.executable, "-c", _RSS_SCRIPT, ROOT, warm, big], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    rc, out, before, after = (int(x) for x in r.stdout.split())
    assert rc == 0 and out == total
    assert (after - before) * 1024 < (512 << 20), (before, after)      # ru_maxrss in KiB


# ---------------------------------------------------------------- 5. errors in a later segment: the whole-frame path's error
def _errors_case():
    src = z.gen_stream(z.GEN_MIX, (8 << 20) + 5, 1 << 20, first=12)
    fr = lz4f(src, blockSizeID=4, blockMode=0, contentChecksumFlag=1, contentSize=int(src.size))
    return src, fr


def _decode(stream, cap, plain_mb, monkeypatch):
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", str(plain_mb))
    rc, back, _ = z.decompress_mem(z.CODEC_LZ4, stream, cap, threads=4, inputsize=1 << 20)
    return rc, back


@pytest.mark.parametrize("damage", ["content_checksum", "block_in_third_segment", "truncated", "content_size"])
def test_errors_in_a_later_segment_match_the_whole_frame_path(gpu, damage, monkeypatch):
    src, fr = _errors_case()
    cuts = boundaries(fr)[0]
    bad = fr.copy()
    if damage == "content_checksum":
        bad[-1] ^= 0x01
    elif damage == "block_in_third_segment":
        k = next(i for i, x in enumerate(cuts) if x > (5 << 19) and not bad[x + 3] >> 7)    # 1 MiB segments: a compressed block in the third
        c = cuts[k]
        bad[c + 4:c + 4 + 64] = 0xFF                             # its first token and what follows
    elif damage == "truncated":
        bad = fr[: cuts[len(cuts) // 2] + 1000]
    else:
        bad[6:14] = np.frombuffer(int(src.size + 1).to_bytes(8, "little"), np.uint8)
        bad[14] = (o.xxh32(bad[4:14]) >> 8) & 0xFF               # a valid header checksum over the wrong size
    L = z.lib()
    rc_whole, _ = _decode(bad, src.size + 64, 64, monkeypatch)
    rc_seg, out_seg = _decode(bad, src.size + 64, 1, monkeypatch)
    assert L.LZ4MT_isError(rc_whole) and L.LZ4MT_isError(rc_seg)
    assert L.LZ4MT_getErrorString(rc_seg) == L.LZ4MT_getErrorString(rc_whole), (L.LZ4MT_getErrorString(rc_seg), L.LZ4MT_getErrorString(rc_whole))
    # what was written before the failing segment is the frame's leading content; a damaged block that still parses
    # decodes to wrong bytes, which are written like any others until the content checksum fails on the last segment
    good = out_seg.size if damage != "block_in_third_segment" else min(out_seg.size, (k + 1) * 65536)
    assert out_seg.size > 0 and np.array_equal(out_seg[:good], src[:good])
    if damage == "content_checksum":
        assert b"contentChecksum" in L.LZ4MT_getErrorString(rc_seg)
