"""zstd frames larger than a batch, decoded as chains of segments of whole blocks: through the device API
(zmt_zstd_decompress_segments_device) cut at block boundaries, and through ZSTDCB_decompressDCtx on plain .zst streams
with small batches (ZSTDMT_B200_PLAIN_MB).  What crosses a cut — the window, the repeat offsets, inherited Huffman trees
and sequence tables, the running XXH64 and the content size — is exercised on the corpus frames of tests/_zcorpus.py,
whose oracle traces show that the cuts chosen here do carry it.  Every case compares the GPU's output with the source."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import _zcorpus as zc
import zstdmt_b200 as z
from test_gpu_plain_streams import zstd1, zstd_adv
from test_zstd_decode_corpus import host_scan
from test_zstd_frame_segments import header_walk

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CORPUS = ["reps", "reps_predef", "tables", "literals", "deep", "dense", "far"]


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def sample(xs, k=20):
    if len(xs) <= k:
        return list(xs)
    return [xs[int(i)] for i in np.linspace(0, len(xs) - 1, k)]


def block_cuts(fr):
    """Frame offsets behind every block but the last."""
    return [a + n for a, n, _ in header_walk(fr)["blocks"]][:-1]


# ---------------------------------------------------------------- 1. the device API, cut at block boundaries
def carried_state(tr):
    """What a cut in front of block k carries, per k, from the oracle's trace: a treeless block from k on whose tree lies
    before k, a Repeat_Mode table from k on whose describer lies before k, block k's first sequence a repeat-offset code,
    and how many blocks back the farthest match of block k reaches."""
    lt = tr.col("lit_type")
    last_tree, tree_src = None, {}
    for b in range(len(lt)):
        if lt[b] == 2:
            last_tree = b
        elif lt[b] == 3:
            tree_src[b] = last_tree
    reps = [(r["block"], r["src"]) for r in zc.repeat_sources(tr) if isinstance(r["src"], (int, np.integer))]
    sb, first = zc.seq_blocks(tr), tr.col("seq_first")
    dist = zc.match_block_distance(tr)
    far = np.zeros(len(lt), np.int64)
    if len(sb):
        np.maximum.at(far, sb, dist)
    nseq = tr.col("nseq")
    rep_first = [b for b in range(len(lt)) if nseq[b] > 0 and tr.seq[first[b], 1] <= 3]
    return tree_src, reps, rep_first, far


@pytest.mark.parametrize("name", CORPUS)
def test_device_segments_on_corpus_frames(gpu, name):
    src, fr = zc.case(name)
    tr = zc.trace(name)
    cuts = block_cuts(fr)
    ks = sample(list(range(1, len(cuts) + 1)), 12)
    for k in ks:                                              # one cut in front of block k
        back, st = z.zstd_decode_segments(fr, [cuts[k - 1]])
        assert st == 0 and np.array_equal(back, src), (name, k)
    back, st = z.zstd_decode_segments(fr, cuts)               # every block a segment of its own
    assert st == 0 and np.array_equal(back, src), name
    # the cuts above carried what the case exists for (every block its own segment: any earlier block is in history)
    tree_src, reps, rep_first, far = carried_state(tr)
    if name == "literals":
        assert any(s is not None for s in tree_src.values())              # a treeless block's tree in an earlier segment
    if name == "tables":
        assert any(s < b for b, s in reps)                                 # a Repeat_Mode table described in an earlier segment
    if name in ("reps", "reps_predef"):
        assert any(b > 0 for b in rep_first)                               # a segment whose first sequence is a repeat code
    if name == "deep":
        assert far.max() >= 100                                            # matches hundreds of segments back
    if name == "far":
        assert zc.of_codes(tr).max() >= 25 and header_walk(fr)["window"] >= 32 << 20      # offsets 16-33 MiB back


def test_device_segments_cross_state_at_single_cuts(gpu):
    """One cut exactly where the state must cross it: in front of a treeless block whose tree lies before the cut, in front
    of a Repeat_Mode block whose describer lies before the cut, in front of a block whose first sequence is a repeat code."""
    for name, pick in (("literals", lambda ts, rp, rf: [b for b, s in ts.items() if s is not None and s < b - 1]),
                       ("tables", lambda ts, rp, rf: [b for b, s in rp if s < b - 1]),
                       ("reps", lambda ts, rp, rf: [b for b in rf if b > 0])):
        src, fr = zc.case(name)
        cuts = block_cuts(fr)
        ks = pick(*carried_state(zc.trace(name))[:3])
        assert ks, name
        for k in sample(ks, 6):
            back, st = z.zstd_decode_segments(fr, [cuts[k - 1]])
            assert st == 0 and np.array_equal(back, src), (name, k)


@pytest.mark.parametrize("level,chk,cs", [(1, 1, 1), (3, 1, 0), (19, 0, 1)])
def test_device_segments_on_libzstd_frames(gpu, level, chk, cs):
    src = z.gen_stream(z.GEN_MIX, (9 << 20) + 777, 1 << 20, first=4)
    fr = zstd_adv(src, level, checksum=chk, content_size=cs) if cs else zstd_adv(src, level, checksum=chk, pieces=[src.size // 2, src.size - src.size // 2])
    cuts = block_cuts(fr)
    for c in sample(cuts, 10):
        back, st = z.zstd_decode_segments(fr, [c])
        assert st == 0 and np.array_equal(back, src), c
    back, st = z.zstd_decode_segments(fr, sample(cuts, 7))
    assert st == 0 and np.array_equal(back, src)
    if chk:                                                   # the checksum runs across the segments: a flipped stored byte fails
        bad = fr.copy(); bad[-2] ^= 0x10
        _, st = z.zstd_decode_segments(bad, sample(cuts, 3))
        assert z.ST_NAMES[st] == "content_checksum"


# ---------------------------------------------------------------- 2. the callback API in small batches
def test_callback_api_decodes_frames_larger_than_a_batch(gpu, monkeypatch):
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", "1")
    a = z.gen_stream(z.GEN_MIX, (24 << 20) + 12345, 1 << 20, first=7)
    b = z.gen_stream(z.GEN_TEXT, (13 << 20) + 99, 1 << 20, first=8)
    small = [z.gen_stream(z.GEN_TEXT, n, 1 << 20, first=n) for n in (1000, 300000)]
    skip = np.frombuffer(bytes.fromhex("502a4d18") + (6).to_bytes(4, "little") + b"abcdef", np.uint8)
    fa = zstd_adv(a, 3, checksum=1, pieces=[a.size // 2, a.size - a.size // 2])     # the CLI's layout, no content size
    fb = zstd_adv(b, 19, checksum=1)                                                # 8 MiB window
    stream = np.concatenate([zstd1(small[0], 3), fa, skip, zstd1(small[1], 1), fb, skip, fa])
    want = np.concatenate([small[0], a, small[1], b, a])
    rc, back, st = z.decompress_mem(z.CODEC_ZSTD, stream, want.size + 16, threads=4, inputsize=1 << 20)
    assert rc == 0, z.lib().ZSTDCB_getErrorString(rc)
    assert back.size == want.size and np.array_equal(back, want)
    assert st["insize"] == stream.size and st["outsize"] == want.size


def test_callback_api_segments_a_small_frame_with_a_large_output(gpu, monkeypatch):
    """A frame far smaller than a batch whose content is more than four batches: cut by its output room (128 KiB per
    compressed block), so the output stays bounded too."""
    src = np.tile(z.gen_stream(z.GEN_TEXT, 4096, 1 << 20, first=5), 4096)             # 16 MiB of content
    fr = zstd_adv(src, 3, checksum=1)
    assert fr.size < (1 << 20) // 2
    rc, end, room, flags, last, _, _ = z.zstd_segment(fr, z.ZstdWalk(), 1 << 20, 4 << 20)
    assert rc == 0 and not last and room == 4 << 20 and end < fr.size                    # the output room ends the first segment
    small = z.gen_stream(z.GEN_MIX, 70000, 1 << 20, first=6)
    stream = np.concatenate([zstd1(small, 3), fr, zstd1(small, 1)])
    want = np.concatenate([small, src, small])
    for mb in ("1", "64"):                                   # segmented by output room / one batch, as before
        monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", mb)
        rc, back, st = z.decompress_mem(z.CODEC_ZSTD, stream, want.size + 16, threads=4, inputsize=1 << 20)
        assert rc == 0, z.lib().ZSTDCB_getErrorString(rc)
        assert np.array_equal(back, want) and st["insize"] == stream.size and st["outsize"] == want.size


def test_first_write_comes_before_the_last_read(gpu, monkeypatch):
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", "1")
    src = z.gen_stream(z.GEN_MIX, 32 << 20, 1 << 20, first=9)
    fr = zstd_adv(src, 1, checksum=1)
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
    ctx = L.ZSTDCB_createDCtx(4, 1 << 20)
    try:
        rc = L.ZSTDCB_decompressDCtx(ctx, ctypes.byref(rw))
        assert rc == 0, L.ZSTDCB_getErrorString(rc)
        assert L.ZSTDCB_GetInsizeDCtx(ctx) == fr.size and L.ZSTDCB_GetOutsizeDCtx(ctx) == src.size
    finally:
        L.ZSTDCB_freeDCtx(ctx)
    assert bytes(out) == src.tobytes()
    first_w = next(at for kind, at in events if kind == "w")
    assert first_w <= fr.size - (1 << 20), (first_w, fr.size)


# ---------------------------------------------------------------- 3. memory stays bounded (a subprocess without torch)
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
        ctx = L.ZSTDCB_createDCtx(4, 1 << 20)
        rc = L.ZSTDCB_decompressDCtx(ctx, ctypes.byref(rw))
        out = L.ZSTDCB_GetOutsizeDCtx(ctx)
        L.ZSTDCB_freeDCtx(ctx); f.close()
        return rc, out
    rc, _ = run(sys.argv[2])
    assert rc == 0, rc
    before = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    rc, out = run(sys.argv[3])
    after = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    print(rc, out, before, after)
""")


def write_zstd_stream(path, total, level=1, piece=8 << 20, pledged=False, window_log=0):
    """One zstd frame of `total` content bytes (GEN_MIX) with a content checksum, written by libzstd's streaming API in
    pieces: without a content size (what `zstd < pipe` writes), or with one when the size is pledged (what `zstd file`
    writes).  window_log: ZSTD_c_windowLog, else the level's."""
    L = ctypes.CDLL("libzstd.so.1")

    class Buf(ctypes.Structure):
        _fields_ = [("p", ctypes.c_void_p), ("size", ctypes.c_size_t), ("pos", ctypes.c_size_t)]
    L.ZSTD_createCCtx.restype = ctypes.c_void_p
    L.ZSTD_CCtx_setParameter.restype = ctypes.c_size_t; L.ZSTD_CCtx_setParameter.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    L.ZSTD_compressStream2.restype = ctypes.c_size_t
    L.ZSTD_compressStream2.argtypes = [ctypes.c_void_p, ctypes.POINTER(Buf), ctypes.POINTER(Buf), ctypes.c_int]
    L.ZSTD_freeCCtx.argtypes = [ctypes.c_void_p]
    L.ZSTD_compressBound.restype = ctypes.c_size_t; L.ZSTD_compressBound.argtypes = [ctypes.c_size_t]
    cctx = L.ZSTD_createCCtx()
    assert L.ZSTD_CCtx_setParameter(cctx, 100, level) < (1 << 62)
    assert L.ZSTD_CCtx_setParameter(cctx, 201, 1) < (1 << 62)
    if window_log:
        assert L.ZSTD_CCtx_setParameter(cctx, 101, window_log) < (1 << 62)
    if pledged:
        L.ZSTD_CCtx_setPledgedSrcSize.restype = ctypes.c_size_t; L.ZSTD_CCtx_setPledgedSrcSize.argtypes = [ctypes.c_void_p, ctypes.c_ulonglong]
        assert L.ZSTD_CCtx_setPledgedSrcSize(cctx, total) < (1 << 62)
    cap = L.ZSTD_compressBound(piece) + 1024
    dst = np.empty(cap, np.uint8)
    with open(path, "wb") as f:
        at = 0
        while True:
            k = min(piece, total - at)
            src = z.gen_stream(z.GEN_MIX, k, 1 << 20, first=at // (1 << 20)) if k else np.zeros(1, np.uint8)
            ib = Buf(src.ctypes.data, k, 0)
            end = at + k >= total
            while True:
                ob = Buf(dst.ctypes.data, cap, 0)
                r = L.ZSTD_compressStream2(cctx, ctypes.byref(ob), ctypes.byref(ib), 2 if end else 0)
                assert r < (1 << 62)
                f.write(dst[: ob.pos].tobytes())
                if (end and r == 0) or (not end and ib.pos == ib.size):
                    break
            at += k
            if end:
                break
    L.ZSTD_freeCCtx(cctx)


def test_memory_is_bounded_for_a_2gib_frame(gpu, tmp_path):
    total = 2 << 30
    big, warm = str(tmp_path / "big.zst"), str(tmp_path / "warm.zst")
    write_zstd_stream(big, total)
    write_zstd_stream(warm, 40 << 20)
    env = dict(os.environ, ZSTDMT_B200_PLAIN_MB="16")
    r = subprocess.run([sys.executable, "-c", _RSS_SCRIPT, ROOT, warm, big], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    rc, out, before, after = (int(x) for x in r.stdout.split())
    assert rc == 0 and out == total
    assert (after - before) * 1024 < (512 << 20), (before, after)      # ru_maxrss in KiB


# ---------------------------------------------------------------- 4. errors in a later segment: the whole-frame path's error
def _errors_case():
    src = z.gen_stream(z.GEN_MIX, (8 << 20) + 5, 1 << 20, first=12)
    return src, zstd_adv(src, 3, checksum=1, content_size=1)


def _decode(stream, cap, plain_mb, monkeypatch):
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", str(plain_mb))
    rc, back, _ = z.decompress_mem(z.CODEC_ZSTD, stream, cap, threads=4, inputsize=1 << 20)
    return rc, back


@pytest.mark.parametrize("damage", ["content_checksum", "block_in_third_segment", "truncated", "content_size"])
def test_errors_in_a_later_segment_match_the_whole_frame_path(gpu, damage, monkeypatch):
    src, fr = _errors_case()
    hw = header_walk(fr)
    bad = fr.copy()
    bound = None
    if damage == "content_checksum":
        bad[-1] ^= 0x01
    elif damage == "block_in_third_segment":
        _, blk, _, _ = host_scan(fr)
        # 1 MiB segments: a compressed block with sequences in the third; its bitstream loses its end mark
        b = next(i for i in range(len(blk)) if blk["comp_off"][i] > (5 << 19) and blk["type"][i] == 2 and blk["nseq"][i] > 0)
        bad[int(blk["comp_off"][b]) + int(blk["comp_size"][b]) - 1] = 0
        # at most the content of the blocks before it (128 KiB bounds a compressed block)
        bound = int(sum(int(r) if t != 2 else 128 << 10 for r, t in zip(blk["regen_hint"][:b], blk["type"][:b])))
    elif damage == "truncated":
        bad = fr[: hw["blocks"][len(hw["blocks"]) // 2][0] + 1000]
    else:
        fhd = int(fr[4]); fcs = fhd >> 6
        at = 5 + (0 if (fhd >> 5) & 1 else 1)
        n = [1, 2, 4, 8][fcs]
        assert fcs >= 2
        bad[at:at + n] = np.frombuffer(int(src.size + 1).to_bytes(n, "little"), np.uint8)
    L = z.lib()
    rc_whole, _ = _decode(bad, src.size + 64, 64, monkeypatch)
    rc_seg, out_seg = _decode(bad, src.size + 64, 1, monkeypatch)
    assert L.ZSTDCB_isError(rc_whole) and L.ZSTDCB_isError(rc_seg)
    assert L.ZSTDCB_getErrorString(rc_seg) == L.ZSTDCB_getErrorString(rc_whole), (L.ZSTDCB_getErrorString(rc_seg), L.ZSTDCB_getErrorString(rc_whole))
    # what was written before the failing segment is the frame's leading content
    assert out_seg.size > 0 and np.array_equal(out_seg, src[: out_seg.size])
    if bound is not None:
        assert out_seg.size <= bound
    if damage == "content_checksum":                          # checked on the last segment, which is not written
        assert out_seg.size < src.size and b"hecksum" in L.ZSTDCB_getErrorString(rc_seg)
