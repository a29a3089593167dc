"""The device frame index (zmt_lz4_index_device, zmt_zstd_index_device, zmt_zstd_blocks_device) against the host walkers.

For every stream the tables built on the GPU equal the ones the host builds from the same bytes: for LZ4 the frame
offsets and sizes of scan_frames, the room each LZ4F header gives and the block-table slots; for zstd the block
descriptors, first blocks, flags, scratch and content sizes of zmt_zstd_scan_frame_host, with expect = ~0 for a frame
without a content size.  Decoding from device-built tables restores every source; malformed streams get the status,
frame and offset the header documents."""
import ctypes
import json
import os

import numpy as np
import pytest

import _lz4corpus as lc
import _oracle as o
import _zcorpus as zc
import zstdmt_b200 as z

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ST_OK, ST_TRUNC, ST_MAGIC, ST_HEADER, ST_BLOCK, ST_DST_SMALL, ST_TRAILING, ST_UNSUP = 0, 1, 2, 3, 5, 6, 9, 10
ZF_NO_SIZE = 4
P_CONTENT_SIZE, P_CHECKSUM, P_LEVEL = 200, 201, 100
NO_EXPECT = np.uint64(0xFFFFFFFFFFFFFFFF)


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def header(n, magic=0x184D2A50, four=4):
    return np.frombuffer(int(magic).to_bytes(4, "little") + int(four).to_bytes(4, "little") + int(n).to_bytes(4, "little"), np.uint8)


def framed(frames):
    parts = [p for f in frames for p in (header(len(f)), np.asarray(f, np.uint8))]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


# ------------------------------------------------------------------ host-built tables
def lz4_room(p):
    """lz4f_out_size restated: (ok, room) of one payload."""
    n = p.size
    if n < 7 or int.from_bytes(p[:4].tobytes(), "little") != 0x184D2204:
        return True, 0
    flg, bd = int(p[4]), int(p[5])
    if flg & 8:
        if n < 15:
            return False, 0
        v = int.from_bytes(p[6:14].tobytes(), "little")
        return (False, 0) if v > n * 255 + 65536 else (True, v)
    if (bd >> 4) & 7 < 4:
        return False, 0
    blkmax = 1 << (8 + 2 * ((bd >> 4) & 7))
    q, bound = 4 + 2 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0) + 1, 0
    while q + 4 <= n:
        bh = int.from_bytes(p[q: q + 4].tobytes(), "little"); q += 4
        if bh == 0:
            break
        bound += (bh & 0x7FFFFFFF) if bh & 0x80000000 else blkmax
        q += (bh & 0x7FFFFFFF) + (4 if flg & 0x10 else 0)
    return True, bound


def host_lz4(fb):
    offs, sizes = z.scan_frames(fb)
    rooms = []
    for off, cs in zip(offs, sizes):
        ok, r = lz4_room(fb[int(off) + 12: int(off) + 12 + int(cs)])
        assert ok
        rooms.append(r)
    rooms = np.array(rooms, np.int64)
    out_off = np.concatenate([[0], np.cumsum(rooms)]).astype(np.int64)
    slots = int(np.maximum(1, (rooms + 65535) // 65536).sum())
    return offs.astype(np.int64), sizes.astype(np.int64), out_off, slots


def host_zstd(fb):
    """What the host pipeline builds for a framed zstd stream: descriptors, first block, expect, flags, output offsets, scratch."""
    L = z.lib()
    offs, sizes = z.scan_frames(fb)
    n, dsz = len(offs), L.zmt_zstd_blk_desc_bytes()
    cap = fb.size // 3 + n + 16
    blocks = np.zeros(cap * dsz, np.uint8)
    nblk, scr = ctypes.c_uint32(0), ctypes.c_uint64(0)
    first, expect, flags, sizes_out = [], [], [], []
    for i in range(n):
        first.append(nblk.value)
        cs, fl = ctypes.c_uint64(0), ctypes.c_uint32(0)
        rc = L.zmt_zstd_scan_frame_host(fb[int(offs[i]) + 12:].ctypes.data, int(sizes[i]), int(offs[i]) + 12, i, blocks.ctypes.data,
                                        ctypes.byref(nblk), cap, ctypes.byref(scr), ctypes.byref(cs), ctypes.byref(fl))
        assert rc == 0, (i, rc)
        sizes_out.append(cs.value); flags.append(fl.value)
        expect.append(NO_EXPECT if fl.value & ZF_NO_SIZE else np.uint64(cs.value))
    first.append(nblk.value)
    out_off = np.concatenate([[0], np.cumsum(np.array(sizes_out, np.uint64))]).astype(np.uint64)
    return dict(blocks=blocks[: nblk.value * dsz], first=np.array(first, np.uint32), expect=np.array(expect, np.uint64),
                flags=np.array(flags, np.uint32), out_off=out_off, scratch=scr.value, frame_off=offs, frame_csize=sizes)


def u(t, n, dt):
    return t[:n].cpu().numpy().view(dt)


def check_lz4(torch, fb, srcs=None, max_frames=None):
    d = torch.from_numpy(np.ascontiguousarray(fb)).cuda()
    dec = z.Lz4DeviceDecompressor.from_device(d, max_frames=max_frames)
    offs, sizes, out_off, slots = host_lz4(fb)
    n, info = len(offs), dec.index_info
    assert (info.status, info.nframes, info.nblocks, info.out_bytes) == (0, n, slots, int(out_off[-1]))
    assert np.array_equal(u(dec.d_off, n, np.int64), offs) and np.array_equal(u(dec.d_cs, n, np.int32), sizes.astype(np.int32))
    assert np.array_equal(u(dec.d_out_off, n + 1, np.int64), out_off)
    if srcs is not None:
        out, st = dec.run(d)
        torch.cuda.synchronize()
        assert not st.cpu().numpy()[:n].any(), st.cpu().numpy()[:n]
        want = np.concatenate(srcs) if len(srcs) else np.zeros(0, np.uint8)
        assert int(dec.out_size[:n].sum()) == want.size if n else True
        got = np.concatenate([out[int(out_off[i]): int(out_off[i]) + srcs[i].size].cpu().numpy() for i in range(n)]) if n else want
        assert np.array_equal(got, want)
    return dec


def check_zstd(torch, fb, srcs=None, max_frames=None):
    d = torch.from_numpy(np.ascontiguousarray(fb)).cuda()
    dec = z.ZstdDeviceDecompressor.from_device(d, max_frames=max_frames)
    h = host_zstd(fb)
    n, info = len(h["frame_off"]), dec.index_info
    assert (info.status, info.nframes, info.nblocks, info.out_bytes, info.scratch_bytes) == \
        (0, n, len(h["blocks"]) // 64, int(h["out_off"][-1]), h["scratch"])
    assert np.array_equal(dec.d_blocks[: len(h["blocks"])].cpu().numpy(), h["blocks"])
    assert np.array_equal(u(dec.d_first, n + 1, np.uint32), h["first"])
    assert np.array_equal(u(dec.d_expect, n, np.uint64), h["expect"])
    assert np.array_equal(u(dec.d_fseq, n, np.uint32), h["flags"])
    assert np.array_equal(u(dec.d_out_off, n + 1, np.uint64), h["out_off"])
    assert dec.d_frame_scratch[n].item() == h["scratch"]
    if srcs is not None:
        out, st = dec.run(d)
        torch.cuda.synchronize()
        assert not st.cpu().numpy()[:n].any(), st.cpu().numpy()[:n]
        oo = h["out_off"].astype(np.int64)
        for i, s in enumerate(srcs):
            assert int(dec.out_size[i]) == s.size, i
            assert np.array_equal(out[oo[i]: oo[i] + s.size].cpu().numpy(), s), i
    return dec


def raw_index(torch, fb, codec, max_frames):
    """One index call without the binding's retry: the summary struct."""
    L = z.lib()
    d = torch.from_numpy(np.ascontiguousarray(fb)).cuda() if len(fb) else torch.zeros(1, dtype=torch.uint8, device="cuda")
    m = max_frames
    e = lambda k, dt: torch.zeros(max(k, 1), dtype=dt, device="cuda")
    off, cs, oo, fb_, fs, ex, sq = e(m, torch.int64), e(m, torch.int32), e(m + 1, torch.int64), e(m + 1, torch.int32), e(m + 1, torch.int64), \
        e(m, torch.int64), e(m, torch.int32)
    work = torch.empty(L.zmt_index_workspace_bytes(m), dtype=torch.uint8, device="cuda")
    info = torch.zeros(40, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    if codec == "lz4":
        rc = L.zmt_lz4_index_device(d.data_ptr(), len(fb), m, off.data_ptr(), cs.data_ptr(), oo.data_ptr(), info.data_ptr(), work.data_ptr(), s)
    else:
        rc = L.zmt_zstd_index_device(d.data_ptr(), len(fb), m, off.data_ptr(), cs.data_ptr(), fb_.data_ptr(), fs.data_ptr(), ex.data_ptr(),
                                     sq.data_ptr(), oo.data_ptr(), info.data_ptr(), work.data_ptr(), s)
    assert rc == 0
    torch.cuda.synchronize()
    return z.FrameIndex.from_buffer_copy(info.cpu().numpy().tobytes())


# ------------------------------------------------------------------ table parity and decode
def golden_cases():
    with open(os.path.join(GOLD, "manifest.json")) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["file"])
def test_golden_streams(torch, case):
    fb = np.fromfile(os.path.join(GOLD, case["file"]), dtype=np.uint8)
    src = z.gen_stream(case["kind"], case["n"], case["chunk"], first=case["first"])
    offs, _ = z.scan_frames(fb)
    srcs = [src[i * case["chunk"]: (i + 1) * case["chunk"]] for i in range(len(offs))]
    (check_lz4 if case["codec"] == "lz4" else check_zstd)(torch, fb, srcs)


KINDS = {"text": z.GEN_TEXT, "mix": z.GEN_MIX, "zeros": z.GEN_ZEROS, "random": z.GEN_RANDOM}
ENCODERS = [("lz4", 1), ("lz4", 10), ("lz4", 12), ("zstd", 1), ("zstd", 3), ("zstd", 9), ("zstd", 12)]
CHUNK = 1 << 18


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("codec,level", ENCODERS, ids=["%s%d" % e for e in ENCODERS])
def test_device_compressor_streams(torch, codec, level, kind):
    """Device compressor output at 0 bytes, 1 byte, two whole chunks and a short last chunk."""
    for n in (0, 1, 2 * CHUNK, 2 * CHUNK + 4321):
        src = z.gen_stream(KINDS[kind], n, CHUNK)
        cls = z.Lz4DeviceCompressor if codec == "lz4" else z.ZstdDeviceCompressor
        out, foff = cls(n, CHUNK, level=level).run(torch.from_numpy(src).cuda())
        torch.cuda.synchronize()
        fb = out[: int(foff[-1])].cpu().numpy()
        srcs = [src[i: i + CHUNK] for i in range(0, max(n, 1), CHUNK)]
        (check_lz4 if codec == "lz4" else check_zstd)(torch, fb, srcs)


@pytest.mark.parametrize("bchk", [False, True])
@pytest.mark.parametrize("lay", lc.LAYOUTS)
def test_lz4_edge_corpus(torch, lay, bchk):
    """Every _lz4corpus case in one stream: linked blocks, stored blocks, content sizes and checksums, block checksums."""
    items = [(f, s) for n in lc.CASES for f, s, _ in lc.case(n, lay, bchk)]
    check_lz4(torch, framed([f for f, _ in items]), [s for _, s in items])


def test_zstd_edge_corpus(torch):
    """Every _zcorpus case in one stream (described and repeated tables, treeless literals, far offsets), and each alone."""
    cases = [zc.case(n) for n in zc.CASES]
    check_zstd(torch, framed([f for _, f in cases]), [s for s, _ in cases])
    for s, f in cases:
        check_zstd(torch, framed([f]), [s])


def libzstd_frames():
    """libzstd frames with a content checksum and without a content size, of 0 bytes to several 128 KiB blocks."""
    out = []
    for i, n in enumerate((0, 1, 1000, 131072, 131073, 400000)):
        src = z.gen_stream(z.GEN_MIX if i % 2 else z.GEN_TEXT, n, 1 << 20, first=i)
        for params in ({P_LEVEL: 3, P_CHECKSUM: 1}, {P_LEVEL: 3, P_CONTENT_SIZE: 0}, {P_LEVEL: 19, P_CHECKSUM: 1, P_CONTENT_SIZE: 0}):
            out.append((src, zc.compress(src, params)))
    return out


def test_libzstd_frames_with_checksums_and_without_content_size(torch):
    fr = libzstd_frames()
    dec = check_zstd(torch, framed([f for _, f in fr]), [s for s, _ in fr])
    assert (dec.d_expect[: len(fr)].cpu().numpy().view(np.uint64) == NO_EXPECT).sum() == 12


@pytest.mark.skipif(not o.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_reference_written_streams(torch, codec):
    n, chunk = (3 << 20) + 777, 1 << 20
    src = z.gen_stream(z.GEN_MIX, n, chunk)
    for level in (1, 3, 9):
        rc, fb, _ = o.ref_compress(o.CODEC_LZ4 if codec == "lz4" else o.CODEC_ZSTD, src, threads=2, level=level, chunk=chunk)
        assert rc == 0
        srcs = [src[i: i + chunk] for i in range(0, n, chunk)]
        (check_lz4 if codec == "lz4" else check_zstd)(torch, fb, srcs)


# ------------------------------------------------------------------ round trip, damage, scale
def test_device_round_trip_copies_only_the_summary(torch):
    """Device compress -> device index -> device decode: the only device-to-host copy is the 40-byte summary, nothing goes
    to the device from the host.  The stream's length comes from a first run of the same (deterministic) compression."""
    from torch.profiler import ProfilerActivity, profile
    n, chunk = (4 << 20) + 99, 1 << 20
    d_src = torch.from_numpy(z.gen_stream(z.GEN_TEXT, n, chunk)).cuda()
    for codec in ("lz4", "zstd"):
        comp = z.Lz4DeviceCompressor(n, chunk) if codec == "lz4" else z.ZstdDeviceCompressor(n, chunk)
        dcls = z.Lz4DeviceDecompressor if codec == "lz4" else z.ZstdDeviceDecompressor
        out, foff = comp.run(d_src)
        total = int(foff[-1])
        dcls.from_device(out[:total], max_frames=8).run(out[:total])     # warm-up: module loads, constant tables
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out, _ = comp.run(d_src)
            dec = dcls.from_device(out[:total], max_frames=5)
            dout, st = dec.run(out[:total])
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        assert sum("Memcpy DtoH" in x for x in names) == 1, (codec, [x for x in names if "Memcpy" in x])
        assert sum("Memcpy HtoD" in x for x in names) == 0, codec
        assert dec.index_info.nframes == 5 and not st.cpu().numpy()[:5].any()
        assert torch.equal(dout[:n], d_src)


def test_damaged_payload_gives_the_same_statuses_through_both_table_sources(torch):
    n, chunk = (3 << 20) + 5, 1 << 20
    src = z.gen_stream(z.GEN_MIX, n, chunk)
    for codec in ("lz4", "zstd"):
        comp = z.Lz4DeviceCompressor(n, chunk) if codec == "lz4" else z.ZstdDeviceCompressor(n, chunk)
        out, foff = comp.run(torch.from_numpy(src).cuda())
        fb = out[: int(foff[-1])].cpu().numpy().copy()
        offs, sizes = z.scan_frames(fb)
        if codec == "lz4":
            pos = int(offs[1]) + 12 + 15 + 4 + 200                          # inside frame 1's first block (header 15 bytes, block header 4)
        else:
            from test_zstd_decode_corpus import ZBLK
            blk = host_zstd(fb)["blocks"].view(ZBLK)
            b = blk[(blk["frame"] == 1) & (blk["type"] == 2) & (blk["nseq"] > 0)][3]
            pos = int(b["comp_off"]) + int(b["comp_size"]) - 1               # the last byte of a sequence bitstream: its end marker
        fb[pos] = 0 if codec == "zstd" else fb[pos] ^ 0x5A
        d = torch.from_numpy(fb).cuda()
        if codec == "lz4":
            rooms = host_lz4(fb)[2]
            host = z.Lz4DeviceDecompressor(offs, sizes, np.diff(rooms))
        else:
            host = z.ZstdDeviceDecompressor(fb)
        dev = type(host).from_device(d)
        _, st_h = host.run(d)
        _, st_d = dev.run(d)
        torch.cuda.synchronize()
        a, b_ = st_h.cpu().numpy()[: len(offs)], st_d.cpu().numpy()[: len(offs)]
        assert np.array_equal(a, b_) and a[1] != 0 and not a[[0, 2, 3]].any(), (codec, a, b_)


def tiny_lz4_stream(nframes):
    src = z.gen_stream(z.GEN_TEXT, 16 * nframes, 16)
    return o.orc_encode_lz4(src, 16), [src[i: i + 16] for i in range(0, src.size, 16)]


def test_scale_fifty_thousand_frames(torch):
    """More frames than one CTA covers in every pass, and more than a first attempt of 1000 frames (retried at the exact count)."""
    nf = 50021
    fb, srcs = tiny_lz4_stream(nf)
    for m in (None, 1000):
        dec = check_lz4(torch, fb, srcs, max_frames=m)
        assert dec.index_info.nframes == nf
    # one pool frame has no content size: zeros, an RLE block whose bound is its size
    pool = [(s, zc.compress(s, {P_LEVEL: 3, P_CHECKSUM: i % 2, P_CONTENT_SIZE: int(i != 0)}))
            for i, s in enumerate([np.zeros(40, np.uint8)] + list(z.gen_stream(z.GEN_TEXT, 6 * 40, 40).reshape(6, 40)))]
    items = [pool[i % 7] for i in range(nf)] + [(np.zeros(0, np.uint8), zc.compress(np.zeros(0, np.uint8), {P_LEVEL: 3}))]
    for m in (None, 1000):
        dec = check_zstd(torch, framed([f for _, f in items]), [s for s, _ in items], max_frames=m)
        assert dec.index_info.nframes == nf + 1


def test_no_content_size_frame_decodes_through_the_host_built_tables(torch):
    """A frame without a content size that decodes to less than its block bound: ZstdDeviceDecompressor passes ~0 as its
    expected size, as the host pipeline does, so the decoder does not report a content-size mismatch."""
    src = z.gen_stream(z.GEN_TEXT, 300000, 1 << 20)
    fb = framed([zc.compress(src, {P_LEVEL: 3, P_CONTENT_SIZE: 0})])
    dec = z.ZstdDeviceDecompressor(fb)
    assert dec.out_total > src.size
    out, st = dec.run(torch.from_numpy(fb).cuda())
    torch.cuda.synchronize()
    assert st.cpu().numpy()[0] == 0 and int(dec.out_size[0]) == src.size
    assert np.array_equal(out[: src.size].cpu().numpy(), src)


# ------------------------------------------------------------------ malformed streams
def lz4_frames(k=3):
    fb, _ = tiny_lz4_stream(k)
    offs, sizes = z.scan_frames(fb)
    return [fb[int(a) + 12: int(a) + 12 + int(c)] for a, c in zip(offs, sizes)]


def assert_info(info, status, bad_frame, bad_offset, nframes=None):
    assert (info.status, info.bad_frame, info.bad_offset) == (status, bad_frame, bad_offset), info
    if nframes is not None:
        assert info.nframes == nframes, info


@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_malformed_container(torch, codec):
    frames = lz4_frames() if codec == "lz4" else [zc.compress(np.arange(50, dtype=np.uint8), {P_LEVEL: 3})] * 3
    fb = framed(frames)
    off2 = 2 * (12 + frames[0].size)
    for bad in (header(frames[2].size, magic=0x184D2A51), header(frames[2].size, four=5)):
        g = fb.copy(); g[off2: off2 + 12] = bad
        assert_info(raw_index(torch, g, codec, 8), ST_MAGIC, 2, off2, 2)
    assert_info(raw_index(torch, np.concatenate([fb, header(0)[:5]]), codec, 8), ST_TRUNC, 3, fb.size, 3)
    g = fb.copy(); g[off2 + 8: off2 + 12] = header(frames[2].size + 1)[8:]
    assert_info(raw_index(torch, g, codec, 8), ST_TRUNC, 2, off2, 2)
    assert_info(raw_index(torch, fb, codec, 2), ST_DST_SMALL, 2, off2, 3)
    assert_info(raw_index(torch, np.concatenate([fb, fb]), codec, 2), ST_DST_SMALL, 2, off2, 6)
    assert_info(raw_index(torch, np.zeros(0, np.uint8), codec, 4), ST_OK, 0, 0, 0)
    # the first failure in stream order: a bad frame before a bad container header
    g = np.concatenate([framed([frames[0], np.zeros(20, np.uint8) if codec == "zstd" else frames[1]]), header(0, magic=7)])
    info = raw_index(torch, g, codec, 8)
    assert (info.status, info.bad_frame) == ((ST_MAGIC, 1) if codec == "zstd" else (ST_MAGIC, 2))
    d = torch.from_numpy(g).cuda()
    with pytest.raises(ValueError, match="bad_magic in frame"):
        (z.Lz4DeviceDecompressor if codec == "lz4" else z.ZstdDeviceDecompressor).from_device(d)


def test_malformed_lz4_headers(torch):
    f = lz4_frames(2)
    base = 12 + f[0].size
    # no content-size field and a block size id below 4
    g = f[1].copy(); g[4] &= ~0x08 & 0xFF; g[5] = 3 << 4
    assert_info(raw_index(torch, framed([f[0], g]), "lz4", 4), ST_HEADER, 1, base + 12)
    # a content size above 255 x payload + 65536, and one just at it
    big = np.concatenate([np.frombuffer(bytes([0x04, 0x22, 0x4D, 0x18, 0x6C, 0x40]), np.uint8), np.zeros(9, np.uint8), np.zeros(20, np.uint8)])
    for v, st in ((35 * 255 + 65537, ST_HEADER), (35 * 255 + 65536, ST_OK)):
        h = big.copy(); h[6:14] = np.frombuffer(int(v).to_bytes(8, "little"), np.uint8)
        info = raw_index(torch, framed([f[0], h]), "lz4", 4)
        assert info.status == st
        if st == ST_HEADER:
            assert_info(info, ST_HEADER, 1, base + 12)
        else:
            assert info.out_bytes == 16 + v
    # a content-size flag with fewer than 15 bytes of payload
    assert_info(raw_index(torch, framed([f[0], big[:14]]), "lz4", 4), ST_HEADER, 1, base + 12)
    # a payload without the LZ4F magic: room 0, the index is fine, the decoder reports bad_magic for that frame
    junk = np.full(30, 7, np.uint8)
    fb = framed([f[0], junk, f[1]])
    d = torch.from_numpy(fb).cuda()
    dec = z.Lz4DeviceDecompressor.from_device(d)
    assert dec.index_info.status == 0 and dec.d_out_off[:4].cpu().tolist() == [0, 16, 16, 32]
    _, st = dec.run(d)
    torch.cuda.synchronize()
    assert st.cpu().tolist()[:3] == [0, ST_MAGIC, 0]


def zstd_header_len(f):
    fhd = int(f[4]); single = (fhd >> 5) & 1; fcs = fhd >> 6
    return 5 + (0 if single else 1) + [0, 1, 2, 4][fhd & 3] + ([1 if single else 0, 2, 4, 8][fcs])


def test_malformed_zstd_frames(torch):
    """Each failure of the frame walk, at frame 1 of three, against zmt_zstd_scan_frame_host on the same frame."""
    from test_zstd_decode_corpus import host_scan
    good = zc.compress(z.gen_stream(z.GEN_TEXT, 5000, 1 << 20), {P_LEVEL: 3})
    hl = zstd_header_len(good)
    cases = []
    g = good.copy(); g[0] ^= 1; cases.append((g, 0))                                  # bad magic
    g = good.copy(); g[4] |= 0x08; cases.append((g, 0))                               # reserved FHD bit
    g = np.concatenate([good[:4], [good[4] | 0x01], [9], good[5:]]).astype(np.uint8)   # a one-byte dictionary ID
    cases.append((g, 0))
    g = good.copy(); g[hl] |= 0x06; cases.append((g, hl))                             # block type 3
    cases.append((good[: hl + 2], hl))                                                # cut inside the first block header
    cases.append((np.concatenate([good, [0]]).astype(np.uint8), good.size))            # a byte behind the frame
    want = [ST_MAGIC, ST_HEADER, ST_UNSUP, ST_BLOCK, ST_TRUNC, ST_TRAILING]
    for (g, at), st in zip(cases, want):
        assert host_scan(g)[0] == st
        fb = framed([good, g, good])
        off1 = 12 + good.size
        assert_info(raw_index(torch, fb, "zstd", 4), st, 1, off1 + 12 + at, 3)
        d = torch.from_numpy(fb).cuda()
        with pytest.raises(ValueError, match="%s in frame 1 at offset %d" % (z.ST_NAMES[st], off1 + 12 + at)):
            z.ZstdDeviceDecompressor.from_device(d)
