"""The device frame index for plain streams (zmt_lz4_index_plain_device, zmt_zstd_index_plain_device) against the plain
rule restated in Python and the callback API's plain path.

A plain stream is what the lz4 and zstd tools write: codec frames and skippable frames back to back, without container
headers.  For every stream the tables built on the GPU equal host-built ones: the frame offsets and lengths of a Python
walk of the stream, for LZ4 the room (content size, or the block bound) and the slots, for zstd the descriptors, first
blocks, expect, flags and scratch of zmt_zstd_scan_frame_host on each frame at base 12 + its offset.  Decoding from
them gives the source bytes, and the same bytes as the callback API on the same stream.  Rejections get the status,
frame and offset the header documents, and the callback API rejects the same streams."""
import ctypes
import json
import os

import numpy as np
import pytest

import _lz4corpus as lc
import _zcorpus as zc
import zstdmt_b200 as z
from test_gpu_frame_index import golden_cases, libzstd_frames, zstd_header_len
from test_gpu_plain_segments import write_lz4_stream_prefs
from test_gpu_plain_streams import lz4f, zstd_adv

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ST_OK, ST_TRUNC, ST_MAGIC, ST_HEADER, ST_BLOCK, ST_DST_SMALL, ST_CONTENT_SIZE, ST_UNSUP = 0, 1, 2, 3, 5, 6, 8, 10
ZF_NO_SIZE = 4
NO_EXPECT = np.uint64(0xFFFFFFFFFFFFFFFF)
SMALL = 4 << 20          # streams up to this size are placed at every device address 0..15 mod 16


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def rd(b, p, k=4):
    return int.from_bytes(b[p: p + k].tobytes(), "little")


def skippable(size, magic=0x184D2A50):
    return np.frombuffer(int(magic).to_bytes(4, "little") + int(size).to_bytes(4, "little") + bytes((7 * i + 1) & 0xFF for i in range(size)), np.uint8)


def cat(parts):
    parts = [np.asarray(p, np.uint8) for p in parts]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


# ------------------------------------------------------------------ the plain rule, restated
def lz4_walk(b, pos, end):
    """The LZ4F frame at b[pos] walked inside b[:end]: (length or None when it runs past end, block bound, stop offset)."""
    flg, bd = int(b[pos + 4]), int(b[pos + 5])
    blkmax = 1 << (8 + 2 * ((bd >> 4) & 7))
    q, bound = pos + 7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0), 0
    while True:
        if q + 4 > end:
            return None, bound, min(q, end)
        bh = rd(b, q); q += 4
        if bh == 0:
            q += 4 if flg & 4 else 0
            break
        bound += (bh & 0x7FFFFFFF) if bh >> 31 else blkmax
        q += (bh & 0x7FFFFFFF) + (4 if flg & 0x10 else 0)
    return (None, bound, end) if q > end else (q - pos, bound, None)


def zstd_walk(b, pos):
    """(length, blocks) of the well-formed zstd frame at b[pos]."""
    q, nblk = pos + zstd_header_len(b[pos: pos + 18]), 0
    while True:
        bh = rd(b, q, 3); q += 3; nblk += 1
        q += 1 if (bh >> 1) & 3 == 1 else bh >> 3
        if bh & 1:
            break
    return q + (4 if b[pos + 4] & 4 else 0) - pos, nblk


def plain_frames(b, codec):
    """[(offset, length, room, blocks)] of the codec frames of a well-formed plain stream."""
    pos, out = 0, []
    while pos < b.size:
        if rd(b, pos) & 0xFFFFFFF0 == 0x184D2A50:
            pos += 8 + rd(b, pos + 4)
            continue
        if codec == "lz4":
            n, bound, _ = lz4_walk(b, pos, b.size)
            room = rd(b, pos + 6, 8) if b[pos + 4] & 8 else bound
            out.append((pos, n, room, 0))
        else:
            n, nblk = zstd_walk(b, pos)
            out.append((pos, n, None, nblk))
        pos += n
    assert pos == b.size
    return out


def host_zstd(b, frames):
    """zmt_zstd_scan_frame_host on every frame, at base 12 + its offset: descriptors, first blocks, expect, flags, rooms, scratch."""
    L = z.lib()
    cap = sum(f[3] for f in frames) + 16
    blocks = np.zeros(cap * L.zmt_zstd_blk_desc_bytes(), np.uint8)
    nblk, scr = ctypes.c_uint32(0), ctypes.c_uint64(0)
    first, expect, flags, rooms = [], [], [], []
    for i, (off, n, _, _) in enumerate(frames):
        first.append(nblk.value)
        cs, fl = ctypes.c_uint64(0), ctypes.c_uint32(0)
        rc = L.zmt_zstd_scan_frame_host(b[off:].ctypes.data, n, 12 + off, i, blocks.ctypes.data, ctypes.byref(nblk), cap, ctypes.byref(scr),
                                        ctypes.byref(cs), ctypes.byref(fl))
        assert rc == 0, (i, rc)
        rooms.append(cs.value); flags.append(fl.value)
        expect.append(NO_EXPECT if fl.value & ZF_NO_SIZE else np.uint64(cs.value))
    first.append(nblk.value)
    return dict(blocks=blocks[: nblk.value * L.zmt_zstd_blk_desc_bytes()], first=np.array(first, np.uint32), expect=np.array(expect, np.uint64),
                flags=np.array(flags, np.uint32), rooms=rooms, scratch=scr.value)


# ------------------------------------------------------------------ device index and decode
def place(torch, b, k):
    """The stream at a device address = k mod 16."""
    buf = torch.zeros(b.size + 32, dtype=torch.uint8, device="cuda")
    if b.size:
        buf[k: k + b.size] = torch.from_numpy(np.ascontiguousarray(b)).cuda()
    assert (buf.data_ptr() + k) % 16 == k
    return buf[k: k + b.size]


def u(t, n, dt):
    return t[:n].cpu().numpy().view(dt)


def device_decode(torch, codec, d, max_frames=None):
    cls = z.Lz4DeviceDecompressor if codec == "lz4" else z.ZstdDeviceDecompressor
    dec = cls.from_device(d, max_frames=max_frames, plain=True)
    out, st = dec.run(d)
    torch.cuda.synchronize()
    n = dec.n
    assert not st.cpu().numpy()[:n].any(), st.cpu().numpy()[:n]
    oo, sz = u(dec.d_out_off, n + 1, np.int64), dec.out_size[:n].cpu().numpy()
    return dec, [out[int(oo[i]): int(oo[i]) + int(sz[i])].cpu().numpy() for i in range(n)]


def callback(codec, b, cap):
    rc, back, _ = z.decompress_mem(z.CODEC_LZ4 if codec == "lz4" else z.CODEC_ZSTD, b, cap, threads=4)
    return rc, back


def is_error(codec, rc):
    return bool(z.lib().LZ4MT_isError(rc) if codec == "lz4" else z.lib().ZSTDCB_isError(rc))


def check(torch, codec, b, srcs, aligns=None, max_frames=None, api=True):
    """Tables against the restated rule, decode against the sources and the callback API, at every address mod 16 for a
    small stream (aligns: the addresses to use)."""
    b = np.ascontiguousarray(b, np.uint8)
    frames = plain_frames(b, codec)
    n = len(frames)
    assert n == len(srcs)
    want = cat(srcs)
    h = host_zstd(b, frames) if codec == "zstd" else None
    for k in aligns if aligns is not None else (range(16) if b.size <= SMALL else (0, 13)):
        d = place(torch, b, k)
        dec, got = device_decode(torch, codec, d, max_frames)
        info = dec.index_info
        assert np.array_equal(u(dec.d_off if codec == "lz4" else dec.d_frame_off, n, np.int64), np.array([f[0] for f in frames], np.int64))
        assert np.array_equal(u(dec.d_cs if codec == "lz4" else dec.d_frame_csize, n, np.uint32), np.array([f[1] for f in frames], np.uint32))
        if codec == "lz4":
            rooms = [f[2] for f in frames]
            slots = sum(max(1, (r + 65535) // 65536) for r in rooms)
            assert (info.status, info.nframes, info.nblocks, info.out_bytes) == (0, n, slots, sum(rooms)), info
        else:
            rooms = h["rooms"]
            assert (info.status, info.nframes, info.nblocks, info.out_bytes, info.scratch_bytes) == \
                (0, n, len(h["blocks"]) // z.lib().zmt_zstd_blk_desc_bytes(), sum(rooms), h["scratch"]), info
            assert np.array_equal(dec.d_blocks[: len(h["blocks"])].cpu().numpy(), h["blocks"])
            assert np.array_equal(u(dec.d_first, n + 1, np.uint32), h["first"])
            assert np.array_equal(u(dec.d_expect, n, np.uint64), h["expect"])
            assert np.array_equal(u(dec.d_fseq, n, np.uint32), h["flags"])
            assert dec.d_frame_scratch[n].item() == h["scratch"]
        assert np.array_equal(u(dec.d_out_off, n + 1, np.int64), np.concatenate([[0], np.cumsum(np.array(rooms, np.int64))]))
        for i, s in enumerate(srcs):
            assert np.array_equal(got[i], s), (k, i)
        del d, dec
    if api and b.size:
        rc, back = callback(codec, b, want.size + 16)
        assert rc == 0 and np.array_equal(back, want)
    return frames


# ------------------------------------------------------------------ streams
@pytest.mark.parametrize("bchk", [False, True])
@pytest.mark.parametrize("lay", lc.LAYOUTS)
def test_lz4_corpus_back_to_back(torch, lay, bchk):
    """Every _lz4corpus case as one plain stream: linked and stored blocks, content sizes, checksums, block checksums
    ("short" takes the decoder's frame-sequential fallback)."""
    items = [(f, s) for n in lc.CASES for f, s, _ in lc.case(n, lay, bchk)]
    check(torch, "lz4", cat([f for f, _ in items]), [s for _, s in items])


def liblz4_frames(tmp_path):
    out = []
    for bd, size in ((4, 200000), (5, 700000), (6, 2500000), (7, 6000000)):
        for linked in (0, 1):
            for csize in (0, 1):
                src = z.gen_stream(z.GEN_MIX, size, 1 << 20)
                path = tmp_path / ("f%d%d%d.lz4" % (bd, linked, csize))
                write_lz4_stream_prefs(str(path), size, dict(blockSizeID=bd, blockMode=1 - linked, contentChecksumFlag=1, contentSize=size * csize))
                f = np.fromfile(str(path), np.uint8)
                assert bool(f[4] & 8) == bool(csize) and bool(f[4] & 0x20) != bool(linked) and (f[5] >> 4) & 7 == bd
                out.append((f, src))
    return out


def test_liblz4_streaming_frames(torch, tmp_path):
    """liblz4 streaming frames for block sizes 64 KiB..4 MiB, linked and independent, with and without a content size."""
    fr = liblz4_frames(tmp_path)
    check(torch, "lz4", cat([f for f, _ in fr]), [s for _, s in fr])
    for f, s in fr[:4]:
        check(torch, "lz4", f, [s], aligns=(0, 5))


def test_zstd_corpus_back_to_back(torch):
    cases = [zc.case(n) for n in zc.CASES]
    check(torch, "zstd", cat([f for _, f in cases]), [s for s, _ in cases])


def test_libzstd_frames(torch):
    """libzstd frames with a checksum, without a content size and at level 19."""
    fr = libzstd_frames()
    check(torch, "zstd", cat([f for _, f in fr]), [s for s, _ in fr])


def mixed_stream(codec, k=3):
    """k frames with skippable frames of sizes 0, 1, 4 and 13 (magics ...50 and ...5F) between them."""
    srcs = [z.gen_stream(z.GEN_TEXT if i % 2 else z.GEN_MIX, 300 + 700 * i, 1 << 20, first=i) for i in range(k)]
    if codec == "lz4":
        frames = [lz4f(s, blockMode=i % 2, contentSize=s.size, contentChecksumFlag=1) for i, s in enumerate(srcs)]
    else:
        frames = [zc.compress(s, {100: 3, 201: i % 2}) for i, s in enumerate(srcs)]
    skips = [skippable(0), skippable(1, 0x184D2A5F), skippable(4), skippable(13, 0x184D2A5F)]
    parts = []
    for i, f in enumerate(frames):
        parts.append(f)
        if i < k - 1:
            parts += skips[i % 2 * 2: i % 2 * 2 + 2]
    return cat(parts), frames, srcs


@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_skippable_frames(torch, codec):
    b, frames, srcs = mixed_stream(codec)
    assert all(f.size > 9 for f in frames) and b.size > sum(f.size for f in frames)
    check(torch, codec, b, srcs)
    # only skippable frames, and the empty stream: OK with 0 frames
    for s in (cat([skippable(0), skippable(13, 0x184D2A5F), skippable(1), skippable(4, 0x184D2A5F)]), np.zeros(0, np.uint8)):
        info = raw_index(torch, s, codec, 4)
        assert (info.status, info.nframes, info.bad_frame, info.bad_offset, info.out_bytes, info.nblocks) == (0, 0, 0, 0, 0, 0), info
        check(torch, codec, s, [], aligns=(0, 3), api=False)


def big_lz4(tmp_path, total):
    path = tmp_path / "big.lz4"
    write_lz4_stream_prefs(str(path), total, dict(blockSizeID=4, blockMode=0, contentChecksumFlag=1))
    piece = 8 << 20
    src = cat([z.gen_stream(z.GEN_MIX, min(piece, total - at), 1 << 20, first=at // (1 << 20)) for at in range(0, total, piece)])
    return np.fromfile(str(path), np.uint8), src


@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_one_256mib_frame(torch, codec, tmp_path):
    """liblz4 64 KiB linked blocks with a content checksum; libzstd level 3 with a checksum and no content size."""
    total = 256 << 20
    if codec == "lz4":
        f, src = big_lz4(tmp_path, total)
    else:
        src = z.gen_stream(z.GEN_MIX, total, 1 << 20)
        f = zstd_adv(src, level=3, checksum=1, content_size=0, pieces=[8 << 20] * 32)
        assert (f[4] >> 6) == 0 and f[4] & 4
    check(torch, codec, f, [src])


# ------------------------------------------------------------------ container streams read as plain ones
def container_check(torch, codec, fb):
    """A container-framed stream through both indexes: the same frames and bytes, every frame_off 12 bytes further on."""
    cls = z.Lz4DeviceDecompressor if codec == "lz4" else z.ZstdDeviceDecompressor
    d = torch.from_numpy(np.ascontiguousarray(fb)).cuda()
    a = cls.from_device(d)
    b = cls.from_device(d, plain=True)
    n = a.index_info.nframes
    assert b.index_info.status == 0 and b.index_info.nframes == n
    k = "d_off" if codec == "lz4" else "d_frame_off"
    assert np.array_equal(u(getattr(b, k), n, np.int64), u(getattr(a, k), n, np.int64) + 12)
    outs = []
    for dec in (a, b):
        out, st = dec.run(d)
        torch.cuda.synchronize()
        assert not st.cpu().numpy()[:n].any()
        oo, sz = u(dec.d_out_off, n + 1, np.int64), dec.out_size[:n].cpu().numpy()
        outs.append(cat([out[int(oo[i]): int(oo[i]) + int(sz[i])].cpu().numpy() for i in range(n)]))
    assert np.array_equal(outs[0], outs[1])
    return outs[1]


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["file"])
def test_golden_container_streams(torch, case):
    fb = np.fromfile(os.path.join(GOLD, case["file"]), dtype=np.uint8)
    got = container_check(torch, case["codec"], fb)
    assert np.array_equal(got, z.gen_stream(case["kind"], case["n"], case["chunk"], first=case["first"]))


@pytest.mark.parametrize("codec,level", [("lz4", 1), ("lz4", 12), ("zstd", 3), ("zstd", 9)])
def test_device_compressor_streams(torch, codec, level):
    chunk = 1 << 18
    for n in (0, 1, 2 * chunk + 4321):
        src = z.gen_stream(z.GEN_MIX, n, chunk)
        cls = z.Lz4DeviceCompressor if codec == "lz4" else z.ZstdDeviceCompressor
        out, foff = cls(n, chunk, level=level).run(torch.from_numpy(src).cuda())
        torch.cuda.synchronize()
        assert np.array_equal(container_check(torch, codec, out[: int(foff[-1])].cpu().numpy()), src)


# ------------------------------------------------------------------ rejections
def raw_index(torch, b, codec, max_frames):
    """One plain index call without the binding's retry: the summary struct."""
    L = z.lib()
    d = torch.from_numpy(np.ascontiguousarray(b)).cuda() if len(b) else torch.zeros(1, dtype=torch.uint8, device="cuda")
    m = max_frames
    e = lambda k, dt: torch.zeros(max(k, 1), dtype=dt, device="cuda")
    off, cs, oo, fb_, fs, ex, sq = e(m, torch.int64), e(m, torch.int32), e(m + 1, torch.int64), e(m + 1, torch.int32), e(m + 1, torch.int64), \
        e(m, torch.int64), e(m, torch.int32)
    work = torch.empty(L.zmt_index_workspace_bytes(m), dtype=torch.uint8, device="cuda")
    info = torch.zeros(40, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    if codec == "lz4":
        rc = L.zmt_lz4_index_plain_device(d.data_ptr(), len(b), m, off.data_ptr(), cs.data_ptr(), oo.data_ptr(), info.data_ptr(), work.data_ptr(), s)
    else:
        rc = L.zmt_zstd_index_plain_device(d.data_ptr(), len(b), m, off.data_ptr(), cs.data_ptr(), fb_.data_ptr(), fs.data_ptr(), ex.data_ptr(),
                                           sq.data_ptr(), oo.data_ptr(), info.data_ptr(), work.data_ptr(), s)
    assert rc == 0
    torch.cuda.synchronize()
    return z.FrameIndex.from_buffer_copy(info.cpu().numpy().tobytes())


def rejections(codec):
    """[(name, stream, status, bad_offset)]: each row of the header's status table, hit in frame 1 behind a good frame 0."""
    b, frames, _ = mixed_stream(codec, 2)
    good, second = frames
    g0 = good.size
    rows = [("short", cat([good, [0x04, 0x22, 0x4D]]), ST_TRUNC, g0),
            ("skip_past_end", cat([good, skippable(13)[:20]]), ST_TRUNC, g0),
            ("foreign_magic", cat([good, [1, 2, 3, 4, 5, 6, 7, 8, 9, 10]]), ST_MAGIC, g0)]
    if codec == "lz4":
        rows.append(("zstd_magic", cat([good, zc.compress(np.arange(40, dtype=np.uint8), {100: 3})]), ST_MAGIC, g0))
        g = second.copy(); g[4] = (g[4] & 0x3F) | 0x80
        rows.append(("version", cat([good, g]), ST_HEADER, g0))
        g = second.copy(); g[5] = 3 << 4
        rows.append(("block_size_id", cat([good, g]), ST_HEADER, g0))
        rows.append(("header_cut", cat([good, second[:6]]), ST_TRUNC, g0))
        for cut in (second.size - 1, 9, 7 + (8 if second[4] & 8 else 0) + 2):
            b = cat([good, second[:cut]])
            _, _, stop = lz4_walk(b, g0, b.size)
            rows.append(("cut%d" % cut, b, ST_TRUNC, stop))
        assert second[4] & 8
        n, bound, _ = lz4_walk(second, 0, second.size)
        g = second.copy(); g[6:14] = np.frombuffer(int(bound + 1).to_bytes(8, "little"), np.uint8)
        rows.append(("content_size", cat([good, g]), ST_CONTENT_SIZE, g0))
    else:
        g = second.copy(); g[:4] = np.frombuffer((0xFD2FB527).to_bytes(4, "little"), np.uint8)
        rows.append(("legacy_magic", cat([good, g]), ST_MAGIC, g0))
        hl = zstd_header_len(second)
        g = second.copy(); g[4] |= 0x08
        rows.append(("reserved_bit", cat([good, g]), ST_HEADER, g0))
        g = cat([second[:4], [second[4] | 0x01], [9], second[5:]])
        rows.append(("dictionary", cat([good, g]), ST_UNSUP, g0))
        g = second.copy(); g[hl] |= 0x06
        rows.append(("block_type3", cat([good, g]), ST_BLOCK, g0 + hl))
        rows.append(("block_header_cut", cat([good, second[: hl + 2]]), ST_TRUNC, g0 + hl))
        rows.append(("frame_header_cut", cat([good, second[:5]]), ST_TRUNC, g0))
    return rows


@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_each_status_row_behind_a_good_frame(torch, codec):
    for name, b, st, at in rejections(codec):
        info = raw_index(torch, b, codec, 4)
        assert (info.status, info.bad_frame, info.bad_offset, info.nframes) == (st, 1, at, 1), (name, info)
        cls = z.Lz4DeviceDecompressor if codec == "lz4" else z.ZstdDeviceDecompressor
        with pytest.raises(ValueError, match="plain stream rejected: %s in frame 1 at offset %d" % (z.ST_NAMES[st], at)):
            cls.from_device(torch.from_numpy(b).cuda(), plain=True)
        rc, _ = callback(codec, b, 1 << 20)
        assert is_error(codec, rc), name


@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_frame_of_4gib_is_unsupported(torch, codec):
    """A frame of 2^32 bytes or more behind a good one: the decode calls take a 32-bit frame length.  The frame is stored
    (LZ4) or raw (zstd) blocks of zeros, its block headers written on the device."""
    b, frames, _ = mixed_stream(codec, 1)
    g0 = b.size
    if codec == "lz4":
        head, bsz, hsz, mark = bytes([0x04, 0x22, 0x4D, 0x18, 0x60, 0x70, 0x00]), 4 << 20, 4, 0x80000000
    else:
        head, bsz, hsz, mark = bytes([0x28, 0xB5, 0x2F, 0xFD, 0x00, 0x58]), 128 << 10, 3, 0
    nblk = (1 << 32) // bsz + 1
    total = g0 + len(head) + nblk * (hsz + bsz) + 4
    d = torch.zeros(total, dtype=torch.uint8, device="cuda")
    d[:g0] = torch.from_numpy(b).cuda()
    d[g0: g0 + len(head)] = torch.tensor(list(head), dtype=torch.uint8, device="cuda")
    at = g0 + len(head) + torch.arange(nblk, device="cuda", dtype=torch.int64) * (hsz + bsz)
    bh = (bsz | mark) if codec == "lz4" else (bsz << 3)
    for i in range(hsz):
        d[at + i] = (bh >> (8 * i)) & 0xFF
    if codec == "zstd":
        d[at[-1]] = (bh | 1) & 0xFF                                           # the last block
    else:
        e = g0 + len(head) + nblk * (hsz + bsz)
        d[e: e + 4] = 0                                                       # the end mark
    d = d[: total - (4 if codec == "zstd" else 0)]
    with pytest.raises(ValueError, match="plain stream rejected: unsupported in frame 1 at offset %d" % g0):
        (z.Lz4DeviceDecompressor if codec == "lz4" else z.ZstdDeviceDecompressor).from_device(d, plain=True)
    del d
    torch.cuda.empty_cache()


def boundaries(b, codec):
    """Offsets at which a prefix of the stream ends on a frame boundary (codec or skippable)."""
    pos, out = 0, {0}
    while pos < b.size:
        if rd(b, pos) & 0xFFFFFFF0 == 0x184D2A50:
            pos += 8 + rd(b, pos + 4)
        else:
            pos += lz4_walk(b, pos, b.size)[0] if codec == "lz4" else zstd_walk(b, pos)[0]
        out.add(pos)
    return out


@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_every_prefix(torch, codec):
    """Every prefix of three frames with skippable frames between them: OK exactly at frame boundaries, TRUNCATED
    elsewhere; the callback API agrees on a sample."""
    b, _, srcs = mixed_stream(codec)
    bounds = boundaries(b, codec)
    L = z.lib()
    m = 8
    e = lambda k, dt: torch.zeros(k, dtype=dt, device="cuda")
    off, cs, oo, fb_, fs, ex, sq = e(m, torch.int64), e(m, torch.int32), e(m + 1, torch.int64), e(m + 1, torch.int32), e(m + 1, torch.int64), \
        e(m, torch.int64), e(m, torch.int32)
    work = torch.empty(L.zmt_index_workspace_bytes(m), dtype=torch.uint8, device="cuda")
    infos = torch.zeros((b.size + 1, 40), dtype=torch.uint8, device="cuda")
    d = torch.from_numpy(b).cuda()
    s = torch.cuda.current_stream().cuda_stream
    for n in range(b.size + 1):
        if codec == "lz4":
            rc = L.zmt_lz4_index_plain_device(d.data_ptr(), n, m, off.data_ptr(), cs.data_ptr(), oo.data_ptr(), infos[n].data_ptr(), work.data_ptr(), s)
        else:
            rc = L.zmt_zstd_index_plain_device(d.data_ptr(), n, m, off.data_ptr(), cs.data_ptr(), fb_.data_ptr(), fs.data_ptr(), ex.data_ptr(),
                                               sq.data_ptr(), oo.data_ptr(), infos[n].data_ptr(), work.data_ptr(), s)
        assert rc == 0
    torch.cuda.synchronize()
    allinfo = infos.cpu().numpy()
    st = [z.FrameIndex.from_buffer_copy(allinfo[n].tobytes()).status for n in range(b.size + 1)]
    assert [n for n in range(b.size + 1) if st[n] == ST_OK] == sorted(bounds)
    assert all(st[n] == ST_TRUNC for n in range(b.size + 1) if n not in bounds)
    rng = np.random.default_rng(5)
    sample = sorted(set(rng.choice(np.arange(16, b.size + 1), 24, replace=False).tolist()) | {n for n in bounds if n >= 16})
    whole = cat(srcs)
    for n in sample:
        rc, back = callback(codec, b[:n], whole.size + 16)
        if st[n] == ST_OK:
            assert rc == 0 and np.array_equal(back, whole[: back.size]), n
        else:
            assert is_error(codec, rc), n


@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_max_frames_below_the_count(torch, codec):
    b, frames, srcs = mixed_stream(codec)
    f2 = plain_frames(b, codec)[2][0]
    info = raw_index(torch, b, codec, 2)
    assert (info.status, info.nframes, info.bad_frame, info.bad_offset) == (ST_DST_SMALL, 3, 2, f2), info
    info = raw_index(torch, b, codec, 0)
    assert (info.status, info.nframes, info.bad_frame) == (ST_DST_SMALL, 3, 0), info
    dec, got = device_decode(torch, codec, torch.from_numpy(b).cuda(), max_frames=1)
    assert dec.index_info.nframes == 3 and all(np.array_equal(g, s) for g, s in zip(got, srcs))
