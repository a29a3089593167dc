"""Range reads on the GPU (RangeReader: zmt_*_content_offsets_device, zmt_*_range_plan_device, zmt_*_range_read_device):
bytes compared with slices of the source, the plan's summary with the rule of tests/_ranges.py, and the per-range
statuses on damaged streams."""
import ctypes

import numpy as np
import pytest

import _oracle as o
import _ranges as rr
import zstdmt_b200 as z
from test_gpu_plain_index import place, plain_frames, skippable, cat
from test_gpu_plain_streams import lz4f, zstd_adv

pytestmark = pytest.mark.gpu

ST_OK, ST_BLOCK, ST_CHK, ST_UNSUP, ST_BAD_ARG = 0, 5, 7, 10, 12


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def container(frames):
    parts = []
    for f in frames:
        parts += [np.frombuffer((0x184D2A50).to_bytes(4, "little") + (4).to_bytes(4, "little") + int(f.size).to_bytes(4, "little"), np.uint8), f]
    return cat(parts)


def gpu_compress(torch, codec, level, src, chunk):
    cls = z.Lz4DeviceCompressor if codec == "lz4" else z.ZstdDeviceCompressor
    c = cls(src.size, chunk, level=level)
    d = torch.from_numpy(src.copy() if src.size else np.zeros(1, np.uint8)).cuda()
    out, off = c.run(d)
    torch.cuda.synchronize()
    return out[: int(off[c.nchunks].item())].cpu().numpy()


def frames_of(b, codec, plain):
    """The codec frames of a stream, as (offset of the frame, bytes)."""
    if plain:
        return [b[f[0]: f[0] + f[1]] for f in plain_frames(b, codec)]
    return o.mt_frames(b)


def rule(b, codec, plain):
    fr = frames_of(b, codec, plain)
    st, bad, off = rr.content_table(rr.content_sizes(fr, codec), [f.size for f in fr])
    assert st == rr.ST_OK, (st, bad)
    return fr, off


def expected(src, ranges):
    return cat([src[s: s + n] for s, n in ranges])


def read(torch, reader, ranges, on_gpu):
    t = torch.tensor(np.array(ranges, dtype=np.int64).reshape(-1, 2))
    out, dst_off, st = reader.read(t.cuda() if on_gpu else t)
    torch.cuda.synchronize()
    return out.cpu().numpy(), dst_off.cpu().numpy(), st.cpu().numpy()


def check(torch, codec, b, src, plain=False, aligns=range(16), seed=1):
    """Every range of the test set, byte for byte, at every device address in `aligns`; the summary against the rule."""
    b = np.ascontiguousarray(b, np.uint8)
    fr, off = rule(b, codec, plain)
    assert off[-1] == src.size
    rng = np.random.default_rng(seed)
    full = rr.ranges_for(off, rng, nrandom=10000, max_len=70000)
    small = rr.ranges_for(off, rng, nrandom=200, max_len=70000)
    for k in aligns:
        d = place(torch, b, k)
        R = z.RangeReader(d, codec, plain=plain)
        assert R.content_size == src.size and R.n == len(fr)
        assert np.array_equal(R.content_off.cpu().numpy(), np.array(off, np.int64))
        ranges = full if k in (0, 13) else small
        got, dst_off, st = read(torch, R, ranges, on_gpu=k % 2 == 1)
        p = rr.plan(off, ranges, [f.size for f in fr])
        assert not st.any(), np.unique(st)
        assert np.array_equal(dst_off, np.array(p["dst_off"], np.int64))
        assert np.array_equal(got, expected(src, ranges)), k
        P = R.plan
        assert (P.status, P.nsel, P.dst_bytes, P.scratch_bytes, P.npieces) == (0, len(p["sel"]), p["dst_off"][-1], p["scratch_off"][-1], p["pieces"])
        if codec == "lz4":
            assert P.packed_bytes == p["packed"]
            assert P.nunits == sum(max(1, -(-(off[f + 1] - off[f]) // 65536)) for f in p["sel"])


def pieces(src, n):
    cut = [0] + sorted(np.random.default_rng(n).choice(np.arange(1, src.size), n - 1, replace=False).tolist()) + [src.size]
    return [src[a:b] for a, b in zip(cut, cut[1:])]


ENCODERS = [("lz4", 1), ("lz4", 12), ("zstd", 3), ("zstd", 9)]


@pytest.mark.parametrize("chunk,n", [(1 << 20, (3 << 20) + 12345), (100003, (1 << 20) + 777)], ids=["1MiB", "odd"])
@pytest.mark.parametrize("codec,level", ENCODERS, ids=["%s%d" % e for e in ENCODERS])
def test_device_compressor_streams(torch, codec, level, chunk, n):
    src = z.gen_stream(z.GEN_MIX, n, 1 << 20, first=level)
    check(torch, codec, gpu_compress(torch, codec, level, src, chunk), src)


@pytest.mark.parametrize("codec,level", [("lz4", 1), ("zstd", 3)])
def test_empty_input_and_zero_size_frames_between_others(torch, codec, level):
    e = o.mt_frames(gpu_compress(torch, codec, level, np.zeros(0, np.uint8), 1 << 16))
    assert len(e) == 1
    check(torch, codec, container(e), np.zeros(0, np.uint8))
    src = z.gen_stream(z.GEN_TEXT, 300000, 1 << 20)
    fr = o.mt_frames(gpu_compress(torch, codec, level, src, 65536))
    b = container([e[0], fr[0], e[0], e[0], fr[1], fr[2], e[0], fr[3], fr[4], e[0]])
    check(torch, codec, b, src)


@pytest.mark.parametrize("plain", [False, True], ids=["container", "plain"])
@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_library_frames(torch, codec, plain):
    """liblz4 frames (linked blocks, content size, content checksum) and libzstd frames (content checksum), in a container
    or as a plain stream with skippable frames between them."""
    src = z.gen_stream(z.GEN_MIX, 700001, 1 << 20, first=3)
    ps = pieces(src, 7) + [np.zeros(0, np.uint8)]
    if codec == "lz4":
        fr = [lz4f(p, blockMode=0, contentSize=max(1, p.size), contentChecksumFlag=1, blockSizeID=4) for p in ps]
    else:
        fr = [zstd_adv(p, level=3, checksum=1, content_size=1) for p in ps]
    if plain:
        b = cat([fr[0], skippable(5)] + fr[1:4] + [skippable(0)] + fr[4:] + [skippable(3, magic=0x184D2A5F)])
    else:
        b = container(fr)
    check(torch, codec, b, src, plain=plain)


def test_workspace_and_work_follow_the_selection(torch):
    L = z.lib()
    assert L.zmt_range_workspace_bytes(1024, 4096) > L.zmt_range_workspace_bytes(1024, 0) > 0
    src = z.gen_stream(z.GEN_MIX, 64 << 16, 1 << 20)
    for codec, level in (("lz4", 1), ("zstd", 3)):
        b = gpu_compress(torch, codec, level, src, 1 << 16)
        fr, off = rule(b, codec, False)
        assert len(fr) == 64
        d = place(torch, b, 0)
        R = z.RangeReader(d, codec)
        got, _, st = read(torch, R, [(40 * 65536 + 777, 1)], on_gpu=False)
        assert st.tolist() == [0] and got.tolist() == [src[40 * 65536 + 777]]
        P = R.plan
        assert P.nsel == 1 and P.scratch_bytes == 65536
        if codec == "lz4":
            assert P.packed_bytes == 16 + (fr[40].size + 15) // 16 * 16 and P.nunits == 1
            want = ((P.packed_bytes + 255) & ~255) + L.zmt_lz4d_workspace_bytes(1, 1, P.packed_bytes)
            assert R.read_work_bytes == want
            assert R.read_work_bytes * 16 < L.zmt_lz4d_workspace_bytes(64, 64, b.size)


def test_bad_ranges_fail_alone(torch):
    src = z.gen_stream(z.GEN_MIX, 500000, 1 << 20)
    for codec, level in (("lz4", 1), ("zstd", 3)):
        d = place(torch, gpu_compress(torch, codec, level, src, 65536), 5)
        R = z.RangeReader(d, codec)
        T = src.size
        ranges = [(0, 10), (T - 1, 2), (5, -3), (T + 1, 0), (70000, 5), (T, 0), (T - 3, 3)]
        got, dst_off, st = read(torch, R, ranges, on_gpu=True)
        assert st.tolist() == [0, ST_BAD_ARG, ST_BAD_ARG, ST_BAD_ARG, 0, 0, 0]
        assert dst_off.tolist() == [0, 10, 10, 10, 10, 15, 15, 18]
        assert np.array_equal(got, cat([src[:10], src[70000:70005], src[T - 3:]]))
        assert (R.plan.status, R.plan.bad_range, R.plan.nsel) == (ST_BAD_ARG, 1, 3)


def test_frames_without_a_content_size_are_named(torch):
    a, b = z.gen_stream(z.GEN_TEXT, 90000, 1 << 20), z.gen_stream(z.GEN_MIX, 50000, 1 << 20)
    cases = [("lz4", container([lz4f(a, contentSize=1), lz4f(b, contentSize=0)]), False),
             ("lz4", cat([lz4f(a, contentSize=1), lz4f(b)]), True),
             ("zstd", container([zstd_adv(a), zstd_adv(b, content_size=0)]), False),
             ("zstd", cat([zstd_adv(a), skippable(4), zstd_adv(b, content_size=0)]), True)]
    for codec, s, plain in cases:
        d = place(torch, s, 3)
        with pytest.raises(ValueError, match="unsupported in frame 1 "):
            z.RangeReader(d, codec, plain=plain)


def lz4_break_block(frame):
    """The first block header of an LZ4F frame set to one byte over the block maximum."""
    f = frame.copy()
    h = 7 + (8 if f[4] & 8 else 0) + (4 if f[4] & 1 else 0)
    f[h: h + 4] = np.frombuffer(((1 << (8 + 2 * ((int(f[5]) >> 4) & 7))) + 1).to_bytes(4, "little"), np.uint8)
    return f


def zstd_break_block(frame):
    """The jump table of the first 4-stream compressed literals section of a zstd frame overwritten: its stream sizes
    then exceed the section."""
    f = frame.copy()
    fhd = int(f[4])
    q = 5 + (0 if fhd & 0x20 else 1) + [0, 1, 2, 4][fhd & 3] + [1 if fhd & 0x20 else 0, 2, 4, 8][fhd >> 6]
    while True:
        bh = rr.rd(f, q, 3)
        bs, typ = bh >> 3, (bh >> 1) & 3
        s = q + 3
        if typ == 2 and f[s] & 3 == 2 and (f[s] >> 2) & 3:
            lhdr = 3 + max(0, ((f[s] >> 2) & 3) - 1)
            hb = int(f[s + lhdr])
            jt = s + lhdr + 1 + (hb if hb < 128 else (hb - 127 + 1) // 2)
            f[jt: jt + 6] = 0xFF
            return f
        assert not bh & 1, "no 4-stream literals section"
        q = s + (1 if typ == 1 else bs)


def corrupt_checksum(frame):
    f = frame.copy()
    f[-1] ^= 0x5A
    return f


@pytest.mark.parametrize("damage", ["block", "checksum"])
@pytest.mark.parametrize("codec", ["lz4", "zstd"])
def test_damage_reaches_exactly_the_ranges_that_touch_it(torch, codec, damage):
    src = z.gen_stream(z.GEN_MIX, 6 * 65536 + 1000, 1 << 20, first=9)
    if codec == "zstd" and damage == "checksum":
        fr = [zstd_adv(src[i: i + 65536], level=3, checksum=1) for i in range(0, src.size, 65536)]
    else:
        fr = o.mt_frames(gpu_compress(torch, codec, 1 if codec == "lz4" else 3, src, 65536))
    k = 2
    bad = (lz4_break_block if codec == "lz4" else zstd_break_block)(fr[k]) if damage == "block" else corrupt_checksum(fr[k])
    b = container(fr[:k] + [bad] + fr[k + 1:])
    off = [min(i * 65536, src.size) for i in range(len(fr))] + [src.size]
    R = z.RangeReader(place(torch, b, 7), codec)
    ranges = [(off[f] + 11, 5) for f in range(len(fr))] + [(off[k] - 1, 2), (off[k + 1] - 1, 2), (off[1], off[4] - off[1]), (0, off[k]),
                                                            (off[k + 1], src.size - off[k + 1]), (off[k] + 100, 0)]
    got, dst_off, st = read(torch, R, ranges, on_gpu=False)
    touch = [n > 0 and s < off[k + 1] and s + n > off[k] for s, n in ranges]
    want = ST_BLOCK if damage == "block" else ST_CHK
    assert st.tolist() == [want if t else 0 for t in touch]
    assert R.plan.nsel == len(fr)
    for (s, n), t, a, e in zip(ranges, touch, dst_off[:-1], dst_off[1:]):
        if not t:
            assert np.array_equal(got[a:e], src[s: s + n]), (s, n)
    # the same damage in a frame no range touches: every range OK, and frame k is not decoded
    far = [(s, n) for (s, n), t in zip(ranges, touch) if not t]
    got, _, st = read(torch, R, far, on_gpu=True)
    assert not st.any() and np.array_equal(got, expected(src, far))
    assert R.plan.nsel == len(fr) - 1


def test_reader_over_growing_batches(torch):
    src = z.gen_stream(z.GEN_TEXT, (2 << 20) + 99, 1 << 20)
    for codec, level in (("lz4", 1), ("zstd", 3)):
        R = z.RangeReader(place(torch, gpu_compress(torch, codec, level, src, 1 << 18), 0), codec)
        rng = np.random.default_rng(level)
        for i, m in enumerate((1, 16, 256, 4096, 16)):
            st_ = rng.integers(0, src.size, size=m)
            ln = np.minimum(rng.integers(0, 5000 * (i + 1), size=m), src.size - st_)
            ranges = list(zip(st_.tolist(), ln.tolist()))
            got, dst_off, st = read(torch, R, ranges, on_gpu=i % 2 == 0)
            assert not st.any() and np.array_equal(got, expected(src, ranges))
            assert dst_off.tolist() == [0] + np.cumsum(ln).tolist()
