"""The GPU zstd decoder on the edge corpus of _zcorpus.py (frames libzstd wrote from dictated parses): offsets of 16 MiB and
more, 3-byte sequence counts, repeat offsets, inherited and RLE tables, every literal-section form, matches hundreds of
blocks back; through each of the three entropy routes, through the callback API, with content checksums, and in
batches larger than one ticket window (both decoders)."""
import numpy as np
import pytest

import _oracle as o
import _zcorpus as zc
import zstdmt_b200 as z
from test_zstd_decode_corpus import ZF_NEEDS_SEQ, expected_flags, host_scan

pytestmark = pytest.mark.gpu
CASES = list(zc.CASES)
ZMT_ST_CONTENT_CHECKSUM = 7
TICKET_WIN = 16384                                   # MX_TICKET_WIN (match_exec.cuh): frames per ticket window of the execute passes


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def header(n):
    return np.frombuffer((0x184D2A50).to_bytes(4, "little") + (4).to_bytes(4, "little") + int(n).to_bytes(4, "little"), np.uint8)


def framed(frames):
    return np.concatenate([p for f in frames for p in (header(f.size), f)])


def device_decode(torch, frames):
    """One zmt_zstd_decompress_device call over the frames: (decoder, output, per-frame status, per-frame size)."""
    fb = framed(frames)
    dec = z.ZstdDeviceDecompressor(fb)
    assert dec.scan_ok, dec.scan_status
    out, st = dec.run(torch.from_numpy(fb).cuda())
    torch.cuda.synchronize()
    return dec, out.cpu().numpy(), st.cpu().numpy()[: len(frames)], dec.out_size.cpu().numpy()[: len(frames)]


def check_outputs(out, status, sizes, srcs):
    pos = 0
    for i, s in enumerate(srcs):
        assert status[i] == 0, (i, z.ST_NAMES.get(int(status[i]), status[i]))
        assert sizes[i] == s.size, i
        assert np.array_equal(out[pos: pos + s.size], s), i
        pos += s.size


@pytest.mark.parametrize("name", CASES)
def test_gpu_decodes_each_edge_case_alone(gpu, name):
    """(a) Every case as a batch of its own: status 0, the content size, the source bit for bit.  The edge each frame
    reaches is asserted on the CPU (test_zstd_decode_corpus.py)."""
    src, frame = zc.case(name)
    _, out, st, sz = device_decode(gpu, [frame])
    check_outputs(out, st, sz, [src])


@pytest.fixture(scope="module")
def batch(gpu):
    srcs, frames = zip(*(zc.case(n) for n in CASES))
    dec, out, st, sz = device_decode(gpu, list(frames))
    return list(srcs), list(frames), dec, out, st, sz


def test_gpu_decodes_all_edge_cases_in_one_batch_through_three_routes(batch):
    """(b) All cases in one batch, so that frames of the three entropy routes decode side by side: frames the host scan
    flags (dependent-block kernel + offset resolution), self-contained frames without repeat offsets (lane and warp
    kernels), and self-contained frames with repeat offsets (flagged at run time: frame-sequential pass)."""
    srcs, frames, dec, out, st, sz = batch
    check_outputs(out, st, sz, srcs)
    fseq = dec.d_fseq.cpu().numpy()[: len(frames)]
    routes = {}
    for i, n in enumerate(CASES):
        tr = zc.trace(n)
        assert fseq[i] == expected_flags(frames[i], tr), n
        routes[n] = "dep" if fseq[i] & ZF_NEEDS_SEQ else ("runtime" if (tr.seq[:, 1] <= 3).any() else "self")
    assert routes["far"] == routes["tables"] == routes["literals"] == routes["dense"] == "dep"
    assert routes["far_predef"] == routes["reference_ultra"] == "self"
    assert routes["reps_predef"] == "runtime"


@pytest.mark.parametrize("name", CASES)
def test_gpu_callback_api_decodes_each_edge_case(gpu, name):
    """(d) ZSTDCB_decompressDCtx on every case, as a plain .zst stream and behind 12-byte headers."""
    src, frame = zc.case(name)
    for stream in (frame, framed([frame])):
        rc, back, stt = z.decompress_mem(z.CODEC_ZSTD, stream, src.size + 16, threads=4)
        assert rc == 0, z.lib().ZSTDCB_getErrorString(rc)
        assert back.size == src.size and np.array_equal(back, src)
        assert stt["outsize"] == src.size


def test_gpu_callback_api_far_offsets_in_small_plain_batches(gpu, monkeypatch):
    """(d) The far case as a plain stream read in 1 MiB batches (ZSTDMT_B200_PLAIN_MB=1): a 34 MiB frame larger than a batch."""
    monkeypatch.setenv("ZSTDMT_B200_PLAIN_MB", "1")
    src, frame = zc.case("far")
    rc, back, _ = z.decompress_mem(z.CODEC_ZSTD, frame, src.size + 16, threads=4, inputsize=1 << 16)
    assert rc == 0, z.lib().ZSTDCB_getErrorString(rc)
    assert np.array_equal(back, src)


CHK_SIZES = list(range(41)) + [63, 64, 65] + [(1 << 20) + r for r in range(32)]


def test_gpu_content_checksum_tail_lengths(gpu):
    """(e) XXH64 content checksums over every tail length: frames of 0-40, 63-65 and 1 MiB + 0..31 bytes (n < 32 and every
    length mod 32), written by libzstd with ZSTD_c_checksumFlag, are accepted; with one stored checksum bit flipped, exactly
    the damaged frames fail, with ZMT_ST_CONTENT_CHECKSUM."""
    rng = np.random.default_rng(1234)
    base = z.gen_stream(z.GEN_TEXT, (1 << 20) + 64, 1 << 20)
    srcs = [base[: n] if n > 100 else rng.integers(0, 256, n, dtype=np.uint8) for n in CHK_SIZES]
    frames = [zc.compress(s, {zc.P_LEVEL: 1, zc.P_CHECKSUM: 1}) for s in srcs]
    assert all(f[4] & 4 for f in frames)
    _, out, st, sz = device_decode(gpu, frames)
    check_outputs(out, st, sz, srcs)
    for parity in (0, 1):
        bad = [f.copy() for f in frames]
        for i in range(parity, len(bad), 2):
            bad[i][bad[i].size - 4 + (i // 8) % 4] ^= np.uint8(1 << (i % 8))
        _, out, st, sz = device_decode(gpu, bad)
        want = [ZMT_ST_CONTENT_CHECKSUM if i % 2 == parity else 0 for i in range(len(frames))]
        assert list(st) == want
        pos = 0
        for i, s in enumerate(srcs):
            if i % 2 != parity:
                assert np.array_equal(out[pos: pos + s.size], s), i
            pos += s.size


def window_kinds(blocks_per_frame):
    """The execute passes' ticket order per window of TICKET_WIN frames: block-major, unless the grid of frames x the
    window's largest block count exceeds 8 x the real blocks + 65536 — then frame-major."""
    kinds = []
    for w in range(0, len(blocks_per_frame), TICKET_WIN):
        c = np.asarray(blocks_per_frame[w: w + TICKET_WIN], np.int64)
        real, grid = int(c.sum()), int(c.size * c.max())
        kinds.append("frame" if grid > 8 * real + 65536 else "block")
    return kinds


def test_gpu_zstd_batch_of_two_ticket_windows(gpu):
    """(f) More than 16,384 frames in one call: a window of tiny frames (block-major tickets) and a window holding the
    700-block `deep` frame among tiny ones (frame-major tickets)."""
    rng = np.random.default_rng(55)
    tiny_src = [rng.integers(97, 101, int(rng.integers(1, 300)), dtype=np.uint8) for _ in range(64)]
    tiny = [zc.compress(s, {zc.P_LEVEL: 1}) for s in tiny_src]
    dsrc, dframe = zc.case("deep")
    n = TICKET_WIN + 300
    pick = [i % 64 for i in range(n)]
    frames, srcs = [tiny[k] for k in pick], [tiny_src[k] for k in pick]
    frames[TICKET_WIN + 100], srcs[TICKET_WIN + 100] = dframe, dsrc
    nblk = [len(host_scan(f)[1]) for f in tiny]
    counts = [nblk[k] for k in pick]; counts[TICKET_WIN + 100] = len(host_scan(dframe)[1])
    assert counts[TICKET_WIN + 100] >= 600
    assert window_kinds(counts) == ["block", "frame"]
    _, out, st, sz = device_decode(gpu, frames)
    check_outputs(out, st, sz, srcs)


def test_gpu_lz4_batch_of_two_ticket_windows(gpu):
    """(f) The LZ4 decoder, more than 16,384 frames in one call: a window of tiny frames (block-major) and a window holding
    a 40 MiB frame of 640 blocks among tiny ones (frame-major)."""
    torch = gpu
    tiny = 64
    a = z.gen_stream(z.GEN_MIX, (TICKET_WIN + 100) * tiny, tiny)
    big = z.gen_stream(z.GEN_TEXT, 40 << 20, 1 << 20, first=3)
    c = z.gen_stream(z.GEN_TEXT, 200 * tiny, tiny, first=9)
    fb = np.concatenate([o.orc_encode_lz4(a, tiny), o.orc_encode_lz4(big, big.size), o.orc_encode_lz4(c, tiny)])
    offs, sizes = z.scan_frames(fb)
    outs = [tiny] * (TICKET_WIN + 100) + [big.size] + [tiny] * 200
    assert len(offs) == len(outs)
    slots = [max(1, -(-s // 65536)) for s in outs]                  # the decoder's slots per frame: its block bound
    assert slots[TICKET_WIN + 100] == 640
    assert window_kinds(slots) == ["block", "frame"]
    dec = z.Lz4DeviceDecompressor(offs, sizes, outs)
    out, st = dec.run(torch.from_numpy(fb).cuda())
    torch.cuda.synchronize()
    assert int(st.abs().sum()) == 0
    assert np.array_equal(out[: dec.out_total].cpu().numpy(), np.concatenate([a, big, c]))
