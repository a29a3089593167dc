"""The LZ4 high-compression class of levels 10-12 (lz4_hc.cuh) held byte for byte to its CPU twin (pytest -m gpu).
Every stream written by zmt_lz4_compress_level_device must equal oracle/chain_twin.c's, keep the class's frame layout
(tests/_lz4hc.py:check_structure) and be restored by zmt_lz4_decompress_device, LZ4MT_decompressDCtx, the oracle and,
when oracle/_ref exists, liblz4 (T=1 and T>1).  Inputs are built here with fixed seeds; each edge case asserts from the
parsed stream that it reached its edge."""
import ctypes

import numpy as np
import pytest

import _lz4hc as hc
import _oracle as o
import zstdmt_b200 as z

pytestmark = pytest.mark.gpu
LEVELS = hc.LEVELS


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def gpu_compress(torch, src, chunk, level, chunk_bytes=None):
    """zmt_lz4_compress_level_device.  chunk_bytes: explicit per-chunk sizes, chunk c read from src[c * chunk:]."""
    L = z.lib()
    n = int(src.size)
    if chunk_bytes is None:
        nch = L.zmt_chunk_count(n, chunk); d_cb = None
    else:
        nch = len(chunk_bytes); d_cb = torch.from_numpy(np.asarray(chunk_bytes, np.int32)).cuda()
    d_in = torch.from_numpy(src).cuda() if n else torch.empty(1, dtype=torch.uint8, device="cuda")
    work = torch.empty(L.zmt_lz4c_level_workspace_bytes(nch, chunk, level), dtype=torch.uint8, device="cuda")
    out = torch.empty(L.zmt_lz4c_out_bound(nch, chunk), dtype=torch.uint8, device="cuda")
    foff = torch.zeros(nch + 1, dtype=torch.int64, device="cuda")
    rc = L.zmt_lz4_compress_level_device(d_in.data_ptr(), n, chunk, d_cb.data_ptr() if d_cb is not None else None, nch, level,
                                         work.data_ptr(), out.data_ptr(), foff.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return out[: int(foff[-1].item())].cpu().numpy()


def gpu_decompress(torch, framed, out_sizes):
    offs, sizes = z.scan_frames(framed)
    dec = z.Lz4DeviceDecompressor(offs, sizes, out_sizes)
    out, status = dec.run(torch.from_numpy(np.ascontiguousarray(framed)).cuda())
    torch.cuda.synchronize()
    return out[: dec.out_total].cpu().numpy(), status.cpu().numpy()


def check_roundtrip(torch, framed, parts):
    content = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    n = int(content.size)
    out, status = gpu_decompress(torch, framed, [p.size for p in parts])
    assert not status.any() and np.array_equal(out, content)
    rc, out, _ = z.decompress_mem(z.CODEC_LZ4, framed, n + 16)
    assert rc == 0 and np.array_equal(out, content)
    rc, out = o.orc_decode(o.CODEC_LZ4, framed, n)
    assert rc == 0 and np.array_equal(out, content)
    # the reference's reader takes an empty frame for the end of the input (it does so on level-1 streams too), so
    # streams with an empty chunk before their last one are left to the three decoders above
    if o.have_ref() and all(p.size for p in parts[:-1]):
        for T in (1, 3):
            rc, out, _ = o.ref_decompress(o.CODEC_LZ4, framed, n, threads=T)
            assert rc == 0 and np.array_equal(out, content)


def check(torch, src, chunk, level, chunk_bytes=None):
    """GPU stream == twin stream, layout, round trips; returns (framed, parsed frames, matches into earlier blocks)."""
    framed = gpu_compress(torch, src, chunk, level, chunk_bytes)
    if chunk_bytes is None:
        parts = [src[i: i + chunk] for i in range(0, max(src.size, 1), chunk)]
        want = hc.twin_compress(src, chunk, level)
    else:
        parts = [src[c * chunk: c * chunk + int(b)] for c, b in enumerate(chunk_bytes)]
        want = np.concatenate([hc.twin_compress(p, chunk, level) for p in parts])
    assert framed.size == want.size and np.array_equal(framed, want), "the GPU stream differs from the twin's"
    back = hc.check_structure(framed, parts)
    check_roundtrip(torch, framed, parts)
    return framed, hc.parse_stream(framed), back


def match_starts(frames, chunk):
    """(absolute match start, offset, length) of every match of every frame."""
    res = []
    for fi, (_, _, blocks) in enumerate(frames):
        for k, (raw, _, seqs) in enumerate(blocks):
            p = fi * chunk + k * hc.BLOCK
            for ll, off, ml in (seqs or []):
                p += ll
                res.append((p, off, ml))
                p += ml
    return np.array(res, np.int64).reshape(-1, 3)


# ------------------------------------------------------------------------------------------------- inputs
def periodic(rng, period, n):
    return np.resize(rng.integers(0, 256, period, dtype=np.uint8), n)


def kinds_stream(rng, chunk):
    """One chunk each of text, mix, zeros, random and periods 1-4, then a tail whose last block is short."""
    parts = [z.gen_stream(z.GEN_TEXT, chunk, chunk), z.gen_stream(z.GEN_MIX, chunk, chunk, first=3), np.zeros(chunk, np.uint8),
             rng.integers(0, 256, chunk, dtype=np.uint8)]
    parts += [periodic(rng, p, chunk) for p in (1, 2, 3, 4)]
    parts.append(z.gen_stream(z.GEN_TEXT, 40000 + 1234, chunk, first=7))
    return np.concatenate(parts)


@pytest.mark.parametrize("level", LEVELS)
def test_every_kind_matches_the_twin(torch, level):
    rng = np.random.default_rng(level)
    chunk = 256 << 10
    src = kinds_stream(rng, chunk)
    framed, frames, back = check(torch, src, chunk, level)
    m = match_starts(frames, chunk)
    assert back > 0                                                    # linked blocks are used
    assert m[:, 2].max() > hc.LCAP                                     # merged matches longer than the cap of best[]
    raw = [r for _, _, blocks in frames for r, _, _ in blocks]
    assert any(raw) and not all(raw)


@pytest.mark.parametrize("level", LEVELS)
def test_chunks_that_are_not_multiples_of_64k(torch, level):
    src = np.concatenate([z.gen_stream(z.GEN_TEXT, 500000, 1 << 20), z.gen_stream(z.GEN_MIX, 400000, 1 << 20, first=9)])
    for chunk in (200000, 70001):
        check(torch, src, chunk, level)


@pytest.mark.parametrize("level", LEVELS)
def test_explicit_chunk_bytes_empty_and_tiny(torch, level):
    rng = np.random.default_rng(11)
    check(torch, np.zeros(0, np.uint8), 1 << 20, level)
    check(torch, np.array([7], np.uint8), 1 << 20, level)
    chunk = 128 << 10
    src = np.concatenate([z.gen_stream(z.GEN_TEXT, chunk, chunk), rng.integers(0, 4, chunk, dtype=np.uint8),
                          z.gen_stream(z.GEN_MIX, 5 * chunk, chunk)])
    check(torch, src, chunk, level, chunk_bytes=[chunk, 1, 0, 12, 13, 70000, chunk - 5])


@pytest.mark.parametrize("level", LEVELS)
def test_match_at_exactly_the_window(torch, level):
    """In random bytes, a 4 KiB segment recurs at exactly 65535 bytes (matched, across a block boundary) and another at
    65536 (not).  The segments are long enough for their block to shrink, so it is not stored raw."""
    W, S = hc.WINDOW, 4096
    rng = np.random.default_rng(21)
    src = rng.integers(0, 256, 2 * W + 4096, dtype=np.uint8)
    a, b = 1000, 10000
    src[a + W: a + W + S] = src[a: a + S]
    src[b + W + 1: b + W + 1 + S] = src[b: b + S]
    framed, frames, back = check(torch, src, 1 << 20, level)
    m = match_starts(frames, 1 << 20)
    assert ((m[:, 0] == a + W) & (m[:, 1] == W) & (m[:, 2] >= S)).any()
    assert not ((m[:, 0] >= b + W + 1) & (m[:, 0] < b + W + 1 + S)).any()


def test_lazy_choice_defers_a_short_match(torch):
    """At p the best match is 4 bytes long, at p + 1 it is 64: the parse emits p as a literal and takes the long one."""
    rng = np.random.default_rng(31)
    R = rng.integers(0, 256, 64, dtype=np.uint8)
    A = np.array([0xAB], np.uint8)
    junk = lambda k: rng.integers(0, 256, k, dtype=np.uint8)
    src = np.concatenate([junk(3000), R, junk(3000), A, R[:3], junk(3000), A, R, junk(3000)])
    p = 3000 + 64 + 3000 + 4 + 3000
    for level in LEVELS:
        framed, frames, _ = check(torch, src, 1 << 20, level)
        m = match_starts(frames, 1 << 20)
        assert ((m[:, 0] == p + 1) & (m[:, 2] >= 64)).any() and not (m[:, 0] == p).any()


@pytest.mark.parametrize("level", LEVELS)
def test_random_chunk_is_all_raw(torch, level):
    src = np.random.default_rng(5).integers(0, 256, (300 << 10) + 17, dtype=np.uint8)
    framed, frames, _ = check(torch, src, 1 << 20, level)
    raw = [r for _, _, blocks in frames for r, _, _ in blocks]
    assert raw and all(raw)


def test_levels_through_the_c_api_default_chunks(torch):
    """LZ4MT_compressCCtx with inputsize 0 (4 MiB chunks) at levels 10 and 12: the device path's bytes, counters as the
    reference's, restored by LZ4MT_decompressDCtx and by the reference."""
    M = z.memio_lib()
    n = (20 << 20) + 12345
    src = z.gen_stream(z.GEN_MIX, n, 1 << 20)
    cap = n + n // 64 + (1 << 20)
    for level in (10, 12):
        out = np.empty(cap, np.uint8); st = (ctypes.c_size_t * 5)()
        rc = M.zmt_lz4_compress_mem(4, level, 0, src.ctypes.data, n, out.ctypes.data, cap, st)
        assert rc == 0, z.lib().LZ4MT_getErrorString(rc)
        framed = out[: int(st[0])]
        assert np.array_equal(framed, gpu_compress(torch, src, 4 << 20, level))
        assert st[1] == -(-n // (4 << 20)) and st[2] == n and st[3] == framed.size
        back = np.empty(n + 16, np.uint8); dst = (ctypes.c_size_t * 5)()
        rc = M.zmt_lz4_decompress_mem(4, 0, framed.ctypes.data, framed.size, back.ctypes.data, n + 16, dst)
        assert rc == 0 and dst[0] == n and np.array_equal(back[:n], src)
        if o.have_ref():
            R = o.ref()
            rout = np.empty(cap, np.uint8); rst = (ctypes.c_size_t * 5)()
            assert R.ref_lz4_compress_mem(4, level, 0, src.ctypes.data, n, rout.ctypes.data, cap, rst) == 0
            assert (st[1], st[2]) == (rst[1], rst[2])                  # frames, insize
            assert (st[4] & 0xFFFFFFFF) == (rst[4] & 0xFFFFFFFF) == st[1]  # one write per frame
            for T in (1, 3):
                rc, rback, _ = o.ref_decompress(o.CODEC_LZ4, framed, n, threads=T)
                assert rc == 0 and np.array_equal(rback, src)


def test_one_call_over_all_gpus_is_byte_identical(torch, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    src = z.gen_stream(z.GEN_MIX, (40 << 20) + 77, 4 << 20)
    monkeypatch.setenv("ZSTDMT_GPUS", "0")
    rc, one, _ = z.compress_mem(z.CODEC_LZ4, src, threads=4, level=12, chunk=4 << 20)
    assert rc == 0
    monkeypatch.setenv("ZSTDMT_GPUS", "all")
    rc, allg, _ = z.compress_mem(z.CODEC_LZ4, src, threads=4, level=12, chunk=4 << 20)
    assert rc == 0 and np.array_equal(one, allg)


@pytest.mark.parametrize("kind", [z.GEN_TEXT, z.GEN_MIX])
def test_level12_ratio_over_level1(torch, kind, capsys):
    """64 MiB in 4 MiB chunks: the ratio does not fall from level 10 to 11 to 12, and level 12 beats level 1 by 10 %."""
    n, chunk = 64 << 20, 4 << 20
    src = z.gen_stream(kind, n, chunk)
    r = {lv: n / gpu_compress(torch, src, chunk, lv).size for lv in (1, 10, 11, 12)}
    with capsys.disabled():
        print("\n[ratio] %s: " % ("text" if kind == z.GEN_TEXT else "mix") + ", ".join("level %d %.4f" % kv for kv in r.items()))
    assert r[10] <= r[11] <= r[12]
    assert r[12] >= 1.10 * r[1]
