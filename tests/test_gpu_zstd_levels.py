"""The zstd search class of levels 6-12 (zstd_lazy.cuh) held block by block to its rule (pytest -m gpu).  Every frame
written by zmt_zstd_compress_level_device is traced by the oracle (orc_zstd_trace) and checked:
  - every compressed block's sequences equal the CPU twin's (oracle/chain_twin.c) for that block, offsets explicit;
  - blocks are raw or compressed, 16 KiB (the chunk's last one may be short), predefined modes, own Huffman tree;
  - the Huffman lengths are _zenc.huf_lengths of the block's literal histogram;
  - the framed stream equals _zenc.framed_b200 byte for byte (the entropy stage's CPU twin on the twin's parse), so
    every raw block is raw for the twin's reason;
  - the oracle, libzstd (T=1 and T>1, when oracle/_ref exists) and the GPU decoder restore the frames.
Inputs are built here with fixed seeds; each edge case asserts from the trace that it reached its edge."""
import ctypes

import numpy as np
import pytest

import _oracle as o
import _zenc as ze
import _zlazy as zl
import zstdmt_b200 as z
from test_gpu_zstd_encoder import check_huffman, check_modes, check_roundtrip

pytestmark = pytest.mark.gpu
ZT = o.ZT
LEVELS = [6, 9, 12, 19]


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def gpu_compress(torch, src, chunk, level, chunk_bytes=None):
    """zmt_zstd_compress_level_device.  chunk_bytes: explicit per-chunk sizes, chunk c read from src[c * chunk:]."""
    L = z.lib()
    n = int(src.size)
    if chunk_bytes is None:
        nch = L.zmt_chunk_count(n, chunk); d_cb = None
    else:
        nch = len(chunk_bytes); d_cb = torch.from_numpy(np.asarray(chunk_bytes, np.int32)).cuda()
    d_in = torch.from_numpy(src).cuda() if n else torch.empty(1, dtype=torch.uint8, device="cuda")
    work = torch.empty(L.zmt_zstdc_level_workspace_bytes(nch, chunk, level), dtype=torch.uint8, device="cuda")
    out = torch.empty(L.zmt_zstdc_out_bound(nch, chunk), dtype=torch.uint8, device="cuda")
    foff = torch.zeros(nch + 1, dtype=torch.int64, device="cuda")
    rc = L.zmt_zstd_compress_level_device(d_in.data_ptr(), n, chunk, d_cb.data_ptr() if d_cb is not None else None, nch, level,
                                          work.data_ptr(), out.data_ptr(), foff.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return out[: int(foff[-1].item())].cpu().numpy()


class Report:
    def __init__(self):
        self.seqs = []                   # (frame, block start in the frame, traced (ll, off, ml) rows) of every compressed block
        self.types = []
        self.huf = 0
        self.raw_by = {}                 # raw blocks by reason, from the twin's traces (_zenc.raw_counts)

    @property
    def raw_bitbuf(self):
        return self.raw_by.get("bitbuf", 0)

    def all_seqs(self):
        return np.concatenate([s for _, _, s in self.seqs]) if self.seqs else np.zeros((0, 3), np.int64)


def check(torch, src, chunk, level, chunk_bytes=None):
    framed = gpu_compress(torch, src, chunk, level, chunk_bytes)
    frames = o.mt_frames(framed)
    parts = [src[i: i + chunk] for i in range(0, max(src.size, 1), chunk)] if chunk_bytes is None else \
            [src[c * chunk: c * chunk + int(b)] for c, b in enumerate(chunk_bytes)]
    assert len(frames) == len(parts)
    rep = Report()
    rep.framed = framed
    rep.twin = ze.assert_twin(framed, src, chunk, level, chunk_bytes)
    rep.raw_by = ze.raw_counts(rep.twin)
    for fi, (f, content) in enumerate(zip(frames, parts)):
        tr = o.zstd_trace(f)
        assert np.array_equal(tr.content, content)
        check_modes(tr)
        twin = zl.twin_sequences(content, level)
        regen = tr.col("regen")
        blocks = [b for b in range(len(tr.blk)) if regen[b]]
        n = content.size
        assert [int(regen[b]) for b in blocks] == [min(zl.BLOCK, n - i) for i in range(0, n, zl.BLOCK)]
        for k, b in enumerate(blocks):
            rep.types.append(int(tr.blk[b, ZT["type"]]))
            if tr.blk[b, ZT["type"]] != 2:
                continue
            q = tr.block_seqs(b).astype(np.int64)
            assert (q[:, 1] == q[:, 3] + 3).all()                     # Offset_Value = offset + 3: no repeat codes
            mine = q[:, [0, 3, 2]]
            assert np.array_equal(mine, twin[k].astype(np.int64)), ("parse differs from the twin", fi, k)
            rep.seqs.append((fi, k * zl.BLOCK, mine))
            check_huffman(tr, b, rep)
    check_roundtrip(torch, framed, np.concatenate(parts) if chunk_bytes is not None and parts else src)
    return rep


def starts(seqs, base):
    """Match start positions of one block's sequences."""
    return base + np.cumsum(seqs[:, 0] + seqs[:, 2]) - seqs[:, 2]


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
def test_levels_match_the_twin_on_every_kind(torch, level):
    rng = np.random.default_rng(level)
    chunk = 256 << 10
    src = kinds_stream(rng, chunk)
    rep = check(torch, src, chunk, level)
    s = rep.all_seqs()
    assert s[:, 2].max() > zl.LCAP                                    # merged matches longer than the cap of best[]
    assert s[:, 1].max() > 65535                                      # offsets beyond the level-3 window
    assert 0 in rep.types and 2 in rep.types


@pytest.mark.parametrize("level", LEVELS)
def test_random_chunk_is_all_raw(torch, level):
    src = np.random.default_rng(5).integers(0, 256, (200 << 10) + 17, dtype=np.uint8)
    rep = check(torch, src, 1 << 20, level)
    assert rep.types and set(rep.types) == {0}


@pytest.mark.parametrize("level", LEVELS)
def test_tiny_empty_and_ragged_chunks(torch, level):
    rng = np.random.default_rng(11)
    check(torch, np.zeros(0, np.uint8), 1 << 20, level)
    check(torch, np.array([7], np.uint8), 1 << 20, level)
    check(torch, np.array([1, 2, 1], np.uint8), 1 << 20, level)           # fewer bytes than minMatch
    chunk = 128 << 10
    src = np.concatenate([z.gen_stream(z.GEN_TEXT, chunk, chunk), rng.integers(0, 4, chunk, dtype=np.uint8),
                          z.gen_stream(z.GEN_MIX, 4 * chunk, chunk)])
    check(torch, src, chunk, level, chunk_bytes=[chunk, 1, 0, 3, 70000, chunk - 5])


def window_edge_stream(rng, W):
    """Random bytes in which a 64-byte segment recurs at exactly W and another at W + 1."""
    n = 2 * W + 128
    src = rng.integers(0, 256, n, dtype=np.uint8)
    a, b = 1000, 5000
    src[a + W: a + W + 64] = src[a: a + 64]
    src[b + W + 1: b + W + 65] = src[b: b + 64]
    return src, a + W, b + W + 1


@pytest.mark.parametrize("level", [9, 12])
def test_match_at_exactly_the_window(torch, level):
    W = zl.window(level)
    src, at_w, at_w1 = window_edge_stream(np.random.default_rng(21), W)
    rep = check(torch, src, 16 << 20, level)
    found_w = found_w1 = False
    for _, base, s in rep.seqs:
        st = starts(s, base)
        found_w |= bool(((s[:, 1] == W) & (st == at_w)).any())
        found_w1 |= bool(((st >= at_w1) & (st < at_w1 + 64)).any())
    assert (rep.all_seqs()[:, 1] <= W).all()
    assert found_w and not found_w1


def test_lazy_choice_defers_a_short_match(torch):
    """At p the best match is 5 bytes long, at p + 1 it is 64: the parse emits p as a literal and takes the long one."""
    rng = np.random.default_rng(31)
    R = rng.integers(0, 256, 64, dtype=np.uint8)
    A = np.array([0xAB], np.uint8)
    junk = lambda k: rng.integers(0, 256, k, dtype=np.uint8)
    src = np.concatenate([junk(3000), R, junk(3000), A, R[:4], junk(3000), A, R, junk(3000)])
    p = 3000 + 64 + 3000 + 5 + 3000
    rep = check(torch, src, 1 << 20, 9)
    (fi, base, s), = [x for x in rep.seqs]
    st = starts(s, base)
    assert ((st == p + 1) & (s[:, 2] >= 64)).any() and not (st == p).any()


def test_levels_through_the_c_api_default_chunks(torch):
    """ZSTDCB_compressCCtx with inputsize 0 (4 MiB chunks at levels 6 and 9, 8 MiB at 12): counters as the reference's,
    restored by ZSTDCB_decompressDCtx and by the reference."""
    M = z.memio_lib()
    n = (20 << 20) + 12345
    src = z.gen_stream(z.GEN_MIX, n, 1 << 20)
    cap = n + n // 64 + (1 << 20)
    for level in (6, 9, 12):
        out = np.empty(cap, np.uint8); st = (ctypes.c_size_t * 5)()
        rc = M.zmt_zstd_compress_mem(4, level, 0, src.ctypes.data, n, out.ctypes.data, cap, st)
        assert rc == 0, z.lib().ZSTDCB_getErrorString(rc)
        framed = out[: int(st[0])]
        chunk = 8 << 20 if level >= 10 else 4 << 20
        assert st[1] == -(-n // chunk) and st[2] == n and st[3] == framed.size
        back = np.empty(n + 16, np.uint8); dst = (ctypes.c_size_t * 5)()
        rc = M.zmt_zstd_decompress_mem(4, 0, framed.ctypes.data, framed.size, back.ctypes.data, n + 16, dst)
        assert rc == 0 and dst[0] == n and np.array_equal(back[:n], src)
        if o.have_ref():
            R = o.ref()
            rout = np.empty(cap, np.uint8); rst = (ctypes.c_size_t * 5)()
            assert R.ref_zstd_compress_mem(4, level, 0, src.ctypes.data, n, rout.ctypes.data, cap, rst) == 0
            assert (st[1], st[2]) == (rst[1], rst[2])                  # frames, insize
            assert (st[4] & 0xFFFFFFFF) == (rst[4] & 0xFFFFFFFF) == st[1]  # one write per frame
            # reads: every frame, then a 0-byte read at the end of the input; each of the reference's 4 workers makes its own
            assert st[4] >> 32 == st[1] + 1 and rst[4] >> 32 == rst[1] + 4
            for T in (1, 3):
                rc, rback, _ = o.ref_decompress(o.CODEC_ZSTD, framed, n, threads=T)
                assert rc == 0 and np.array_equal(rback, src)


def test_one_call_over_all_gpus_is_byte_identical(torch, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    src = z.gen_stream(z.GEN_MIX, (40 << 20) + 77, 4 << 20)
    monkeypatch.setenv("ZSTDMT_GPUS", "0")
    rc, one, _ = z.compress_mem(z.CODEC_ZSTD, src, threads=4, level=9, chunk=4 << 20)
    assert rc == 0
    monkeypatch.setenv("ZSTDMT_GPUS", "all")
    rc, allg, _ = z.compress_mem(z.CODEC_ZSTD, src, threads=4, level=9, chunk=4 << 20)
    assert rc == 0 and np.array_equal(one, allg)


@pytest.mark.parametrize("kind", [z.GEN_TEXT, z.GEN_MIX])
def test_level9_ratio_over_level3(torch, kind, capsys):
    """64 MiB in 4 MiB chunks: the level-9 frames carry the twin's parse, and level 9 beats level 3 by at least 5 %."""
    n, chunk = 64 << 20, 4 << 20
    src = z.gen_stream(kind, n, chunk)
    f3 = gpu_compress(torch, src, chunk, 3)
    rep = check(torch, src, chunk, 9)
    r3, r9 = n / f3.size, n / rep.framed.size
    with capsys.disabled():
        print("\n[ratio] %s: level 3 %.4f, level 9 %.4f (%+.1f %%)" % ("text" if kind == z.GEN_TEXT else "mix", r3, r9, 100 * (r9 / r3 - 1)))
    assert rep.seqs
    assert r9 >= 1.05 * r3
