"""The chain-search encoders (zstd levels 6-12, LZ4 levels 10-12) at the edges of their GPU schedule (pytest -m gpu).
Every case of tests/_searchcorpus.py goes through zmt_zstd_compress_level_device or zmt_lz4_compress_level_device and
the check() of test_gpu_zstd_levels.py or test_gpu_lz4_hc.py: GPU sequences equal the CPU twin's block for block (the
LZ4 stream byte for byte), raw zstd blocks are raw for a reason, and the frames round-trip through the GPU decoder,
the oracle and the reference.  The scale cases make each CTA of the persistent block kernels encode two different
windows, and make a batch span several groups of chunks (ZL_GROUP_BYTES of positions each)."""
import struct

import numpy as np
import pytest

import _lz4hc as hc
import _oracle as o
import _searchcorpus as sc
import _zlazy as zl
import test_gpu_lz4_hc as tl
import test_gpu_zstd_levels as tz
import zstdmt_b200 as z

pytestmark = pytest.mark.gpu
CASES = sc.cases()
BY_NAME = {c.name: c for c in CASES}
GROUP_BYTES = 256 << 20                  # ZL_GROUP_BYTES
MAX_GRID = 132 * 8                       # ZSTD_MAX_GRID


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def run_check(torch, codec, src, chunk, level, chunk_bytes=None):
    if codec == "zstd":
        return tz.check(torch, src, chunk, level, chunk_bytes)
    return tl.check(torch, src, chunk, level, chunk_bytes)


@pytest.mark.parametrize("name,level", [(c.name, lv) for c in CASES for lv in c.levels])
def test_corpus_case_on_the_gpu(torch, name, level):
    case = BY_NAME[name]
    rep = run_check(torch, case.codec, case.src, case.chunk, level, case.chunk_bytes)
    if case.gpu_check:
        case.gpu_check(level, rep)


def grid(torch):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return min(sm * 8, MAX_GRID)


# ------------------------------------------------------------------------------------------------- 13: persistent loop
def corpus_windows():
    """64 KiB windows of the corpus cases with content (the last one of a case may be short)."""
    wins = []
    for case in CASES:
        for part in sc.parts(case):
            wins += [part[i: i + 65536] for i in range(0, min(part.size, 4 << 20), 65536) if part[i: i + 65536].size >= 1000]
    return wins


@pytest.mark.parametrize("codec,level", [("zstd", 6), ("zstd", 12), ("lz4", 10)])
def test_each_cta_encodes_two_different_windows(torch, codec, level, capsys):
    """Chunk size 64 KiB (one window per chunk) and explicit sizes from 1 byte to 64 KiB: more non-empty windows than
    the persistent grid has CTAs, so every CTA c encodes window c and then window c + grid.  The two hold different
    corpus windows, so that whatever one leaves in shared memory, its ZScratch or its job list meets another; the
    windows past 2 * grid are short ones of 1 byte to 4 KiB."""
    g = grid(torch)
    wins = corpus_windows()
    chunk = 65536
    nch = 2 * g + 64
    rng = np.random.default_rng(1300 + level)
    sizes = [int(rng.integers(1, 4097)) for _ in range(nch)]
    src = np.zeros(nch * chunk, np.uint8)
    for c in range(nch):
        src[c * chunk: c * chunk + sizes[c]] = rng.integers(0, 4, sizes[c], dtype=np.uint8)
    for i in range(g):
        a, b = i % len(wins), (i + 1 + i // len(wins)) % len(wins)
        assert a != b
        for c, w in ((i, wins[a]), (i + g, wins[b])):
            src[c * chunk: c * chunk + w.size] = w
            sizes[c] = int(w.size)
    nonempty = sum(1 for s in sizes if s)
    assert g < nonempty and max(sizes) == chunk and min(sizes) >= 1
    run_check(torch, codec, src, chunk, level, sizes)
    with capsys.disabled():
        print("\n[persistent] %s level %d: grid %d, %d non-empty windows" % (codec, level, g, nonempty))


# ------------------------------------------------------------------------------------------------- 14: two groups
def frame_slices(framed):
    """[start, end) of every frame of a framed stream (12-byte container header included)."""
    out, pos = [], 0
    while pos < framed.size:
        _, _, cs = struct.unpack("<III", framed[pos: pos + 12].tobytes())
        out.append((pos, pos + 12 + cs))
        pos += 12 + cs
    return out


@pytest.mark.parametrize("codec,level", [("zstd", 6), ("lz4", 10)])
@pytest.mark.parametrize("chunk", [1 << 20, (3 << 20) + 4096])
def test_batch_over_several_groups_explicit_sizes(torch, codec, level, chunk, capsys):
    """About 300 chunks of 20-70 KiB with explicit sizes: the per-position arrays cover 256 MiB of positions at a time,
    so the batch runs in several groups (chunk 3 MiB + 4 KiB: a group size that does not divide 256 MiB).  Every frame
    is checked against the twin."""
    rng = np.random.default_rng(1400)
    nch = 300
    G = GROUP_BYTES // chunk
    ngroups = -(-nch // G)
    assert ngroups >= 2
    sizes = [int(rng.integers(20 << 10, 70 << 10)) for _ in range(nch)]
    body = z.gen_stream(z.GEN_MIX, 4 << 20, 1 << 20, first=5)
    src = np.zeros(nch * chunk, np.uint8)
    for c, s in enumerate(sizes):
        a = int(rng.integers(0, body.size - s))
        src[c * chunk: c * chunk + s] = body[a: a + s]
    run_check(torch, codec, src, chunk, level, sizes)
    with capsys.disabled():
        print("\n[groups] %s chunk %d: %d chunks per group, %d groups" % (codec, chunk, G, ngroups))


@pytest.mark.parametrize("codec,level", [("zstd", 6), ("lz4", 10)])
def test_batch_over_two_groups_short_last_group(torch, codec, level, capsys):
    """Implicit chunk sizes, 1 MiB chunks and 261 MiB + 12345 bytes: a full group of 256 chunks, then a short one whose
    positions end with the input.  The frames on both sides of the group boundary and the last one are checked against
    the twin; every frame round-trips."""
    chunk = 1 << 20
    n = (261 << 20) + 12345
    src = z.gen_stream(z.GEN_MIX, n, chunk, first=4)
    G = GROUP_BYTES // chunk
    nch = -(-n // chunk)
    assert nch > G
    parts = [src[i: i + chunk] for i in range(0, n, chunk)]
    pick = [G - 1, G, nch - 1]
    if codec == "zstd":
        framed = tz.gpu_compress(torch, src, chunk, level)
        frames = o.mt_frames(framed)
        assert len(frames) == nch
        for fi in pick:
            tr = o.zstd_trace(frames[fi])
            assert np.array_equal(tr.content, parts[fi])
            twin = zl.twin_sequences(parts[fi], level)
            blocks = [b for b in range(len(tr.blk)) if tr.blk[b, o.ZT["regen"]]]
            assert len(blocks) == len(twin)
            for k, b in enumerate(blocks):
                if tr.blk[b, o.ZT["type"]] == 2:
                    q = tr.block_seqs(b).astype(np.int64)
                    assert np.array_equal(q[:, [0, 3, 2]], twin[k].astype(np.int64)), ("parse differs from the twin", fi, k)
        tz.check_roundtrip(torch, framed, src)
    else:
        framed = tl.gpu_compress(torch, src, chunk, level)
        sl = frame_slices(framed)
        assert len(sl) == nch
        for fi in pick:
            a, e = sl[fi]
            assert np.array_equal(framed[a: e], hc.twin_compress(parts[fi], chunk, level)), ("frame differs from the twin", fi)
        tl.check_roundtrip(torch, framed, parts)
    with capsys.disabled():
        print("\n[groups] %s implicit sizes: %d chunks, %d groups" % (codec, nch, -(-nch // G)))
