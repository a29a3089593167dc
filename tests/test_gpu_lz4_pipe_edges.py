"""The LZ4 block compressor on inputs built around its schedule (needs an H100: pytest -m gpu).

The candidate rounds give each thread four consecutive positions, so block ends of every residue mod 4 and short
periods starting at every offset inside a quad are checked.  The back end finds the offset a sequence carries across
segments by a scan over the pieces, so long matches spanning many segments are followed at once by a match with
another offset, or with the same offset after one literal.  Every case compares the GPU stream byte for byte with
the oracle's CPU twin and decodes it back."""
import numpy as np
import pytest

import _oracle as o
import zstdmt_b200 as z

pytestmark = pytest.mark.gpu

CHUNK = 1 << 20


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def check_twin(torch, src, chunk=CHUNK):
    comp = z.Lz4DeviceCompressor(int(src.size), chunk)
    out, foff = comp.run(torch.from_numpy(src).cuda())
    torch.cuda.synchronize()
    framed = out[: int(foff.cpu().numpy()[-1])].cpu().numpy()
    expect = o.orc_encode_lz4(src, chunk)
    assert framed.size == expect.size and np.array_equal(framed, expect), "GPU stream differs from the oracle twin"
    rc, back = o.orc_decode(o.CODEC_LZ4, framed, src.size)
    assert rc == 0 and np.array_equal(back, src)


def periodic(rng, n, period):
    return np.resize(rng.integers(0, 256, period, dtype=np.uint8), n)


# the last block of the chunk has n bytes: quads that straddle the i + 12 <= n test, and limit = n - 5 at every
# residue, including a last piece that ends at limit on a tile boundary (n = 4096 k + 5)
@pytest.mark.parametrize("base", [12, 4096, 4096 + 5, 3 * 4096 + 5, 65536])
@pytest.mark.parametrize("kind", ["mix", "period3", "period7", "zeros"])
def test_block_ends_every_residue(torch, base, kind):
    rng = np.random.default_rng(base)
    for n in range(max(1, base - 4), base + 5):
        total = (CHUNK - 65536 + n) if base == 65536 else n       # 65536: the chunk's last block is full or 1-4 bytes
        if kind == "mix":
            src = z.gen_stream(z.GEN_MIX, total, CHUNK, first=3)
        elif kind == "zeros":
            src = np.zeros(total, np.uint8)
        else:
            src = periodic(rng, total, int(kind[6:]))
        check_twin(torch, src)


def long_match_then(rng, seg_span, align, follow):
    """A random block, then a copy of it spanning seg_span segments that ends `align` bytes into a segment, then
    at once a match with another offset ('other'), or one literal and the same offset again ('same')."""
    head = rng.integers(0, 256, 4096 + align, dtype=np.uint8)
    span = 16 * seg_span + align
    back = 3000
    parts = [head]
    cur = np.concatenate(parts)
    parts.append(cur[cur.size - back: cur.size - back + span])    # offset `back`, span bytes
    cur = np.concatenate(parts)
    if follow == "other":
        parts.append(cur[cur.size - 517: cur.size - 517 + 100])   # offset 517 right after
    else:
        parts.append(np.array([cur[cur.size - back] ^ 0x5A], np.uint8))   # one literal breaks the match ...
        cur = np.concatenate(parts)
        parts.append(cur[cur.size - back: cur.size - back + 100])  # ... then offset `back` again
    parts.append(rng.integers(0, 256, 300, dtype=np.uint8))
    return np.concatenate(parts)


@pytest.mark.parametrize("follow", ["other", "same"])
@pytest.mark.parametrize("seg_span", [40, 63, 255, 300])
def test_long_match_across_segments_then_next_match(torch, follow, seg_span):
    rng = np.random.default_rng(seg_span)
    # sixteen alignments of the match end; the lead-in shifts each case against the tile grid too
    src = np.concatenate([long_match_then(rng, seg_span, a, follow) for a in range(16)])
    check_twin(torch, src)
    check_twin(torch, src, chunk=65536)


@pytest.mark.parametrize("period", [1, 2, 3, 4])
def test_short_periods_at_quad_offsets(torch, period):
    rng = np.random.default_rng(period)
    parts = []
    for lead in range(16):                        # the run starts at every offset inside a quad and a segment
        parts.append(rng.integers(0, 256, 64 + lead, dtype=np.uint8))
        for runlen in (5, 12, 13, 40, 700):
            parts.append(periodic(rng, runlen, period))
            parts.append(rng.integers(0, 256, 3 + lead % 4, dtype=np.uint8))
    src = np.concatenate(parts)
    check_twin(torch, src)
    check_twin(torch, src[: 4096 - 7])
