"""CPU tests of the segment walk of LZ4F frames (zmt_lz4f_segment_host, frame_format.h lz4f_walk_blocks): a frame cut
at block boundaries into segments, as the plain-stream path decodes frames larger than a batch.  Frames come from
liblz4 (block sizes 64 KiB .. 4 MiB, linked and independent blocks, with and without block checksums) and from the
dictated-parse corpus of tests/_lz4corpus.py; the reference for the boundaries is a plain Python walk of the block
headers."""
import numpy as np
import pytest

import zstdmt_b200 as z
import _lz4corpus as lc
from test_gpu_plain_streams import lz4f

OK, TRUNCATED = 0, 1


def header_len(flg):
    return 7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)


def boundaries(fr):
    """Frame offsets behind every block, the output room of every block, and the frame length."""
    flg, bd = int(fr[4]), int(fr[5])
    blkmax = 1 << (8 + 2 * ((bd >> 4) & 7))
    q, cuts, rooms = header_len(flg), [], []
    while True:
        bh = int.from_bytes(fr[q:q + 4].tobytes(), "little"); q += 4
        if bh == 0:
            break
        bs = bh & 0x7FFFFFFF
        q += bs + (4 if flg & 0x10 else 0)
        cuts.append(q); rooms.append(bs if bh >> 31 else blkmax)
    return cuts, rooms, q + (4 if flg & 4 else 0)


def walk(fr, max_in=1, max_out=1 << 62):
    """Segments of fr as the walk cuts them: [(start, end, room, last)]."""
    flg, bd = int(fr[4]), int(fr[5])
    segs, start, first = [], 0, True
    while True:
        rc, end, room, last = z.lz4f_segment(fr[start:], header_len(flg) if first else 0, flg, bd, max_in, max_out)
        assert rc == OK
        segs.append((start, start + end, room, last))
        if last:
            return segs
        start += end; first = False


def liblz4_frames():
    src = z.gen_stream(z.GEN_MIX, (9 << 20) + 4321, 1 << 20, first=3)
    out = []
    for bsid in (4, 5, 6, 7):
        for mode in (0, 1):                                   # blockMode 0 = linked, 1 = independent
            for bchk in (0, 1):
                out.append(("b%d_m%d_bc%d" % (bsid, mode, bchk), lz4f(src, blockSizeID=bsid, blockMode=mode, blockChecksumFlag=bchk,
                                                                      contentChecksumFlag=1, contentSize=int(src.size) if bchk else 0)))
    return out


FRAMES = liblz4_frames()


@pytest.mark.parametrize("name,fr", FRAMES, ids=[n for n, _ in FRAMES])
def test_walk_cuts_liblz4_frames_at_every_block_boundary(name, fr):
    cuts, rooms, length = boundaries(fr)
    assert length == fr.size and len(cuts) >= 2
    segs = walk(fr)                                            # max_in = 1: one block per segment
    assert [e for _, e, _, _ in segs[:-1]] == cuts
    assert [r for _, _, r, _ in segs[:len(rooms)]] == rooms
    assert segs[-1][1] == fr.size and segs[-1][3] == 1 and all(not s[3] for s in segs[:-1])
    # one block per segment: the last segment holds the end mark and the content checksum alone
    assert (segs[-1][0], segs[-1][2]) == (cuts[-1], 0)
    # one segment reaching the whole frame: the frame's bound, as the whole-frame walk gives it
    (s0, e0, r0, l0), = walk(fr, max_in=fr.size)
    assert (s0, e0, l0) == (0, fr.size, 1) and r0 == sum(rooms)


@pytest.mark.parametrize("name,fr", FRAMES[:4], ids=[n for n, _ in FRAMES[:4]])
def test_walk_stops_at_the_first_boundary_past_the_targets(name, fr):
    cuts, rooms, _ = boundaries(fr)
    flg, bd = int(fr[4]), int(fr[5])
    for target in (1, 100000, 1 << 20, 3 << 20):
        rc, end, room, last = z.lz4f_segment(fr, header_len(flg), flg, bd, target, 1 << 62)
        assert rc == OK and end == min(c for c in cuts + [fr.size] if c >= target)
    # an output target: the first boundary where the rooms reach it
    want = 3 * (1 << (8 + 2 * ((bd >> 4) & 7)))
    k = int(np.argmax(np.cumsum(rooms) >= want))
    rc, end, room, last = z.lz4f_segment(fr, header_len(flg), flg, bd, 1 << 40, want)
    assert rc == OK and end == cuts[k] and room == sum(rooms[:k + 1]) and not last


@pytest.mark.parametrize("name,fr", FRAMES[::3], ids=[n for n, _ in FRAMES[::3]])
def test_walk_reports_a_segment_cut_short_as_need_more(name, fr):
    cuts, _, _ = boundaries(fr)
    flg, bd = int(fr[4]), int(fr[5])
    for n in (cuts[0] - 1, cuts[0] - 200, header_len(flg) + 2):
        rc, _, _, _ = z.lz4f_segment(fr[:n], header_len(flg), flg, bd, 1, 1 << 62)
        assert rc == TRUNCATED
    rc, end, _, _ = z.lz4f_segment(fr[:cuts[0]], header_len(flg), flg, bd, 1, 1 << 62)
    assert rc == OK and end == cuts[0]
    # the last segment without its content checksum, and without its end mark
    for cut in (1, 4, 8):
        rc, _, _, _ = z.lz4f_segment(fr[cuts[-1]:fr.size - cut], 0, flg, bd, 1 << 40, 1 << 62)
        assert rc == TRUNCATED


@pytest.mark.parametrize("name", ["linked", "ends", "periods"])
@pytest.mark.parametrize("bchk", [False, True])
def test_walk_on_dictated_frames(name, bchk):
    """Frames of tests/_lz4corpus.py: stored and zero-size blocks, dictionary IDs, content sizes; boundaries at every block."""
    for fr, src, info in lc.case(name, "full", bchk):
        cuts, rooms, length = boundaries(fr)
        assert length == fr.size
        segs = walk(fr)
        assert [e for _, e, _, _ in segs[:-1]] == cuts
        if info:                                               # every block boundary is where the corpus wrote a block
            flg = int(fr[4]); q, ends = header_len(flg), []
            for _, data, _ in info:
                q += 4 + len(data) + (4 if bchk else 0); ends.append(q)
            assert ends == cuts
