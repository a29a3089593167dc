"""CPU tests of the segment walk of zstd frames (zmt_zstd_segment_host, frame_format.h zstd_walk_blocks): a frame cut at
block boundaries into segments, as the plain-stream path decodes frames larger than a batch.  Frames come from the
dictated-parse corpus of tests/_zcorpus.py and from libzstd at levels 1, 3 and 19, with and without a content checksum and
a content size.  The references are a plain Python walk of the frame and block headers, and, for the tables a block
inherits, _zcorpus.repeat_sources on the oracle's block trace."""
import numpy as np
import pytest

import _oracle as o
import _zcorpus as zc
import zstdmt_b200 as z
from test_gpu_plain_streams import zstd_adv
from test_zstd_decode_corpus import NONE, PREDEF, SELF, ZBLK, expected_sources, host_scan

OK, TRUNCATED = 0, 1
ZB_SRC = 3
CORPUS = ["reps", "reps_predef", "tables", "literals", "deep", "dense", "far"]
LIBZSTD = [(lv, chk, cs) for lv in (1, 3, 19) for chk in (0, 1) for cs in (1, 0)]


def header_walk(fr):
    """The frame header and block headers of one zstd frame: Window_Size, content size (None without one), and per block
    (content offset, content bytes, type); `end` = the frame's length."""
    fhd = int(fr[4])
    single, fcs, did = (fhd >> 5) & 1, fhd >> 6, fhd & 3
    pos = 5 + (0 if single else 1) + [0, 1, 2, 4][did]
    fl = [1 if single else 0, 2, 4, 8][fcs]
    cs = int.from_bytes(fr[pos:pos + fl].tobytes(), "little") + (256 if fl == 2 else 0) if fl else None
    if single:
        window = cs
    else:
        wd = int(fr[5]); wb = 1 << (10 + (wd >> 3)); window = wb + (wb >> 3) * (wd & 7)
    pos += fl
    blocks = []
    while True:
        bh = int.from_bytes(fr[pos:pos + 3].tobytes(), "little"); pos += 3
        typ, bs = (bh >> 1) & 3, bh >> 3
        size = 1 if typ == 1 else bs
        blocks.append((pos, size, typ)); pos += size
        if bh & 1:
            break
    return dict(window=window, cs=cs, single=bool(single), blocks=blocks, end=pos + (4 if fhd & 4 else 0))


def libzstd_frame(level, checksum, content_size):
    src = z.gen_stream(z.GEN_MIX if level != 19 else z.GEN_TEXT, (3 << 20) + 4321 * level, 1 << 20, first=level)
    if content_size:
        return zstd_adv(src, level, checksum=checksum, content_size=1)
    return zstd_adv(src, level, checksum=checksum, pieces=[src.size // 3, src.size - src.size // 3])


def frame_of(name):
    if isinstance(name, tuple):
        return libzstd_frame(*name)
    return zc.case(name)[1]


_TRACES = {}


def trace_of(name):
    if isinstance(name, str):
        return zc.trace(name)
    if name not in _TRACES:
        _TRACES[name] = o.zstd_trace(frame_of(name))
    return _TRACES[name]


FRAMES = CORPUS + LIBZSTD
IDS = CORPUS + ["l%d_chk%d_cs%d" % t for t in LIBZSTD]


def segment(fr, w, start, max_in, max_out=1 << 62):
    """One segment of fr from frame offset `start` (= w.pos) with its carried sources below: (rc, end, room, flags, last,
    descriptors, carry bytes, carried source list)."""
    srcs = z.zstd_segment_sources(w)
    carry = b"".join(fr[a:a + n].tobytes() for a, n in srcs)
    rc, end, room, flags, last, blk, _ = z.zstd_segment(fr[start:], w, max_in, max_out, base_off=len(carry))
    return rc, end, room, flags, last, blk.view(ZBLK), carry, srcs


@pytest.mark.parametrize("name", FRAMES, ids=IDS)
def test_segment_walk_matches_the_whole_frame_walk_at_every_cut(name):
    fr = frame_of(name)
    hw = header_walk(fr)
    assert hw["end"] == fr.size
    rc, whole, cs, flags = host_scan(fr)
    assert rc == OK and len(whole) == len(hw["blocks"])
    cuts = [a + n for a, n, _ in hw["blocks"]][:-1]
    exp = expected_sources(trace_of(name), 0)
    ks = list(range(1, len(cuts) + 1))
    if len(ks) > 80:
        ks = sorted(set(int(k) for k in np.linspace(1, len(ks), 80)))
    carried_before = 0
    for k in ks:
        c = cuts[k - 1]
        w = z.ZstdWalk()
        rc, e1, _, f1, last1, b1, carry1, _ = segment(fr, w, 0, c)
        assert rc == OK and e1 == c and not last1 and len(carry1) == 0
        assert (b1 == whole[:k]).all()
        assert w.pos == c and w.window == hw["window"] and w.nblk == k
        rc, e2, room2, f2, last2, b2, carry, srcs = segment(fr, w, c, 1 << 62)
        assert rc == OK and c + e2 == fr.size and last2 and w.done == 1
        assert f2 == flags | 1                                   # the dependent-block route, always
        nc = len(srcs)
        assert (b2["type"][:nc] == ZB_SRC).all() and (b2["type"][nc:] != ZB_SRC).all() and (b2["regen_hint"][:nc] == 0).all()
        real, ref = b2[nc:], whole[k:]
        assert len(real) == len(ref)
        # the same blocks, with comp_off shifted to the segment's input and scratch counted from the segment's start
        assert ((real["comp_off"] - len(carry)).astype(np.int64) == ref["comp_off"].astype(np.int64) - c).all()
        for f in ("comp_size", "frame", "type", "regen_hint", "nseq"):
            assert (real[f] == ref[f]).all(), f
        assert (real["first"] == 0).all()
        cmp_ = ref["type"] == 2                                  # (raw and RLE blocks take no scratch)
        if cmp_.any():
            rs, gs = ref[cmp_], real[cmp_]
            d = int(rs["seq_off"][0]) - int(gs["seq_off"][0])
            assert (rs["seq_off"].astype(np.int64) - gs["seq_off"].astype(np.int64) == d).all()
            assert (rs["lit_off"].astype(np.int64) - gs["lit_off"].astype(np.int64) == d).all()
        # table sources: a describer behind the cut is this segment's block; one before it is a carried descriptor
        # holding the describing block's bytes
        for j in range(len(ref)):
            b = k + j
            if hw["blocks"][b][2] != 2:
                continue
            for t, f in enumerate(("huf_src", "ll_src", "of_src", "ml_src")):
                want, got = exp[b][t], int(real[f][j])
                if want in (SELF, PREDEF, NONE):
                    assert got == want, (name, k, b, f)
                elif want >= k:
                    assert got == nc + want - k, (name, k, b, f)
                else:
                    assert got < nc, (name, k, b, f)
                    a, n, _ = hw["blocks"][want]
                    at = int(b2["comp_off"][got])
                    assert int(b2["comp_size"][got]) == n and carry[at:at + n] == fr[a:a + n].tobytes(), (name, k, b, f)
                    carried_before += 1
        assert room2 == sum(128 << 10 if typ == 2 else (n if typ == 0 else int(whole["regen_hint"][i]))
                            for i, (_, n, typ) in enumerate(hw["blocks"][k:], start=k))
    if name in ("tables", "literals", "reps"):                   # inherited tables across a cut were met
        assert carried_before > 0


@pytest.mark.parametrize("name", FRAMES, ids=IDS)
def test_one_block_per_segment_tiles_the_frame(name):
    fr = frame_of(name)
    hw = header_walk(fr)
    cuts = [a + n for a, n, _ in hw["blocks"]]
    w, start, ends = z.ZstdWalk(), 0, []
    while True:
        rc, end, _, _, last, blk, carry, srcs = segment(fr, w, start, 1)
        assert rc == OK and len(blk) - len(srcs) == 1 and len(srcs) <= 4
        start += end; ends.append(start)
        if last:
            break
    assert ends == cuts[:-1] + [fr.size]


@pytest.mark.parametrize("name", FRAMES[::2], ids=IDS[::2])
def test_walk_stops_at_the_first_boundary_past_the_targets(name):
    fr = frame_of(name)
    hw = header_walk(fr)
    cuts = [a + n for a, n, _ in hw["blocks"]]
    stops = cuts[:-1] + [fr.size]
    for target in (1, 5000, 100000, 1 << 20, 3 << 20):
        w = z.ZstdWalk()
        rc, end, _, _, last, _, _, _ = segment(fr, w, 0, target)
        assert rc == OK and end == min([s for s in stops if s >= target] + [fr.size]) and bool(last) == (end == fr.size)
    # an output target: the first boundary where the rooms reach it
    rooms = np.cumsum([128 << 10 if typ == 2 else n for _, n, typ in hw["blocks"]])
    rle = [i for i, (_, _, typ) in enumerate(hw["blocks"]) if typ == 1]
    if not rle:
        want = int(rooms[len(rooms) // 2])
        k = int(np.argmax(rooms >= want))
        w = z.ZstdWalk()
        rc, end, room, _, last, _, _, _ = segment(fr, w, 0, 1 << 40, want)
        assert rc == OK and room == int(rooms[k]) and end == stops[k]


@pytest.mark.parametrize("name", FRAMES[1::2], ids=IDS[1::2])
def test_a_segment_cut_short_reports_need_more(name):
    fr = frame_of(name)
    hw = header_walk(fr)
    cuts = [a + n for a, n, _ in hw["blocks"]]
    for n in (3, 5, hw["blocks"][0][0] - 1, cuts[0] - 1):
        w = z.ZstdWalk()
        rc, *_ = segment(fr[:n], w, 0, 1)
        assert rc == TRUNCATED and w.pos == 0 and w.nblk == 0              # the walk stays where it was
    if len(cuts) > 2:
        w = z.ZstdWalk()
        assert segment(fr, w, 0, cuts[0])[0] == OK
        before = bytes(w)
        for cut in (cuts[1] - 1, cuts[0] + 2):
            rc, *_ = segment(fr[:cut], w, cuts[0], 1 << 62)
            assert rc == TRUNCATED and bytes(w) == before
    if fr[4] & 4:                                                # the last segment without all of its checksum
        w = z.ZstdWalk()
        assert segment(fr, w, 0, cuts[-2] if len(cuts) > 1 else 1)[0] == OK
        start = w.pos
        if start < cuts[-1]:
            rc, *_ = segment(fr[:fr.size - 2], w, start, 1 << 62)
            assert rc == TRUNCATED


def test_window_size_matches_the_frame_descriptor():
    seen = set()
    for name in FRAMES:
        fr = frame_of(name)
        hw = header_walk(fr)
        w = z.ZstdWalk()
        rc, *_ = segment(fr, w, 0, 1)
        assert rc == OK and w.window == hw["window"], name
        assert w.content_size == (hw["cs"] if hw["cs"] is not None else (1 << 64) - 1)
        seen.add(hw["single"])
    # a Single_Segment frame (Window_Size = Frame_Content_Size) from libzstd's one-shot API, and one with a descriptor
    src = z.gen_stream(z.GEN_TEXT, 700000, 1 << 20, first=2)
    fr = zc.compress(src, {zc.P_LEVEL: 3})
    hw = header_walk(fr)
    assert hw["single"] and hw["window"] == src.size
    w = z.ZstdWalk()
    assert segment(fr, w, 0, 1)[0] == OK and w.window == src.size
    assert False in seen
    fr = zc.compress(src, {zc.P_LEVEL: 19, zc.P_WINDOWLOG: 23})
    w = z.ZstdWalk()
    assert segment(fr, w, 0, 1)[0] == OK and w.window == header_walk(fr)["window"]
