"""GPU tests of zstd frames written with a dictionary: load the dictionary on the device, index and decode container and
plain streams against it, and refuse what libzstd refuses.

Every frame is compared with its source and with libzstd's ZSTD_decompress_usingDict, through three routes: the host scan
(ZstdDeviceDecompressor), the device index of a container stream and the device index of a plain stream with skippable
frames (from_device).  The dictated-parse corpus names the edge each case exists for as a predicate on its parse, and the
test asserts that every edge is reached."""
import ctypes

import numpy as np
import pytest
import torch

import zstdmt_b200 as z
import _zcorpus as zc
import _zdict as zd

pytestmark = pytest.mark.gpu

MX_SPAN, MAXBLOCK = 2048, 1024
BLK = np.dtype([("comp_off", "<u8"), ("comp_size", "<u4"), ("frame", "<u4"), ("type", "<u4"), ("regen_hint", "<u4"), ("nseq", "<u4"),
                ("first", "<u4"), ("seq_off", "<u8"), ("lit_off", "<u8"), ("huf_src", "<u4"), ("ll_src", "<u4"), ("of_src", "<u4"),
                ("ml_src", "<u4")])


def outputs(dec):
    torch.cuda.synchronize()
    out, st = dec.out.cpu().numpy(), dec.status.cpu().numpy()[: dec.n]
    oo = dec.d_out_off.cpu().numpy()
    sizes = dec.out_size.cpu().numpy()[: dec.n]
    return [out[int(oo[i]): int(oo[i]) + int(sizes[i])] for i in range(dec.n)], st, oo[: dec.n]


def decode_everywhere(frames, dct, seed=0):
    """The three routes; returns the per-frame outputs of each, the status arrays, the output offsets and the host-scan decoder."""
    routes = {}
    cont = zd.container(frames)
    dec = z.ZstdDeviceDecompressor(cont, dictionary=dct)
    assert dec.scan_ok, dec.scan_status
    d_cont = torch.from_numpy(cont).cuda()
    dec.run(d_cont)
    routes["host"] = outputs(dec)
    dv = z.ZstdDeviceDecompressor.from_device(d_cont, dictionary=dct)
    dv.run(d_cont)
    routes["device"] = outputs(dv)
    pl = zd.plain(frames, seed)
    d_pl = torch.from_numpy(pl).cuda()
    dp = z.ZstdDeviceDecompressor.from_device(d_pl, plain=True, dictionary=dct)
    dp.run(d_pl)
    routes["plain"] = outputs(dp)
    return routes, dec


def check(frames, srcs, d, dct, seed=0):
    routes, dec = decode_everywhere(frames, dct, seed)
    for i, (fr, s) in enumerate(zip(frames, srcs)):
        bad, ref = zd.decompress(fr, d, s.size)
        assert not bad and np.array_equal(ref, s), "libzstd disagrees with the source, frame %d" % i
    for name, (outs, st, _) in routes.items():
        assert (st == 0).all(), (name, st[st != 0][:8], np.nonzero(st)[0][:8])
        for i, s in enumerate(srcs):
            assert np.array_equal(outs[i], s), (name, i)
    return routes, dec


def host_blocks(dec):
    return np.frombuffer(dec.d_blocks.cpu().numpy().tobytes(), BLK)[: dec.nblk]


def test_trained_and_finalized_dictionaries_at_several_levels():
    recs = zd.records(21, 48)
    rng = np.random.default_rng(3)
    dicts = [("trained_16k", zd.train(7, 16 << 10)), ("trained_112k", zd.train(8, 112 << 10)),
             ("finalized_64k", zd.finalize(9, np.concatenate(zd.records(10, 80))[: 56 << 10], 64 << 10, level=9, dict_id=77))]
    reuse = np.zeros(4, int)
    for name, d in dicts:
        dct = z.ZstdDictionary(d)
        assert dct.info.kind == 1 and dct.info.dict_id == zd.dict_id(d) and dct.info.content_off + dct.info.content_bytes == d.size, name
        frames, srcs = [], []
        for k, lvl in enumerate((1, 3, 9, 19)):
            for j, r in enumerate(recs[k::4][:6]):
                frames.append(zd.compress(r, d, level=lvl, checksum=j & 1, content_size=(j >> 1) & 1, dict_id_flag=int(j % 3 != 2)))
                srcs.append(r)
        _, dec = check(frames, srcs, d, dct, seed=len(name))
        b = host_blocks(dec)
        for t, k in enumerate(("huf_src", "ll_src", "of_src", "ml_src")):
            reuse[t] += int((b[k] == zd.ZB_DICT).sum())
    assert (reuse > 0).all(), reuse            # treeless literals and Repeat_Mode LL / OF / ML tables taken from the dictionary


def test_raw_content_dictionaries():
    recs = zd.records(31, 30)
    for size in (1, 4096, 60000):
        d = np.concatenate(zd.records(32, 40))[:size]
        dct = z.ZstdDictionary(d)
        assert dct.info.kind == 0 and dct.info.dict_id == 0 and dct.info.content_bytes == size
        frames = [zd.compress(r, d, level=(3, 9, 19)[i % 3], checksum=i & 1, kind=zd.DCT_RAW) for i, r in enumerate(recs)]
        check(frames, recs, d, dct)


# ---------------------------------------------------------------- dictated parses reaching into the dictionary
def build(seqs, tail, content, rng):
    """The source a parse describes when the dictionary's content precedes it."""
    C = content.size
    hist = np.concatenate([content, np.zeros(int(sum(a + c for a, _, c in seqs)) + tail, np.uint8)])
    p = C
    for ll, off, ml in seqs:
        hist[p: p + ll] = rng.integers(0, 256, ll); p += ll
        assert 0 < off <= p, (off, p - C)
        for k in range(ml):
            hist[p + k] = hist[p - off + k]
        p += ml
    hist[p: p + tail] = rng.integers(0, 256, tail); p += tail
    return hist[C:p].copy()


EDGES = ("inside", "straddle", "first_byte", "long_straddle", "step_chain", "later_block", "dict_rep", "align")


def edges_of(seqs, C, reps, small_blocks):
    e = set()
    p = 0
    prev = None
    for i, (ll, off, ml) in enumerate(seqs):
        p += ll
        s = p - off
        if s + ml <= 0:
            e.add("inside")
        if s < 0 < s + ml:
            e.add("straddle")
            if ml > MX_SPAN and not small_blocks:
                e.add("long_straddle")                  # one block holds the whole match: the global-memory copy
            if p >= 2 * MAXBLOCK and small_blocks:
                e.add("later_block")                    # reads the content and block 0 while earlier blocks may be in flight
        if s == -C:
            e.add("first_byte")
        if prev is not None and prev[1] < 0 and prev[0] <= s < prev[0] + prev[2] and ml + prev[2] < 256:
            e.add("step_chain")
        if i == 0 and off in reps and s < 0:
            e.add("dict_rep")
        prev = (p, s, ml)
        p += ml
    return e


def dictated_cases(C, reps, rng):
    """(parse, small blocks): small blocks cut the frame into MAXBLOCK-byte blocks."""
    cases = [([(5, C // 2, 20), (3, 40, 10)], True),                              # wholly inside the content
             ([(10, 30, 60), (4, 7, 9)], True),                                   # straddles the content's end and the frame's start
             ([(7, C + 7, 16), (0, C + 23, 12)], True),                            # reaches the content's first byte exactly
             ([(100, 2000, 5000), (8, 9, 40)], False),                            # a straddling match longer than MX_SPAN
             ([(2, 20, 6), (1, 6, 5), (0, 12, 7), (3, 30, 4), (1, 5, 9)], True),  # short matches reading the content and each other
             ([(600, 500, 400)] * 3 + [(50, 3150, 900), (20, 4000, 30)], True)]   # a later block straddling into block 0
    for r in reps:                                                                 # the first sequence takes a repeat offset
        cases.append(([(0 if r == 1 else 2, r, 12), (4, 100, 8)], True))
    for k in range(6):                                                             # random mixes
        seqs, p = [], 0
        for _ in range(int(rng.integers(20, 80))):
            ll = int(rng.integers(0, 40)); p += ll
            off = int(rng.integers(1, p + C + 1)); ml = int(rng.integers(3, 300))
            seqs.append((ll, off, ml)); p += ml
        cases.append((seqs, bool(k & 1)))
    return cases


def test_dictated_parses_reach_every_edge():
    rng = np.random.default_rng(41)
    content = np.concatenate(zd.records(42, 40))[: 6 << 10]
    C = content.size
    # a formatted dictionary whose repeat offsets are not the defaults: the first block's repeat codes must take these
    f = zd.finalize(43, content, C + 4096, level=3, dict_id=4242)
    at = f.size - C - 12
    fr = f.copy()
    reps = (37, 1000, 2500)
    fr[at: at + 12] = np.array(reps, "<u4").view(np.uint8)
    assert zd.libzstd_accepts(fr)
    seen = set()
    for d, cont, rp, kind in ((content, content, (1, 4, 8), zd.DCT_RAW), (fr, content, reps, zd.DCT_AUTO)):
        dct = z.ZstdDictionary(d)
        assert dct.info.content_bytes == C and dct.info.content_off == d.size - C
        assert tuple(np.frombuffer(dct.d_ddict.cpu().numpy().tobytes()[40:52], "<u4")) == tuple(rp)
        frames, srcs = [], []
        for i, (seqs, small) in enumerate(dictated_cases(C, rp, rng)):
            tail = int(rng.integers(0, 20))
            s = build(seqs, tail, cont, rng)
            seen |= edges_of(seqs, C, rp, small)
            frames.append(zd.compress(s, d, level=3, checksum=i & 1, kind=kind, seqs=seqs,
                                      params={zc.P_MAXBLOCK: MAXBLOCK} if small else None))
            srcs.append(s)
        check(frames, srcs, d, dct, seed=7)
        # the dictated frames at every output address mod 16: each behind a frame of 1..16 bytes that places it
        sub, subs, mine, cur = [], [], [], 0
        for r in range(16):
            ps = rng.integers(0, 256, (r - cur) % 16 or 16).astype(np.uint8)
            k = r % len(frames)
            sub += [zd.compress(ps, d, level=1, kind=kind), frames[k]]
            subs += [ps, srcs[k]]
            cur += ps.size + srcs[k].size
            mine.append(len(sub) - 1)
        routes, _ = check(sub, subs, d, dct, seed=8)
        for name, (_, _, oo) in routes.items():
            assert sorted(int(oo[i]) % 16 for i in mine) == list(range(16)), name
        seen.add("align")
    missing = set(EDGES) - seen
    assert not missing, missing


def test_many_small_frames_need_no_more_memory_than_without_a_dictionary():
    d = zd.train(51, 110 << 10)
    dct = z.ZstdDictionary(d)
    recs = zd.records(52, 3000, 200, 4096)
    frames = [zd.compress(r, d, level=3, dict_id_flag=0) for r in recs]
    cont = zd.container(frames)
    d_cont = torch.from_numpy(cont).cuda()
    with_d = z.ZstdDeviceDecompressor.from_device(d_cont, dictionary=dct)
    without = z.ZstdDeviceDecompressor.from_device(d_cont)
    assert with_d.work.numel() == without.work.numel() and with_d.out.numel() == without.out.numel()
    with_d.run(d_cont)
    outs, st, _ = outputs(with_d)
    assert (st == 0).all()
    assert all(np.array_equal(o, r) for o, r in zip(outs, recs))
    h = z.ZstdDeviceDecompressor(cont, dictionary=dct)
    assert h.work.numel() == without.work.numel()


# ---------------------------------------------------------------- rejections, against libzstd's verdicts
def test_a_frame_naming_another_dictionary_is_refused():
    d1 = zd.finalize(61, np.concatenate(zd.records(62, 30))[: 8 << 10], 12 << 10, dict_id=1001)
    d2 = zd.finalize(61, np.concatenate(zd.records(63, 30))[: 8 << 10], 12 << 10, dict_id=1002)
    r = zd.records(64, 3)
    frames = [zd.compress(r[0], d1), zd.compress(r[1], d2), zd.compress(r[2], d1)]
    assert zd.decompress(frames[1], d1, r[1].size)[0]                  # libzstd: dictionary_wrong
    dct = z.ZstdDictionary(d1)
    cont = zd.container(frames)
    h = z.ZstdDeviceDecompressor(cont, dictionary=dct)
    assert h.scan_status == [0, 13, 0]
    for plain in (False, True):
        s = zd.plain(frames) if plain else cont
        start = bytes(s).find(bytes(frames[1]))                        # bad_offset: the frame's start
        with pytest.raises(ValueError, match="dict_wrong in frame 1 at offset %d$" % start):
            z.ZstdDeviceDecompressor.from_device(torch.from_numpy(s).cuda(), plain=plain, dictionary=dct)


def test_a_dictionary_one_byte_short_fails_the_frame_that_reaches_its_first_byte():
    rng = np.random.default_rng(71)
    content = rng.integers(0, 256, 4096).astype(np.uint8)
    seqs = [(3, 4096 + 3, 40)]
    s = build(seqs, 10, content, rng)
    fr = zd.compress(s, content, kind=zd.DCT_RAW, seqs=seqs)
    assert zd.decompress(fr, content[1:], s.size)[0]                   # libzstd refuses the offset
    short = z.ZstdDictionary(content[1:])
    dec = z.ZstdDeviceDecompressor(zd.container([fr]), dictionary=short)
    dec.run(torch.from_numpy(zd.container([fr])).cuda())
    torch.cuda.synchronize()
    assert int(dec.status.cpu()[0]) == 5                               # ZMT_ST_BLOCK


def record_offsets(dct):
    """The table offsets of a loaded formatted dictionary, from the record (ZDDict in frame_format.h)."""
    raw = dct.d_ddict.cpu().numpy().tobytes()
    return np.frombuffer(raw[52:72], "<u4")                            # huf, of, ml, ll, rep


def test_corrupt_dictionaries_are_refused_where_libzstd_refuses_them():
    d = zd.finalize(81, np.concatenate(zd.records(82, 30))[: 8 << 10], 12 << 10, dict_id=9)
    huf, of, ml, ll, rep = (int(x) for x in record_offsets(z.ZstdDictionary(d)))
    assert huf == 8 and huf < of < ml < ll < rep
    bad = {}
    x = d.copy(); x[huf] = 0; bad["huffman_zero_header"] = x
    x = d.copy(); x[huf] = 255; bad["huffman_too_many_weights"] = x
    x = d.copy(); x[of] = (x[of] & 0xF0) | 0xF; bad["of_accuracy_log"] = x
    x = d.copy(); x[ml] = (x[ml] & 0xF0) | 0xF; bad["ml_accuracy_log"] = x
    x = d.copy(); x[ll] = (x[ll] & 0xF0) | 0xF; bad["ll_accuracy_log"] = x
    x = d.copy(); x[rep: rep + 4] = 0; bad["zero_repeat_offset"] = x
    x = d.copy(); x[rep + 4: rep + 8] = np.array([d.size], "<u4").view(np.uint8); bad["repeat_offset_past_content"] = x
    bad["truncated_in_tables"] = d[: (of + ml) // 2].copy()
    bad["truncated_before_repeats"] = d[: rep + 6].copy()
    for name, x in bad.items():
        assert not zd.libzstd_accepts(x), name
        with pytest.raises(ValueError, match="bad_header|truncated"):
            z.ZstdDictionary(x)
    assert zd.libzstd_accepts(d)
