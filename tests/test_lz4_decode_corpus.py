"""CPU tests of the LZ4 edge corpus (_lz4corpus.py): every block and frame is accepted by liblz4 and decodes to its source,
the oracle agrees, its trace is the dictated parse, and every case reaches the edges it exists for, stated on the trace
and on the Python models of the GPU decoder's two passes."""
import numpy as np
import pytest

import _lz4corpus as lc
import _oracle as o
import _zxmodel as zx
from _searchcorpus import kernel_constant

CASES = list(lc.CASES)
S, B = o.L4S, o.L4B


def test_liblz4_version():
    """The end-of-block rules the corpus relies on were checked against liblz4 1.9.x; another version may judge the
    corpus differently, which this names up front instead of as a corpus failure."""
    v = lc.lz4().LZ4_versionNumber()
    if v // 100 != 109:
        pytest.skip("liblz4 %d: the corpus was checked against 1.9.x" % v)


@pytest.mark.parametrize("lay", lc.LAYOUTS)
@pytest.mark.parametrize("name", CASES)
def test_corpus_is_accepted_by_liblz4_and_the_oracle(name, lay):
    """Every block decodes in liblz4 into a buffer of exactly its size (with the previous 64 KiB as dictionary when blocks
    are linked), every frame through LZ4F_decompress, both to the source; orc_lz4f_decode agrees and consumes the frame."""
    for (frame, src, info), tr in zip(lc.case(name, lay), lc.traces(name, lay)):
        linked = not (frame[4] & 0x20)
        for b, (rows, data, p) in enumerate(info):
            n = lc.regen(rows)
            if tr.blk[b, B["stored"]]:
                assert bytes(data) == src[p: p + n].tobytes()
                continue
            got = lc.liblz4_block(np.frombuffer(data, np.uint8), src[max(0, p - 65536): p] if linked else src[:0], n)
            assert got is not None and np.array_equal(got, src[p: p + n]), (name, lay, b)
        out, used = lc.liblz4_frame(frame, src.size)
        assert not isinstance(out, str), out
        assert used == frame.size and np.array_equal(out, src)
        rc, back, used = o.lz4f_decode(frame, src.size)
        assert rc == 0 and used == frame.size and np.array_equal(back, src)
        assert np.array_equal(tr.content, src) and tr.consumed == frame.size


@pytest.mark.parametrize("lay", lc.LAYOUTS)
@pytest.mark.parametrize("name", CASES)
def test_trace_is_the_dictated_parse(name, lay):
    """The oracle's trace gives back, block by block, the (ll, off, ml) rows the writer was given, the extension byte
    counts the lengths imply, and each match's destination."""
    for (frame, src, info), tr in zip(lc.case(name, lay), lc.traces(name, lay)):
        assert len(tr.blk) == len(info)
        for b, (rows, data, p) in enumerate(info):
            assert tr.blk[b, B["bsize"]] == len(data) and tr.blk[b, B["regen"]] == lc.regen(rows) and tr.blk[b, B["dst"]] == p
            sq = tr.block_seqs(b)
            if tr.blk[b, B["stored"]]:
                assert len(sq) == 0
                continue
            assert [tuple(int(x) for x in r) for r in sq[:, [S["ll"], S["off"], S["ml"]]]] == [tuple(r) for r in rows]
            ext = lambda n: 0 if n < 15 else (n - 15) // 255 + 1
            assert list(sq[:, S["llext"]]) == [ext(r[0]) for r in rows]
            assert list(sq[:, S["mlext"]]) == [ext(r[2] - 4) if r[2] else 0 for r in rows]
            dst = np.cumsum([0] + [r[0] + r[2] for r in rows])[:-1] + [r[0] for r in rows]
            assert list(sq[:, S["dst"]]) == list(dst)


def test_trace_pinned_on_liblz4_frames():
    """On frames liblz4 itself wrote (the reference's LZ4F_compressFrame, linked blocks): the trace's content equals
    orc_lz4f_decode's, and re-writing every block from its traced parse gives back the block's bytes."""
    if not o.have_ref():
        pytest.skip("reference library not built")
    import zstdmt_b200 as z
    src = z.gen_stream(z.GEN_MIX, (3 << 20) + 12345, 1 << 20)
    rc, framed, _ = o.ref_compress(o.CODEC_LZ4, src, threads=1, level=1, chunk=1 << 20)
    assert rc == 0
    pos = 0
    for frame in o.mt_frames(framed):
        tr = o.lz4f_trace(frame, 1 << 21)
        rc, back, used = o.lz4f_decode(frame, 1 << 21)
        assert rc == 0 and np.array_equal(tr.content, back) and used == tr.consumed == frame.size
        assert np.array_equal(back, src[pos: pos + back.size])
        for b in range(len(tr.blk)):
            foff, bs, p = (int(tr.blk[b, B[k]]) for k in ("foff", "bsize", "dst"))
            if tr.blk[b, B["stored"]]:
                continue
            rows = [tuple(int(x) for x in r) for r in tr.block_seqs(b)[:, [S["ll"], S["off"], S["ml"]]]]
            assert lc.write_block(rows, back, p) == frame[foff: foff + bs].tobytes()
        pos += back.size
    assert pos == src.size


# ---------------------------------------------------------------------------------------------------- edges
def _seqs(name, lay="full"):
    return np.concatenate([t.seq for t in lc.traces(name, lay)])


def _blocks(name, lay="full"):
    """(trace, block index, block_view) of every compressed block of a case."""
    for tr in lc.traces(name, lay):
        for b in range(len(tr.blk)):
            if not tr.blk[b, B["stored"]]:
                yield tr, b, lc.block_view(tr, b)


def _walk_a(name, lay="full"):
    """Pass A steps of every block, with the window end and each step's sequences (token, literal start, literal length,
    header end) in block coordinates."""
    for tr, b, (tok, bs, recs, abs_src) in _blocks(name, lay):
        sq = tr.block_seqs(b)
        for ip0, sh, i0, cnt, why in lc.step_walk_a(tok, bs, abs_src):
            wend = ip0 - sh + lc.LZD_WIN
            seqs = []
            for j in range(i0, i0 + cnt):
                r = sq[j]
                lit0 = tok[j] + 1 + int(r[S["llext"]])
                hend = lit0 + int(r[S["ll"]]) + (2 + int(r[S["mlext"]]) if r[S["ml"]] else 0)
                seqs.append((tok[j], lit0, int(r[S["ll"]]), hend))
            yield ip0, why, wend, seqs


def _steps_b(name, lay="full"):
    for tr, b, (tok, bs, recs, abs_src) in _blocks(name, lay):
        yield tr, b, recs, lc.steps_b(recs)


def edges_lengths():
    sq = _seqs("lengths")
    ll, ml = set(sq[:, S["ll"]].tolist()), set(sq[:, S["ml"]].tolist())
    m = sq[sq[:, S["ml"]] > 0]
    return {
        "ll 0-15, 269/270, 524/525": set(range(16)) | {269, 270, 524, 525} <= ll,
        "ll runs of 16/17, 63/64, 256/257": {16, 17, 63, 64, 256, 257} <= ll,
        "ll with >= 3 extension bytes": (sq[:, S["llext"]] >= 3).any(),
        "ml 4-19, 273, 274, 528/529": set(range(4, 20)) | {273, 274, 528, 529} <= ml,
        "ml 273 has one extension byte, 274 two": set(m[m[:, S["ml"]] == 273][:, S["mlext"]]) == {1} and set(m[m[:, S["ml"]] == 274][:, S["mlext"]]) == {2},
        "ml with >= 3 extension bytes": (sq[:, S["mlext"]] >= 3).any(),
    }


def edges_window():
    why, pos, cross, leave = set(), False, False, False
    for ip0, w, wend, seqs in _walk_a("window"):
        why.add(w)
        pos |= any(232 <= t - ip0 <= 255 for t, *_ in seqs)
        cross |= any(t < wend < hend for t, _, _, hend in seqs)
        leave |= any(l0 < wend < l0 + ll for _, l0, ll, _ in seqs)
    return {"steps ended by the 32-sequence cap": "cap" in why, "steps ended by the 256-byte limit": "span" in why,
            "tokens at chain positions 232-255": pos, "sequence headers crossing the staged window": cross,
            "literal runs leaving the window": leave}


def record_ranges(name, lay="full"):
    """Per block of each frame (alone behind a 12-byte header): the match-record range [(abs_src + 2) / 3, + nrec)."""
    for tr in lc.traces(name, lay):
        rs = []
        for b, (tok, bs, recs, abs_src) in ((b, lc.block_view(tr, b)) for b in range(len(tr.blk))):
            rs.append(((abs_src + 2) // 3, (abs_src + 2) // 3 + len(recs), bs, len(recs)))
        yield rs


def edges_dense():
    densest, gaps = False, []
    for rs in record_ranges("dense"):
        densest |= any(n == (bs - 6) // 3 and bs % 3 == 0 for _, _, bs, n in rs[1:])
        gaps += [rs[i + 1][0] - rs[i][1] for i in range(len(rs) - 1)]
    return {"blocks of 3-byte sequences only (nrec = (bs - 6) / 3, the densest liblz4 accepts)": densest,
            "neighbouring record ranges 3 records apart (the least a valid block allows)": min(gaps) == 3}


def edges_periods():
    sq = _seqs("periods")
    m = sq[sq[:, S["ml"]] > 0]
    pairs = set(map(tuple, m[:, [S["off"], S["ml"]]].tolist()))
    lone = {recs[st[3][0][0]][2] for _, _, recs, steps in _steps_b("periods") for st in steps if st[0] == "lone"}
    return {"offsets 1-33": set(range(1, 34)) <= set(m[:, S["off"]].tolist()),
            "off = ml - 1, ml, ml + 1": all((ml + d, ml) in pairs for ml in (8, 20, 33, 100) for d in (-1, 0, 1)),
            "lone matches > 2048 with offsets 1, 31, 32, 33, 2047, 65535": {1, 31, 32, 33, 2047, 65535} <= lone}


def edges_steps():
    exact, lone, nlow, ind, dep, mls = False, False, set(), False, False, set()
    for _, _, recs, steps in _steps_b("steps"):
        for i, (kind, d0, span, rs) in enumerate(steps):
            if kind == "lone":
                lone |= span > lc.LZX_SPAN
                continue
            if span == lc.LZX_SPAN and len(rs) < lc.LZD_SEQS and i + 1 < len(steps):
                nd, nml, _ = recs[rs[-1][0] + 1]
                exact |= nd - d0 == lc.LZX_SPAN + 1
            for k, (j, dp, own, nl) in enumerate(rs):
                d, ml, off = recs[j]
                if own:
                    nlow.add(nl); mls.add(ml)
                for dj, mj, _ in (recs[x[0]] for x in rs[:k]):
                    ind |= d - off + ml == dj and not dp and off >= ml
                    dep |= d - off + ml == dj + 1 and dp
            mls |= {recs[j][1] for j, dp, own, _ in rs if not own and not dp and recs[j][1] == 33}
    return {"a step spanning exactly 2048 bytes, the next record at 2049": exact, "a lone record longer than 2048": lone,
            "own-lane sources below d0, nlow 4-7, 8, 9-31": set(range(4, 32)) <= nlow,
            "source ending exactly at an earlier destination: independent": ind, "one byte later: dependent": dep,
            "ml 32 by its own lane, 33 by the warp": 32 in mls and 33 in mls}


def edges_linked():
    trs = lc.traces("linked")
    chain = trs[0]
    first = [chain.block_seqs(b)[0] for b in range(1, len(chain.blk)) if b != 20]
    dists = {int(r[S["off"]]) - int(r[S["dst"]]) for r in first}
    # every block after the first opens with reads of its predecessor, one of them of the predecessor's last 8 bytes
    tails = all(all(r[S["ml"]] and r[S["off"]] > r[S["dst"]] for r in chain.block_seqs(b)[:2])
                and any(-8 <= int(r[S["dst"]]) - int(r[S["off"]]) < 0 for r in chain.block_seqs(b)[:2])
                for b in range(1, len(chain.blk)))
    eq_hist = any(r[S["ml"]] and r[S["off"]] == r[S["dst"]] for r in chain.block_seqs(0))
    after = [False, False]
    long_prev = False
    for tr in trs:
        prev_pub = None
        for b, (tok, bs, recs, _) in ((b, lc.block_view(tr, b)) for b in range(len(tr.blk))):
            steps = lc.steps_b(recs)
            bm = lc.BLKMAX[(int(lc.case("linked")[trs.index(tr)][0][5]) >> 4) & 7]
            if b and prev_pub:
                need = [min(bm, bm + d - off + ml) for d, ml, off in recs if d - off < 0]
                for q in (0, 1):
                    after[q] |= len(prev_pub) > q and any(n > prev_pub[q] for n in need)
            long_prev |= b > 0 and any(d - off < 0 and ml > lc.LZX_SPAN for d, ml, off in recs)
            prev_pub = lc.publications(steps)
    stored = trs[1]
    bsids = {(int(f[5]) >> 4) & 7 for f, _, _ in lc.case("linked")}
    return {"first matches read the previous block at distances 1 .. 65535": {1, 2, 3, 4, 31, 32, 33, 2047, 65535} <= dists,
            "offset == op + hist": eq_hist, "a > 2048-byte match reading the previous block": long_prev,
            "previous-block reads beyond the 4th-step publication": after[0], "... and beyond the 8th": after[1],
            "a stored-raw predecessor read by the next block": bool(stored.blk[1, B["stored"]]) and stored.block_seqs(2)[0, S["off"]] > stored.block_seqs(2)[0, S["dst"]],
            "a chain of >= 60 linked 64 KiB blocks": len(chain.blk) >= 60 and (chain.col("regen")[:-1] == 65536).all(),
            "each block of the chain starts by reading its predecessor's last bytes": tails,
            "linked 256 KiB / 1 MiB / 4 MiB blocks": {5, 6, 7} <= bsids}


def edges_ends():
    trs = lc.traces("ends")
    frames = [f for f, _, _ in lc.case("ends")]
    last = []
    for tr in trs:
        for b in range(len(tr.blk)):
            sq = tr.block_seqs(b)
            if len(sq) >= 2:
                last.append((int(tr.blk[b, B["regen"]]) - int(sq[-2, S["dst"]]), int(sq[-1, S["ll"]])))
    full = {(int(f[5]) >> 4) & 7 for f, tr in zip(frames, trs) if len(tr.blk) == 1 and tr.blk[0, B["regen"]] == lc.BLKMAX[(int(f[5]) >> 4) & 7]}
    return {"last match starting exactly 12 bytes before the block end": any(s == 12 for s, _ in last),
            "a last literal run of exactly 5": any(ll == 5 for _, ll in last), "an extended last literal run": any(ll >= 15 for _, ll in last),
            "a block of exactly blockMaxSize for every size ID": full == {4, 5, 6, 7},
            "an empty frame": any(len(tr.blk) == 0 for tr in trs), "a frame with dictID": any(f[4] & 1 for f in frames),
            "a zero-size stored block between blocks": any(((tr.col("bsize")[:-1] == 0) & (tr.col("stored")[:-1] == 1)).any() for tr in trs),
            "a zero-size stored block before the end mark": any(len(tr.blk) and tr.blk[-1, B["bsize"]] == 0 and tr.blk[-1, B["stored"]] for tr in trs)}


EDGES = {"lengths": edges_lengths, "window": edges_window, "dense": edges_dense, "periods": edges_periods,
         "steps": edges_steps, "linked": edges_linked, "ends": edges_ends}


@pytest.mark.parametrize("name", CASES)
def test_case_reaches_its_edges(name):
    got = EDGES[name]()
    assert all(got.values()), [k for k, v in got.items() if not v]


@pytest.mark.parametrize("lay", lc.LAYOUTS)
@pytest.mark.parametrize("name", CASES)
def test_layouts_select_the_decoder_path(name, lay):
    """`full` frames keep every non-last block at blockMaxSize (two-pass path); `short` frames of two or more blocks do not
    (frame-sequential pass); a zero-size block sends its frame to the frame-sequential pass in either layout."""
    for (frame, _, _), tr in zip(lc.case(name, lay), lc.traces(name, lay)):
        assert lc.expect_fallback(tr, (int(frame[5]) >> 4) & 7) == lc.expect_path_is_sequential(lay, tr)


def test_own_lane_sources_never_straddle_d0():
    """Pass B's own-lane copy has a branch for a source that starts below d0 and ends above it.  The model shows why no
    stream reaches it: the step's first record starts at d0, so such a source touches that record's destination and the
    match is dependent.  Checked on every block of the corpus."""
    for name in CASES:
        for lay in lc.LAYOUTS:
            for _, _, recs, steps in _steps_b(name, lay):
                for kind, d0, _, rs in steps:
                    assert all(nl in (0, recs[j][1]) for j, _, own, nl in rs if own)


def test_model_constants_match_the_kernel():
    """The models' constants are the ones the source states: pass B's step cap, span and own-lane limit are
    match_exec.cuh's (shared with the zstd execute pass), pass A's are lz4_decode.cuh's.  A change in either fails here
    instead of the model quietly following the code."""
    files = ("match_exec.cuh", "lz4_decode.cuh")
    got = {n: kernel_constant(n, files) for n in ("MX_STEP", "MX_SPAN", "MX_OWN", "MX_INACTIVE", "LZD_WIN", "LZD_NJ", "LZD_LONGLIT")}
    assert got == {"MX_STEP": lc.LZD_SEQS, "MX_SPAN": lc.LZX_SPAN, "MX_OWN": lc.LZD_LONG, "MX_INACTIVE": zx.INACTIVE,
                   "LZD_WIN": lc.LZD_WIN, "LZD_NJ": lc.LZD_NJ, "LZD_LONGLIT": lc.LZD_LONGLIT}
    assert (lc.LZD_SEQS, lc.LZX_SPAN, lc.LZD_LONG) == (zx.STEP_CAP, zx.ZX_SPAN, zx.OWN_ML)


def test_dependency_search_agrees_with_the_overlap_on_every_step():
    """steps_b states dependence as the pairwise overlap with the step's earlier destinations; the kernel finds it by a
    lower-bound search over the lanes (mx_independent, restated as _zxmodel.kernel_dependent).  The two agree on every
    record of every step of the corpus, with the inactive lanes the kernel pads with."""
    n = 0
    for name in CASES:
        for lay in lc.LAYOUTS:
            for _, _, recs, steps in _steps_b(name, lay):
                for kind, _, _, rs in steps:
                    if kind != "step":
                        continue
                    pad = [zx.INACTIVE] * (lc.LZD_SEQS - len(rs))
                    d_beg = [recs[j][0] for j, *_ in rs] + pad
                    e_end = [recs[j][0] + recs[j][1] for j, *_ in rs] + pad
                    for lane, (j, dep, _, _) in enumerate(rs):
                        d, ml, off = recs[j]
                        assert zx.kernel_dependent(lane, d - off, ml, d_beg, e_end) == dep, (name, lay, j)
                        n += 1
    assert n


def test_block_ending_with_a_match_is_rejected():
    """A block must end with a literals-only sequence.  One that ends right after a match (token 0x84, 8 literals,
    offset 4: an 8-byte match and nothing behind it) is rejected by liblz4, by orc_lz4f_decode and by orc_lz4f_trace."""
    blk = bytes([0x84]) + b"abcdefgh" + (4).to_bytes(2, "little")
    assert lc.liblz4_block(np.frombuffer(blk, np.uint8), np.zeros(0, np.uint8), 16) is None
    hd = bytes([0x60, 0x40])
    frame = np.frombuffer((0x184D2204).to_bytes(4, "little") + hd + bytes([(o.xxh32(np.frombuffer(hd, np.uint8)) >> 8) & 0xFF])
                          + len(blk).to_bytes(4, "little") + blk + bytes(4), np.uint8)
    assert isinstance(lc.liblz4_frame(frame, 16)[0], str)
    assert o.lz4f_decode(frame, 16)[0] == -5
    with pytest.raises(ValueError):
        o.lz4f_trace(frame, 16)
