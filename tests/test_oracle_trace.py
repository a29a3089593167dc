"""CPU tests of the oracle's zstd block trace (orc_zstd_trace) and of the Python restatements in _zenc.py that the GPU
encoder tests (test_gpu_zstd_encoder.py) hold the encoder to."""
import json
import os

import numpy as np
import pytest

import _oracle as o
import _zenc as ze
import zstdmt_b200 as z

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ZT = o.ZT


def zstd_cases():
    with open(os.path.join(GOLD, "manifest.json")) as f:
        return [c for c in json.load(f)["cases"] if c["codec"] == "zstd"]


def replay(frame, tr):
    """Rebuild a frame's content from its trace alone: raw blocks from the frame bytes, RLE blocks from their byte,
    compressed blocks from the traced literals and sequences, with the repeat offsets resolved here (RFC 8878 §3.1.2.5)
    and checked against the oracle's."""
    frame = np.asarray(frame)
    payload = [int(b) if t != 1 else 1 for t, b in zip(tr.col("type"), tr.col("bsize"))]
    chk = 4 if (frame[4] >> 2) & 1 else 0
    pos = tr.consumed - chk - sum(3 + p for p in payload)            # frame header size
    out, rep = bytearray(), [1, 4, 8]
    for b in range(len(tr.blk)):
        t, bs = int(tr.blk[b, ZT["type"]]), int(tr.blk[b, ZT["bsize"]])
        pos += 3
        if t == 0:
            out += frame[pos: pos + bs].tobytes()
        elif t == 1:
            out += bytes([int(frame[pos])]) * bs
        else:
            start = len(out)
            lits = tr.block_lits(b).tobytes(); lp = 0
            for ll, ofv, ml, off in tr.block_seqs(b).tolist():
                if ofv > 3:
                    res = ofv - 3; rep = [res, rep[0], rep[1]]
                else:
                    idx = ofv + (ll == 0)
                    if idx == 1:
                        res = rep[0]
                    else:
                        res = rep[0] - 1 if idx == 4 else rep[idx - 1]
                        rep = [res, rep[0], rep[2]] if idx == 2 else [res, rep[0], rep[1]]
                assert res == off, (b, ll, ofv, ml, off, res)
                out += lits[lp: lp + ll]; lp += ll
                for _ in range(ml):
                    out.append(out[-res])
            out += lits[lp:]
            assert len(out) - start == tr.blk[b, ZT["regen"]]
        pos += payload[b]
    assert pos + chk == tr.consumed
    return np.frombuffer(bytes(out), np.uint8)


@pytest.mark.parametrize("case", zstd_cases(), ids=lambda c: c["file"])
def test_trace_replay_reproduces_golden_content(case):
    framed = np.fromfile(os.path.join(GOLD, case["file"]), dtype=np.uint8)
    src = z.gen_stream(case["kind"], case["n"], case["chunk"], first=case["first"])
    frames = o.mt_frames(framed)
    assert len(frames) == case["frames"]
    got = []
    for f in frames:
        tr = o.zstd_trace(f)
        assert tr.consumed == f.size
        assert np.array_equal(replay(f, tr), tr.content)
        # the trace's own bookkeeping: regenerated sizes add up, only the last block is flagged last
        assert tr.col("regen").sum() == tr.content.size
        assert list(tr.col("last")) == [0] * (len(tr.blk) - 1) + [1]
        got.append(tr.content)
    assert np.array_equal(np.concatenate(got) if got else np.zeros(0, np.uint8), src)


def test_trace_level19_shows_described_tables_then_treeless_and_repeat():
    """zstd_l19_k2_131584.bin: libzstd level 19, one frame of two blocks.  Block 0 describes its sequence tables
    (FSE_Compressed_Mode) and its Huffman tree; block 1 reuses the tree (treeless literals) and the tables (Repeat_Mode)."""
    framed = np.fromfile(os.path.join(GOLD, "zstd_l19_k2_131584.bin"), dtype=np.uint8)
    (f,) = o.mt_frames(framed)
    tr = o.zstd_trace(f)
    assert list(tr.col("type")) == [2, 2]
    m0, m1 = (int(x) for x in tr.col("modes"))
    fields = lambda m: [(m >> 6) & 3, (m >> 4) & 3, (m >> 2) & 3]
    assert 2 in fields(m0)
    assert 3 in fields(m1)
    assert tr.blk[0, ZT["lit_type"]] == 2 and tr.blk[1, ZT["lit_type"]] == 3
    assert tr.blk[0, ZT["tree_form"]] in (0, 1) and tr.blk[1, ZT["tree_form"]] == -1
    assert tr.blk[0, ZT["maxbits"]] == tr.blk[1, ZT["maxbits"]]           # the treeless block decodes with block 0's tree
    w = tr.weights[0]
    mb = int(tr.blk[0, ZT["maxbits"]])
    assert sum(1 << (int(x) - 1) for x in w if x) == 1 << mb                # the traced weights form a complete code
    # repeat offsets are in use: some Offset_Value is a repeat code (1..3)
    assert (tr.seq[:, 1] <= 3).any()


@pytest.mark.parametrize("case", zstd_cases(), ids=lambda c: c["file"])
def test_trace_on_and_off_decode_identically(case):
    framed = np.fromfile(os.path.join(GOLD, case["file"]), dtype=np.uint8)
    rc, plain = o.orc_decode(o.CODEC_ZSTD, framed, case["n"])
    assert rc == 0
    traced = np.concatenate([o.zstd_trace(f).content for f in o.mt_frames(framed)])
    assert np.array_equal(plain, traced)


def test_trace_reports_full_arrays_as_an_error():
    framed = np.fromfile(os.path.join(GOLD, "zstd_l3_k2_196613.bin"), dtype=np.uint8)
    f = o.mt_frames(framed)[0]
    with pytest.raises(ValueError):
        o.zstd_trace(f, out_cap=1000)


# ---- the Huffman rule of zstd_entropy.cuh, restated -----------------------------------------------------------------------
def fib_hist(k, scale=1):
    h = np.zeros(256, np.int64)
    a, b = 1, 1
    for s in range(k):
        h[(s * 37) % 256] = a * scale
        a, b = b, a + b
    return h


@pytest.mark.parametrize("k", [2, 3, 12, 13, 14, 20, 30])
def test_huffman_twin_is_complete_and_limited(k):
    h = fib_hist(k)
    ln, mb = ze.huf_lengths(h)
    _, unl = ze.huf_lengths(h, limit=False)
    assert unl == max(1, k - 1)                                  # Fibonacci counts give the deepest possible tree
    assert mb == min(unl, 11) and max(ln.values()) == mb
    assert ze.kraft(ln, mb) == 1 << mb
    assert set(ln) == set(np.flatnonzero(h).tolist())


def test_huffman_twin_random_skewed_histograms():
    """Kraft-complete and within 11 bits on skewed histograms, and an optimal (minimum-cost) code whenever the limiter
    does not engage."""
    import heapq
    rng = np.random.default_rng(7)
    engaged = 0
    for trial in range(300):
        k = int(rng.integers(2, 257))
        h = np.zeros(256, np.int64)
        syms = rng.choice(256, k, replace=False)
        h[syms] = np.maximum(1, (rng.pareto(0.6 + trial % 5 * 0.3, k) * 10).astype(np.int64))
        ln, mb = ze.huf_lengths(h)
        _, unl = ze.huf_lengths(h, limit=False)
        engaged += unl > 11
        assert mb <= 11 and ze.kraft(ln, mb) == 1 << mb
        if unl <= 11:
            q = [int(c) for c in h[h > 0]]; heapq.heapify(q); cost = 0
            while len(q) > 1:
                a = heapq.heappop(q); b = heapq.heappop(q); cost += a + b; heapq.heappush(q, a + b)
            assert sum(int(h[s]) * x for s, x in ln.items()) == cost
    assert engaged > 20


def test_lz4_twin_parse_replays_the_window():
    """_zenc.lz4_sequences read back: literals between the matches plus the matches rebuild the window."""
    src = z.gen_stream(z.GEN_MIX, 3 * ze.WINDOW, 1 << 20, first=1)
    for w in range(3):
        win = src[w * ze.WINDOW: (w + 1) * ze.WINDOW]
        seqs = ze.lz4_sequences(ze.lz4_twin_block(win))
        assert len(seqs) > 100
        out = bytearray(); p = 0
        for s, off, ml in seqs.tolist():
            out += win[p:s].tobytes()
            for _ in range(ml):
                out.append(out[-off])
            p = s + ml
        out += win[p:].tobytes()
        assert bytes(out) == win.tobytes()
        parts = ze.window_model(win)
        assert parts[0][0] == 0 and parts[-1][1] == win.size
        assert sum(len(s) for _, _, s in parts) == len(seqs)
